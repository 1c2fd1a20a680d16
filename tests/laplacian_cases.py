"""One table of cv::Laplacian(src, dst, ddepth, ksize, scale, delta, borderType) cases, aimed at the places where the reference's code
or the device's kernels change (opencv_b200/csrc/laplacian.cu):

  sizes     1x1, 1xN, Nx1, 3x4 (smaller than every aperture from 5 on), 31 / 32 / 33 rows and columns (the fused kernel's 32 x 32
            tile +-1), widths 4k..4k+3, one 2160 x 3840
  apertures 1, 3 (filter2D with the scaled 3x3 kernel), 5 (the 16S working depth for 8-bit sources; the float source's special row
            case that skips the zero taps of [1 0 -2 0 1]), 7, 9, 15, 31 (the 32F working depth)
  depths    8U -> 8U / 16S / 32F and 32F -> 32F, 1 to 4 channels
  borders   CONSTANT, REPLICATE, REFLECT, REFLECT_101, some with ISOLATED
  scale     (1, 0) (plain saturate_cast), (0.5, 0.5) and (1, 0.5) (convertTo on .5 rounding ties), (37, -3) (saturates 8U and 16S),
            (-0.25, 10.5) (negative scale)
  contents  random, constant, impulses, checkerboards; float images with +-inf, NaN, -0.0 and subnormals on a sparse lattice, so that
            some sit where only zero taps reach
  refusals  ksize 0, 2, 4, -1, 33 (the reference asserts: no result)

Results are compared with the reference outside its unrestated scalar remainders (remainder_start).
Both CPU oracles share one signature: oracle/_build/liboracle_port.so (port_laplacian, oracle/port/port_laplacian.c) and
oracle/_ref/liblapref.so (ref_laplacian, the reference itself, tests/cpp/laplacian_ref_shim.cpp, built by tools/build_laplacian_ref.py);
run() calls either.
Every case is plain data; its pixels come from PCG64 seeded by the SHA-256 of its image id, so every machine builds the same bytes.
"""
import ctypes
import hashlib
import os
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PORT_LIB = os.path.join(ROOT, "oracle", "_build", "liboracle_port.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "liblapref.so")
REF_HAL_LIB = os.path.join(ROOT, "oracle", "_ref", "liblapref_hal.so")     # against the reference built with this project's HAL

CV_8U, CV_16S, CV_32F = 0, 3, 5
BORDERS = (0, 1, 2, 4)              # CONSTANT, REPLICATE, REFLECT, REFLECT_101
ISOLATED = 16
APERTURES = (1, 3, 5, 7, 9, 15, 31)
PAIRS = ((CV_8U, CV_8U), (CV_8U, CV_16S), (CV_8U, CV_32F), (CV_32F, CV_32F))
SCALES = ((1.0, 0.0), (0.5, 0.5), (1.0, 0.5), (37.0, -3.0), (-0.25, 10.5))
BAD_KSIZES = (0, 2, 4, -1, 33)
NP = {CV_8U: np.uint8, CV_16S: np.int16, CV_32F: np.float32}

Image = namedtuple("Image", "id shape cn depth fill")
Case = namedtuple("Case", "id image ddepth ksize scale delta border")


def _images():
    out = []
    shapes = [(1, 1), (1, 37), (37, 1), (3, 4), (31, 33), (33, 31), (32, 32), (9, 20), (9, 21), (9, 22), (9, 23), (40, 70)]
    fills8 = ("random", "const", "impulse", "checker")
    for i, shape in enumerate(shapes):
        cn = 1 + i % 4
        for depth in (CV_8U, CV_32F):
            fills = fills8[i % 4:i % 4 + 1] + ("random",) if depth == CV_8U else ("random", "special")
            for fill in dict.fromkeys(fills):
                out.append(Image("%dx%dc%d-%s-%s" % (shape[0], shape[1], cn, "8u" if depth == CV_8U else "32f", fill), shape, cn, depth, fill))
    for cn in (1, 3):
        out.append(Image("40x70c%d-8u-impulse" % cn, (40, 70), cn, CV_8U, "impulse"))
        out.append(Image("40x70c%d-32f-checker" % cn, (40, 70), cn, CV_32F, "checker"))
    out.append(Image("2160x3840c1-8u-random", (2160, 3840), 1, CV_8U, "random"))
    out.append(Image("2160x3840c1-32f-special", (2160, 3840), 1, CV_32F, "special"))
    return out


IMAGES = _images()


def _cases():
    out = []
    for n, img in enumerate(IMAGES):
        big = img.shape[0] * img.shape[1] > 1 << 20
        for ai, k in enumerate(APERTURES):
            if big and k not in (1, 3, 5, 7, 31):
                continue
            for pi, (sd, dd) in enumerate(PAIRS):
                if sd != img.depth:
                    continue
                b = BORDERS[(ai + pi + n) % 4] | (ISOLATED if (ai + pi + n) % 5 == 0 else 0)
                sc, de = SCALES[(ai * 4 + pi + n) % len(SCALES)]
                out.append(Case("%s-k%d-d%d-b%d-s%g_%g" % (img.id, k, dd, b, sc, de), img, dd, k, sc, de, b))
                if not big and (sc, de) != (1.0, 0.0):
                    out.append(Case("%s-k%d-d%d-b%d-s1_0" % (img.id, k, dd, b), img, dd, k, 1.0, 0.0, b))
    for img in IMAGES[:4]:
        for k in BAD_KSIZES:
            out.append(Case("%s-k%d-refused" % (img.id, k), img, -1, k, 1.0, 0.0, 4))
    return out


CASES = _cases()


def rng_of(image_id):
    return np.random.Generator(np.random.PCG64(int.from_bytes(hashlib.sha256(image_id.encode()).digest()[:8], "little")))


def image_of(img):
    """the image's pixels, (H, W) for one channel, (H, W, C) otherwise"""
    H, W = img.shape
    g = rng_of(img.id)
    shape = (H, W) if img.cn == 1 else (H, W, img.cn)
    f8 = img.depth == CV_8U
    if img.fill == "const":
        a = np.full(shape, 173 if f8 else -3.75, NP[img.depth])
    elif img.fill == "impulse":
        a = np.zeros(shape, NP[img.depth])
        n = max(1, H * W // 97)
        a[g.integers(0, H, n), g.integers(0, W, n)] = 255 if f8 else 1e30
    elif img.fill == "checker":
        y, x = np.mgrid[0:H, 0:W]
        a = np.where(((y + x) & 1)[..., None] if img.cn > 1 else (y + x) & 1, 255 if f8 else 2.5e3, 0).astype(NP[img.depth])
        a = np.broadcast_to(a, shape).copy()
    elif f8:
        a = g.integers(0, 256, shape, dtype=np.uint8)
    else:
        a = (g.standard_normal(shape) * np.exp2(g.integers(-8, 12, shape))).astype(np.float32)
        if img.fill == "special":
            flat = a.reshape(-1, img.cn)
            y, x = np.divmod(np.arange(H * W), W)
            lat = np.flatnonzero((y % 7 == 3) & (x % 5 == 2))
            specials = np.array([np.inf, -np.inf, np.nan, -0.0, 1e-40, -3e-39], np.float32)
            flat[lat] = specials[np.arange(len(lat)) % len(specials)][:, None]
    return np.ascontiguousarray(a)


def digest(out):
    """'refused', or the SHA-256 of the result's bytes, every NaN written as the same quiet NaN (the payload is not part of the result)"""
    if out is None:
        return "refused"
    out = np.array(out)
    if out.dtype == np.float32:
        out[np.isnan(out)] = np.float32(np.nan)
    return hashlib.sha256(out.tobytes()).hexdigest()


def same_bits(got, want):
    """equal bit for bit, except that any NaN equals any NaN (the device's NaN payload is canonical)"""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.dtype != np.float32:
        return np.array_equal(got, want)
    gn, wn = np.isnan(got), np.isnan(want)
    return np.array_equal(gn, wn) and np.array_equal(got.view(np.int32)[~gn], want.view(np.int32)[~wn])


def remainder_start(img, ksize):
    """first element of a row (of cols * cn) that the reference computes in a scalar remainder loop whose rounding the port does not
    restate, or None: the float-working rows at ksize >= 7 (RowFilter after RowVec_32f's 8 lanes or RowVec_8u32f's 32, and the
    column filter's remainder) and filter2D's float remainder at ksize 1 / 3.  The 32F ksize 5 remainder is restated exactly."""
    we = img.shape[1] * img.cn
    if img.depth == CV_32F and ksize != 5:
        return we - we % 8
    if img.depth == CV_8U and ksize >= 7:
        return we - we % 32
    return None


def masked(img, ksize, out):
    """out with the elements from remainder_start on set to zero (for digests and the port-to-reference comparison)"""
    if out is None:
        return None
    v = remainder_start(img, ksize)
    if v is None:
        return out
    flat = np.array(out).reshape(out.shape[0], -1)
    flat[:, v:] = 0
    return flat.reshape(out.shape)


def ref_available(kind="ref"):
    return os.path.exists(REF_HAL_LIB if kind == "ref_hal" else REF_LIB)


_LIBS = {}


def run(kind, img, ddepth, ksize, scale=1.0, delta=0.0, border=4):
    """cv::Laplacian of a whole image by the port ("port"), the reference ("ref") or the HAL-built reference ("ref_hal"): the result,
    or None where the arguments are refused"""
    if kind not in _LIBS:
        path, name = {"port": (PORT_LIB, "port_laplacian"), "ref": (REF_LIB, "ref_laplacian"), "ref_hal": (REF_HAL_LIB, "ref_laplacian")}[kind]
        _LIBS[kind] = getattr(ctypes.CDLL(path), name)
    src = np.ascontiguousarray(img)
    depth = {np.dtype(np.uint8): CV_8U, np.dtype(np.uint16): 2, np.dtype(np.int16): CV_16S, np.dtype(np.float32): CV_32F}[src.dtype]
    cn = 1 if src.ndim == 2 else src.shape[2]
    dst = np.empty(src.shape, src.dtype if ddepth < 0 else NP[ddepth])
    h, w = src.shape[:2]
    vp, sz, dbl = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_double
    rc = _LIBS[kind](src.ctypes.data_as(vp), sz(src.strides[0]), dst.ctypes.data_as(vp), sz(dst.strides[0]), w, h, depth + ((cn - 1) << 3),
                     int(ddepth), int(ksize), dbl(scale), dbl(delta), int(border))
    return None if rc != 0 else dst
