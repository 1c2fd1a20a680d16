"""One table of cv::distanceTransform(src, dst, distanceType, maskSize, dstType) cases for 8UC1 sources, aimed at the places where the
reference's code or the device's kernels change (opencv_b200/csrc/distance.cu):

  sizes    1x1, 1xN, Nx1, odd small sizes; widths 31-33 and 63-65 (the row pass's 32-lane chunks); widths and heights 4095-4099 (the
           chamfer's 4096-column tile, d^2 above 2^24 in the column pass, rows over 4096 in the row pass); 19 370 / 19 371 columns (the
           row pass's stacks leave shared memory); 4200 x 4200 with a few zeros (chamfer distances above 256 pixels, where (float)t0
           rounds, and squares above 2^24); 1 x 70 000 and 70 000 x 1 (the second envelope loop, from column 65 536 on, and the squares
           that saturate at 65 536); 3 x 70 000 with sparse zeros (an intersection that rounds onto a whole column where the two
           parabolas differ, so `z[k+1] < q` and `<=` give different answers); a 2160 x 3840 edge map
  content  no zero pixel, all zero, a single zero at each corner and in the centre, sparse and dense random zeros, lines, Canny-like
           edge maps (one-pixel contours of a smooth random field), planted ties (zeros on a lattice and in mirrored pairs)
  calls    every row of the reference's table: the four modes on every image (C / L1 / L2 3x3, L2 5x5, precise, 8-bit L1), and on a few
           small images the forced and quirk rows (C and L1 with masks 5 and 0, precise with L12 / FAIR / WELSCH / HUBER / USER, the 8-bit
           L1 call with masks 0 and 7, an 8-bit request with L2, which gives 32F) and the refusals

Every case is plain data; its pixels come from PCG64 seeded by the SHA-256 of its image id, so every machine builds the same bytes.
Both CPU oracles share one signature: oracle/_build/liboracle_port.so (port_distance_transform, oracle/port/port_distance.c) and
oracle/_ref/libdistref.so (ref_distance_transform, the reference itself, tests/cpp/dist_ref_shim.cpp, built by tools/build_dist_ref.py).
"""
import ctypes
import hashlib
import os
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PORT_LIB = os.path.join(ROOT, "oracle", "_build", "liboracle_port.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libdistref.so")

DIST_USER, DIST_L1, DIST_L2, DIST_C, DIST_L12, DIST_FAIR, DIST_WELSCH, DIST_HUBER = -1, 1, 2, 3, 4, 5, 6, 7
CV_8U, CV_32F = 0, 5

# name -> (distanceType, maskSize, dstType)
MODES = {"c3": (DIST_C, 3, CV_32F), "l1_3": (DIST_L1, 3, CV_32F), "l2_3": (DIST_L2, 3, CV_32F), "l2_5": (DIST_L2, 5, CV_32F),
         "precise": (DIST_L2, 0, CV_32F), "l1_u8": (DIST_L1, 3, CV_8U)}
QUIRKS = {"c5": (DIST_C, 5, CV_32F), "c0": (DIST_C, 0, CV_32F), "l1_5": (DIST_L1, 5, CV_32F), "l1_0": (DIST_L1, 0, CV_32F),
          "l12_0": (DIST_L12, 0, CV_32F), "fair_0": (DIST_FAIR, 0, CV_32F), "welsch_0": (DIST_WELSCH, 0, CV_32F),
          "huber_0": (DIST_HUBER, 0, CV_32F), "user_0": (DIST_USER, 0, CV_32F), "l1_u8_m0": (DIST_L1, 0, CV_8U),
          "l1_u8_m7": (DIST_L1, 7, CV_8U), "l2_3_u8": (DIST_L2, 3, CV_8U)}
REFUSED = {"l2_7": (DIST_L2, 7, CV_32F), "c4": (DIST_C, 4, CV_32F), "l12_3": (DIST_L12, 3, CV_32F), "user_5": (DIST_USER, 5, CV_32F),
           "huber_3": (DIST_HUBER, 3, CV_32F), "l2_1_u8": (DIST_L2, 1, CV_8U)}
CALLS = dict(MODES, **QUIRKS, **REFUSED)

Case = namedtuple("Case", "id image shape fill call")          # image: id of the source image; call: a key of CALLS

SMALL_FILLS = ("none", "zero", "tl", "tr", "bl", "br", "center", "sparse", "dense", "lines", "edges", "ties")


def _cases():
    images = []
    for shape in [(1, 1), (1, 7), (7, 1), (1, 33), (33, 1), (3, 5), (5, 3), (7, 9), (13, 11), (31, 17), (64, 96)]:
        images += [(shape, f) for f in SMALL_FILLS]
    for w in (31, 32, 33, 63, 64, 65):
        images += [((5, w), f) for f in ("sparse", "ties", "edges")]
    images += [((120, 257), f) for f in ("sparse", "edges", "ties", "lines")]
    images += [((300, 300), f) for f in ("tl", "center", "few")]
    for n in range(4095, 4100):
        images += [((3, n), "tl"), ((n, 3), "tl"), ((2, n), "few")]
    images += [((2, 19370), "sparse"), ((2, 19371), "sparse"), ((2, 19371), "none")]
    images += [((4200, 4200), "few"), ((1, 70000), "few"), ((70000, 1), "few"), ((1, 70000), "tl"), ((70000, 1), "br"), ((3, 70000), "sparse")]
    images += [((2160, 3840), "edges")]
    out = []
    for shape, fill in images:
        img = "%dx%d-%s" % (shape[0], shape[1], fill)
        for m in MODES:
            out.append(Case("%s-%s" % (img, m), img, shape, fill, m))
    for shape, fill in [((13, 11), "sparse"), ((7, 9), "none"), ((31, 17), "ties")]:
        img = "%dx%d-%s" % (shape[0], shape[1], fill)
        for m in list(QUIRKS) + list(REFUSED):
            out.append(Case("%s-%s" % (img, m), img, shape, fill, m))
    return out


def rng_of(image_id):
    return np.random.Generator(np.random.PCG64(int.from_bytes(hashlib.sha256(image_id.encode()).digest()[:8], "little")))


def image_of(case):
    """the case's 8UC1 source (H, W)"""
    H, W = case.shape
    g = rng_of(case.image)
    img = g.integers(1, 256, (H, W), dtype=np.uint8)
    f = case.fill
    if f == "none":
        return img
    if f == "zero":
        return np.zeros((H, W), np.uint8)
    corners = {"tl": (0, 0), "tr": (0, W - 1), "bl": (H - 1, 0), "br": (H - 1, W - 1), "center": (H // 2, W // 2)}
    if f in corners:
        img[corners[f]] = 0
        return img
    if f == "sparse":
        img[g.random((H, W)) < 0.01] = 0
        return img
    if f == "dense":
        img[g.random((H, W)) < 0.5] = 0
        return img
    if f == "few":                 # 1 to 5 zeros within the first tenth of each axis
        n = int(g.integers(1, 6))
        img[g.integers(0, max(1, H // 10), n), g.integers(0, max(1, W // 10), n)] = 0
        return img
    if f == "lines":               # horizontal, vertical and diagonal lines of zeros
        y, x = np.mgrid[0:H, 0:W]
        for _ in range(3):
            kind, c = int(g.integers(0, 3)), int(g.integers(0, max(H, W)))
            img[(y == c % H) if kind == 0 else (x == c % W) if kind == 1 else (x - y == c - max(H, W) // 2)] = 0
        return img
    if f == "edges":               # one-pixel contours of a smooth random field, as an inverted edge map (0 on edges, 255 elsewhere)
        cell = 12
        coarse = g.random((H // cell + 2, W // cell + 2))
        yy, xx = np.mgrid[0:H, 0:W] / cell
        y0, x0 = yy.astype(int), xx.astype(int)
        fy, fx = yy - y0, xx - x0
        field = (coarse[y0, x0] * (1 - fy) * (1 - fx) + coarse[y0 + 1, x0] * fy * (1 - fx) + coarse[y0, x0 + 1] * (1 - fy) * fx
                 + coarse[y0 + 1, x0 + 1] * fy * fx)
        inside = field > 0.5
        edge = np.zeros((H, W), bool)
        edge[:, :-1] |= inside[:, :-1] != inside[:, 1:]
        edge[:-1, :] |= inside[:-1, :] != inside[1:, :]
        return np.where(edge, 0, 255).astype(np.uint8)
    if f == "ties":                # zeros on a lattice and in mirrored pairs: many pixels equally far from two or more zeros
        sy, sx = (int(v) for v in g.integers(2, 9, 2))
        oy, ox = int(g.integers(0, sy)), int(g.integers(0, sx))
        img[oy::sy, ox::sx] = 0
        for _ in range(3):
            cy, cx, k = int(g.integers(0, H)), int(g.integers(0, W)), int(g.integers(1, 6))
            for dy, dx in ((-k, 0), (k, 0), (0, -k), (0, k)):
                if 0 <= cy + dy < H and 0 <= cx + dx < W:
                    img[cy + dy, cx + dx] = 0
        return img
    raise ValueError(f)


CASES = _cases()
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)


def out_is_u8(call):
    dist_type, _, dst_type = CALLS[call]
    return dist_type == DIST_L1 and dst_type == CV_8U


_libs = {}


def _lib(path, name):
    if path not in _libs:
        L = ctypes.CDLL(path)
        fn = getattr(L, name)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                       ctypes.c_int, ctypes.c_int]
        _libs[path] = fn
    return _libs[path]


def port_available():
    return os.path.exists(PORT_LIB)


def ref_available():
    return os.path.exists(REF_LIB)


def run(which, img, call):
    """(depth, result) from the port or the reference; (-1, None) where the arguments are refused"""
    fn = _lib(PORT_LIB, "port_distance_transform") if which == "port" else _lib(REF_LIB, "ref_distance_transform")
    img = np.ascontiguousarray(img, np.uint8)
    H, W = img.shape
    out = np.zeros((H, W), np.uint8 if out_is_u8(call) else np.float32)
    dt, mask, dst_type = CALLS[call]
    depth = fn(img.ctypes.data, img.strides[0], out.ctypes.data, out.strides[0], W, H, dt, mask, dst_type)
    return (depth, out) if depth >= 0 else (-1, None)


def digest(depth, out):
    if depth < 0:
        return "refused"
    return "%d:%s" % (depth, hashlib.sha256(np.ascontiguousarray(out).tobytes()).hexdigest())
