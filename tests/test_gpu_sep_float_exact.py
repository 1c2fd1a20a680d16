"""The float separable path held to the C port (oracle/port/port_filter.c, sep_float) bit for bit, over the WHOLE destination.

Four kernels run float separable arithmetic: sep_f32_tile_kernel (sep_f32.cu, 1 channel, centred, odd taps, (anti)symmetric columns,
TMA-addressable rows, bucket KB <= 11), sep_f32_tma_kernel (the same from KB = 13 on; it walks nch = 1, 2 or 4 chunks of 32 rows),
sep_fast_kernel<., ., M_FLOAT, KB> (sepfilter.cu: 1 channel, centred, rows that TMA cannot address, BORDER_WRAP, images smaller than
KB) and sep_generic_kernel<., ., M_FLOAT> (channels, anchors, even sizes, asymmetric columns, 33 taps).  The port evaluates every
element, remainder columns included, with the formulas the kernels use, so the device must equal it everywhere.  The comparisons with the
reference itself (test_gpu_filters.py, test_gpu_features.py) hold only the reference's SIMD body exactly.

Equality here is value equality with equal NaN masks: +0 and -0 compare equal, every other float must have the same bits.

predict() restates the dispatch of sep_filter_impl / sep_float_fast / sep_dispatch / launch_sf32, so each test says which kernel it
means; test_predicted_kernel_runs checks the prediction with torch.profiler.
"""
import math

import numpy as np
import pytest

import opencv_b200 as C
from util import cpu, gpu

pytestmark = pytest.mark.gpu

CONST, REPL, REFL, WRAP, R101 = 0, 1, 2, 3, 4
MIRRORS = (REPL, REFL, R101)
BORDERS = (CONST, REPL, REFL, R101)
BUCKETS = (3, 5, 7, 9, 11, 13, 15, 17, 21, 25, 27, 31)
CV_8U, CV_16S, CV_32F = 0, 3, 5


# ---------------------------------------------------------------------------------------------------------------- dispatch restated
def _sym(k):
    k = np.asarray(k, np.float32)
    return 1 if np.array_equal(k, k[::-1]) else 2 if np.array_equal(k, -k[::-1]) else 0


def _bucket(n):
    return next((b for b in BUCKETS if n <= b), 0)


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _exact_mode(kx, ky, ax, ay, ddepth):
    """8-bit source: the 8.8 fixed-point (8U) or integer (16S) mode of sep_filter_impl instead of float arithmetic"""
    def ktype(k, a):
        k = np.asarray(k, np.float32).astype(np.float64)
        t = {"symm": a * 2 + 1 == len(k) and _sym(k) == 1, "asym": a * 2 + 1 == len(k) and _sym(k) == 2,
             "smooth": bool(np.all(k >= 0)) and abs(k.sum() - 1) <= 1.1920928955078125e-07 * (abs(k.sum()) + 1), "int": bool(np.all(k == np.rint(k)))}
        return t
    rx, ry = ktype(kx, ax), ktype(ky, ay)
    ex = lambda k, bits: bool(np.all(np.abs(np.asarray(k, np.float64) * (1 << bits) - np.rint(np.asarray(k, np.float64) * (1 << bits)))
                                     <= 10 * 1.1920928955078125e-07 * (1 << bits)))
    if ddepth in (-1, None, CV_8U):      # kernel type exactly SMOOTH | SYMM in both directions (an integer kernel is not), 8.8-exact taps
        plain = lambda t: t["smooth"] and t["symm"] and not t["asym"] and not t["int"]
        return plain(rx) and plain(ry) and ex(kx, 8) and ex(ky, 8)
    if ddepth == CV_16S:
        return (rx["symm"] or rx["asym"]) and (ry["symm"] or ry["asym"]) and rx["int"] and ry["int"]
    return False


def predict(src, ddepth, kx, ky, anchor=(-1, -1), border=R101, dog_tile=False, has_dog=False):
    """(kernel name, nch) the library launches for sepFilter2D(src, ddepth, kx, ky, anchor) on the float path.  src: the device tensor."""
    m = C.describe(src)
    cn = ((m.type >> 3) & 511) + 1
    s8 = src.dtype.is_floating_point is False
    nx, ny = len(kx), len(ky)
    ax = nx // 2 if anchor[0] < 0 else anchor[0]
    ay = ny // 2 if anchor[1] < 0 else anchor[1]
    centred = ax == nx // 2 and ay == ny // 2
    assert not (s8 and _exact_mode(kx, ky, ax, ay, ddepth)), "8-bit exact taps: not the float path"
    tma = ((m.data | m.step | m.frame_step) & 15) == 0
    frames = max(m.frames, 1)
    if cn == 1 and centred and (ddepth in (-1, None) or (not s8 and ddepth == CV_32F) or (s8 and ddepth == CV_8U)):
        csym = _sym(ky)
        rsym = _sym(kx) if (not s8 and 3 <= nx <= 5) else 0
        KB = _bucket(max(nx, ny))
        if (nx & 1) and (ny & 1) and max(nx, ny) <= 31 and csym and not (rsym and max(nx, ny) > 5) and border != WRAP and tma \
                and m.cols >= KB and m.rows >= KB:
            if KB <= 11:
                return "sep_f32_tile_kernel", 1
            tiles = -(-m.cols // 192) * -(-m.rows // 32) * frames
            nch = 4 if tiles >= 16 * _num_sms() else 2 if tiles >= 8 * _num_sms() else 1
            if has_dog and dog_tile:
                nch = 1
            return "sep_f32_tma_kernel", nch
    col_mode = _sym(ky) if (ny & 1) and ay == ny // 2 else 0
    row_small = _sym(kx) if (not s8 and nx in (3, 5) and ax == nx // 2) else 0
    fast_ok = col_mode != 0 and (not row_small or (nx <= 5 and ny <= 5))
    KB = _bucket(max(nx, ny)) if (nx & 1) and (ny & 1) and centred else 0
    if cn == 1 and KB and fast_ok:
        return "sep_fast_kernel", 1
    return "sep_generic_kernel", 1


def walking_frames(W, H, nch):
    """frames that make launch_sf32 walk nch chunks on W x H frames"""
    per = -(-W // 192) * -(-H // 32)
    lo = {2: 8, 4: 16}[nch] * _num_sms()
    f = -(-lo // per)
    assert nch == 4 or f * per < 16 * _num_sms(), "no frame count gives nch = 2 at %dx%d" % (W, H)
    return f


# ---------------------------------------------------------------------------------------------------------------- data and comparison
def rand_f32(rng, *shape):
    """fractional bits over several magnitudes and both signs: the exponent changes from row to row.
    shape: (H, W), (H, W, cn) or (N, H, W, cn)"""
    ax = 1 if len(shape) == 4 else 0
    e = rng.integers(-6, 9, shape[ax]).astype(np.float64)
    e = e.reshape(tuple(shape[ax] if d == ax else 1 for d in range(len(shape))))
    return ((rng.random(shape) - 0.3) * 2.0 ** e).astype(np.float32)


def rand_taps(rng, n, kind):
    """n float32 taps: "sym", "asym" (antisymmetric) or "rand" (neither), |taps| summing to about 1"""
    if n == 1:
        return np.array([0.75], np.float32)
    k = (rng.random(n) + 0.05).astype(np.float32)
    if kind == "sym":
        k = (k + k[::-1]).astype(np.float32)
    elif kind == "asym":
        k = (k - k[::-1]).astype(np.float32)
    k = (k / np.float32(np.abs(k).sum() or 1)).astype(np.float32)
    if kind == "sym":
        k = ((k + k[::-1]) / np.float32(2)).astype(np.float32)
        assert _sym(k) == 1
    elif kind == "asym":
        k = ((k - k[::-1]) / np.float32(2)).astype(np.float32)
        assert _sym(k) == 2
    return k


def same(got, want, what):
    got = np.asarray(got); want = np.asarray(want)
    assert got.shape == want.shape, "%s: shape %s vs %s" % (what, got.shape, want.shape)
    if got.dtype.kind == "f":
        gn, wn = np.isnan(got), np.isnan(want)
        if not np.array_equal(gn, wn):
            idx = np.argwhere(gn != wn)
            raise AssertionError("%s: NaN masks differ at %d elements, first %s (got %r want %r)" % (what, len(idx), tuple(idx[0]), got[tuple(idx[0])], want[tuple(idx[0])]))
        bad = (got != want) & ~gn
    else:
        bad = got != want
    if bad.any():
        idx = np.argwhere(bad)
        d = np.abs(got.astype(np.float64) - want.astype(np.float64))[bad]
        raise AssertionError("%s: %d/%d elements differ, max |d| = %g, first at %s (got %r want %r)" % (
            what, len(idx), got.size, d.max(), tuple(idx[0]), got[tuple(idx[0])], want[tuple(idx[0])]))


def check_sep(cvb, port, img, ddepth, kx, ky, anchor=(-1, -1), delta=0.0, border=R101, what="", expect=None, dev=None):
    """img: one frame (H, W) / (H, W, cn) or a batch (N, H, W, cn); dev: the device tensor to filter (default: a contiguous copy)"""
    dev = gpu(img) if dev is None else dev
    if expect is not None:
        assert predict(dev, ddepth, kx, ky, anchor, border)[0] == expect, "%s: dispatch predicts %s" % (what, predict(dev, ddepth, kx, ky, anchor, border))
    got = cpu(cvb.sepFilter2D(dev, ddepth, kx, ky, anchor, delta, border))
    if img.ndim == 4:
        for f in range(img.shape[0]):
            fr = img[f] if img.shape[3] > 1 else img[f, :, :, 0]
            same(got[f] if img.shape[3] > 1 else got[f, :, :, 0], port.sepFilter2D(fr, ddepth, kx, ky, anchor, delta, border), "%s frame %d" % (what, f))
    else:
        same(got, port.sepFilter2D(img, ddepth, kx, ky, anchor, delta, border), what)
    return got


def pitched(img, pad_to=16, esz=4):
    """device view of img inside a buffer whose rows are a multiple of 16 bytes apart (TMA-addressable whatever the width)"""
    import torch
    h, w = img.shape[:2]
    per = pad_to // esz
    P = -(-(w + 1) // per) * per
    buf = torch.zeros((h, P), dtype=torch.float32 if esz == 4 else torch.uint8, device="cuda")
    v = buf[:, :w]
    v.copy_(gpu(img))
    return v


# ---------------------------------------------------------------------------------------------------------------- widths and tiles
TILE_WIDTHS = list(range(185, 194)) + [223, 224, 225, 383, 384, 385, 575, 577, 608]


@pytest.mark.parametrize("k", [3, 5, 7, 9, 11, 13, 19, 21, 31])
def test_f32_widths_every_residue(cvb, port, rng, k):
    """Widths covering every W mod 8 around the 192-column tile and the 224-column staging edge, contiguous (TMA only when W % 4 == 0,
    else sep_fast_kernel) and as a 16-byte-pitched view (always the TMA kernels): the right-edge apron patch of sep_f32.cu at every
    offset, all borders."""
    kx = rand_taps(rng, k, "rand") if k > 5 else rand_taps(rng, k, "sym")
    ky = rand_taps(rng, k, "sym")
    for W in TILE_WIDTHS:
        img = rand_f32(rng, 37, W)
        for b in BORDERS:
            want = port.sepFilter2D(img, -1, kx, ky, (-1, -1), 0.0, b)
            d = gpu(img)
            kern = predict(d, -1, kx, ky, border=b)[0]
            assert kern == ("sep_f32_tile_kernel" if k <= 11 else "sep_f32_tma_kernel") if W % 4 == 0 else kern == "sep_fast_kernel"
            same(cpu(cvb.sepFilter2D(d, -1, kx, ky, borderType=b)), want, "f32 k=%d W=%d b=%d contiguous" % (k, W, b))
            v = pitched(img)
            assert predict(v, -1, kx, ky, border=b)[0] in ("sep_f32_tile_kernel", "sep_f32_tma_kernel")
            same(cpu(cvb.sepFilter2D(v, -1, kx, ky, borderType=b)), want, "f32 k=%d W=%d b=%d pitched" % (k, W, b))


@pytest.mark.parametrize("k", [3, 7, 11, 13, 17, 31])
def test_u8_float_taps_widths_every_residue(cvb, port, rng, k):
    """8-bit source, float taps (not 8-bit exact): every W mod 32, 192..225 and 383..385, contiguous (TMA when W % 16 == 0) and pitched;
    8U -> 8U through the TMA kernels or sep_fast_kernel, 8U -> 32F through sep_fast_kernel"""
    kx = rand_taps(rng, k, "rand") * np.float32(1.37)
    ky = rand_taps(rng, k, "sym") * np.float32(0.91)
    for W in list(range(192, 226)) + [383, 384, 385]:
        img = rng.integers(0, 256, (33, W), dtype=np.uint8)
        for b in BORDERS:
            want8 = port.sepFilter2D(img, -1, kx, ky, (-1, -1), 0.5, b)
            same(cpu(cvb.sepFilter2D(gpu(img), -1, kx, ky, delta=0.5, borderType=b)), want8, "u8 k=%d W=%d b=%d" % (k, W, b))
            v = pitched(img, 16, 1)
            assert predict(v, -1, kx, ky, border=b)[0] in ("sep_f32_tile_kernel", "sep_f32_tma_kernel")
            same(cpu(cvb.sepFilter2D(v, -1, kx, ky, delta=0.5, borderType=b)), want8, "u8 k=%d W=%d b=%d pitched" % (k, W, b))
            if W % 8 == 1 or W in (224, 384):
                check_sep(cvb, port, img, CV_32F, kx, ky, delta=0.5, border=b, what="u8->f32 k=%d W=%d b=%d" % (k, W, b), expect="sep_fast_kernel")


@pytest.mark.parametrize("k", list(range(3, 32, 2)) + [33])
def test_every_size_small_images(cvb, port, rng, k):
    """Every odd size 3..31 (19, 23 and 29 padded inside a bucket) and 33 (generic): widths and heights KB-1, KB, KB+1, images narrower
    than the radius (the kernels bounce off both edges), heights 1..9, 16, 17 (the TH = 8 / 16 tiles of launch_fast)"""
    kx = rand_taps(rng, k, "rand")
    ky = rand_taps(rng, k, "sym")
    KB = _bucket(k) or k
    shapes = [(KB - 1, KB + 3), (KB, KB), (KB + 1, KB + 1), (KB + 3, KB - 1), (KB + 2, 2), (3, KB + 5)] + [(h, 45) for h in (1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 17)]
    for (h, w) in shapes:
        img = rand_f32(rng, h, w)
        for b in BORDERS:
            check_sep(cvb, port, img, -1, kx, ky, border=b, what="f32 k=%d %dx%d b=%d" % (k, h, w, b))
            v = pitched(img)
            same(cpu(cvb.sepFilter2D(v, -1, kx, ky, borderType=b)), port.sepFilter2D(img, -1, kx, ky, (-1, -1), 0.0, b), "f32 pitched k=%d %dx%d b=%d" % (k, h, w, b))
        u = rng.integers(0, 256, (h, w), dtype=np.uint8)
        check_sep(cvb, port, u, -1, kx, ky, delta=0.25, border=R101, what="u8 k=%d %dx%d" % (k, h, w))


# ---------------------------------------------------------------------------------------------------------------- taps
@pytest.mark.parametrize("nx,ny", [(3, 3), (5, 5), (3, 5), (5, 3), (3, 7), (7, 3), (5, 11), (11, 5), (9, 19), (19, 9), (13, 29), (29, 13),
                                   (23, 23), (1, 7), (7, 1), (15, 31), (31, 15)])
@pytest.mark.parametrize("rk,ck", [("sym", "sym"), ("asym", "sym"), ("sym", "asym"), ("asym", "asym"), ("rand", "sym"), ("rand", "rand")])
def test_tap_symmetries(cvb, port, rng, nx, ny, rk, ck):
    """Symmetric, antisymmetric and asymmetric rows and columns, the 3/5-tap centre-out rows, nx != ny both ways, non-zero delta, on the
    tile / walking kernels (aligned rows), sep_fast_kernel (W*4 % 16 != 0) and the generic kernel (asymmetric columns, 2 channels)"""
    kx = rand_taps(rng, nx, rk)
    ky = rand_taps(rng, ny, ck)
    for (h, w) in ((70, 388), (53, 201)):
        img = rand_f32(rng, h, w)
        for b in (REPL, R101, CONST):
            check_sep(cvb, port, img, -1, kx, ky, delta=0.375, border=b, what="%dx%d %s/%s %dx%d b=%d" % (nx, ny, rk, ck, h, w, b))
    img2 = rand_f32(rng, 29, 67, 2)
    check_sep(cvb, port, img2, -1, kx, ky, delta=-1.25, border=REFL, what="2 channels %dx%d %s/%s" % (nx, ny, rk, ck), expect="sep_generic_kernel")


@pytest.mark.parametrize("nx,ny,anchor", [(4, 4, (-1, -1)), (6, 3, (1, -1)), (3, 6, (-1, 4)), (5, 5, (0, 4)), (7, 7, (6, 0)), (2, 9, (0, 2)),
                                          (33, 33, (-1, -1)), (33, 5, (3, 1)), (8, 8, (7, 7))])
def test_even_sizes_anchors_wrap(cvb, port, rng, nx, ny, anchor):
    """Even sizes, off-centre anchors, 33 taps and BORDER_WRAP: the generic kernel, 1 to 3 channels, f32 and 8-bit sources"""
    kx = rand_taps(rng, nx, "rand")
    ky = rand_taps(rng, ny, "sym" if ny & 1 else "rand")
    for cn in (1, 3):
        shape = (41, 97) if cn == 1 else (41, 97, cn)
        img = rand_f32(rng, *shape)
        u = rng.integers(0, 256, shape, dtype=np.uint8)
        for b in BORDERS + (WRAP,):
            check_sep(cvb, port, img, -1, kx, ky, anchor, 0.5, b, "f32 %dx%d a=%s cn=%d b=%d" % (nx, ny, anchor, cn, b), expect="sep_generic_kernel")
            check_sep(cvb, port, u, CV_32F, kx, ky, anchor, 0.5, b, "u8->f32 %dx%d a=%s cn=%d b=%d" % (nx, ny, anchor, cn, b))
            check_sep(cvb, port, u, -1, kx, ky, anchor, 0.5, b, "u8 %dx%d a=%s cn=%d b=%d" % (nx, ny, anchor, cn, b))


@pytest.mark.parametrize("k", [7, 13])
def test_wrap_on_centred_kernels(cvb, port, rng, k):
    """BORDER_WRAP with centred odd kernels: never the TMA kernels, sep_fast_kernel instead; images narrower than
    the kernel wrap more than once"""
    kx, ky = rand_taps(rng, k, "rand"), rand_taps(rng, k, "sym")
    for (h, w) in ((64, 256), (5, 3), (33, 130)):
        img = rand_f32(rng, h, w)
        check_sep(cvb, port, img, -1, kx, ky, border=WRAP, what="wrap k=%d %dx%d" % (k, h, w), expect="sep_fast_kernel")
        u = rng.integers(0, 256, (h, w), dtype=np.uint8)
        check_sep(cvb, port, u, -1, kx, ky, delta=0.5, border=WRAP, what="wrap u8 k=%d %dx%d" % (k, h, w))


def test_gaussian_blur_entry(cvb, port, rng):
    """GaussianBlur on float images through its own entry: automatic ksize (sigma 2.25, 2.75, 3.5 give 19, 23, 29 taps, padded inside a
    bucket), sigmaX != sigmaY, explicit rectangular sizes"""
    cases = [((0, 0), 2.25, 0), ((0, 0), 2.75, 0), ((0, 0), 3.5, 0), ((0, 0), 1.2, 2.9), ((0, 0), 3.1, 0.8), ((7, 3), 1.1, 0.6), ((3, 9), 0, 0),
             ((5, 5), 1.3, 1.3), ((0, 0), 1.6, 0), ((11, 0), 1.7, 4.0), ((31, 31), 0, 0), ((1, 9), 0, 2.0)]
    for (h, w) in ((90, 384), (77, 253), (2160 // 8, 3840 // 8)):
        img = rand_f32(rng, h, w)
        for ks, sx, sy in cases:
            for b in BORDERS:
                same(cpu(cvb.GaussianBlur(gpu(img), ks, sx, sy, b)), port.GaussianBlur(img, ks, sx, sy, b), "GaussianBlur %s %g/%g %dx%d b=%d" % (ks, sx, sy, h, w, b))


# ---------------------------------------------------------------------------------------------------------------- depths and entries
def test_u8_half_to_even(cvb, port, rng):
    """8-bit destinations from float taps: results constructed to land exactly on .5 round half to even (saturate_cast), every kernel"""
    kx = np.array([0.5, 0.5, 0.5], np.float32)          # not smooth: float path; (a + b + c) / 2 is x.5 whenever a + b + c is odd
    ky = np.array([0, 1, 0], np.float32)
    kx7 = np.array([0.5, 0, 0, 0.5, 0, 0, 0.5], np.float32)
    ky13 = np.zeros(13, np.float32); ky13[6] = 1
    for W in (64, 96, 1000, 67):
        img = rng.integers(0, 256, (40, W), dtype=np.uint8)
        for kxx, kyy in ((kx, ky), (kx7, ky13), (kx, ky13)):
            got = check_sep(cvb, port, img, -1, kxx, kyy, what="ties W=%d %d/%d" % (W, len(kxx), len(kyy)))
            r = port.sepFilter2D(img, CV_32F, kxx, kyy)
            ties = (r == np.floor(r) + 0.5) & (r < 255)
            assert ties.mean() > 0.2
            assert np.all(got[ties] % 2 == 0), "ties not rounded to even"
        check_sep(cvb, port, img[..., None][None].repeat(2, 0), -1, kx, ky, what="ties batch")


@pytest.mark.parametrize("ksize", [1, 3, 5, 7, -1])
def test_sobel_scharr_float(cvb, port, rng, ksize):
    """Sobel / Scharr with a non-integer scale and a delta: 8U -> 16S and 8U -> 32F through float, f32 -> f32"""
    u = rng.integers(0, 256, (67, 230), dtype=np.uint8)
    f = rand_f32(rng, 67, 232)
    for dx, dy in ((1, 0), (0, 1)) + (((2, 0), (1, 1), (0, 2)) if ksize > 1 else ()):
        for b in BORDERS:
            for src, dd in ((u, CV_16S), (u, CV_32F), (f, CV_32F), (f, -1)):
                want = port.Sobel(src, dd, dx, dy, ksize, 0.37, 3.25, b)
                got = cpu(cvb.Sobel(gpu(src), dd, dx, dy, ksize, 0.37, 3.25, b))
                same(got, want, "Sobel k=%d d=(%d,%d) %s->%d b=%d" % (ksize, dx, dy, src.dtype, dd, b))


# ---------------------------------------------------------------------------------------------------------------- layouts
@pytest.mark.parametrize("k", [5, 9, 15, 27])
def test_layouts(cvb, port, rng, k):
    """Contiguous rows with W*4 % 16 != 0, views of wider 16-byte-pitched buffers, a base pointer 4 bytes off, batches of frames, and
    destination views inside NaN / 0xA5-filled buffers whose guard rows and columns must come back untouched"""
    import torch
    kx, ky = rand_taps(rng, k, "rand"), rand_taps(rng, k, "sym")
    H, W = 75, 301
    img = rand_f32(rng, H, W)
    for b in BORDERS:
        want = port.sepFilter2D(img, -1, kx, ky, (-1, -1), 0.0, b)
        same(cpu(cvb.sepFilter2D(gpu(img), -1, kx, ky, borderType=b)), want, "contiguous W=301")
        big = gpu(rand_f32(rng, H + 6, 320))
        v = big[3:3 + H, 8:8 + W]                                   # 16-byte pitch and base
        v.copy_(gpu(img))
        assert predict(v, -1, kx, ky, border=b)[0] != "sep_fast_kernel"
        same(cpu(cvb.sepFilter2D(v, -1, kx, ky, borderType=b)), want, "pitched view")
        flat = torch.zeros(H * 320 + 8, dtype=torch.float32, device="cuda")
        o = flat[1:1 + H * 320].view(H, 320)[:, :W]                 # base 4 bytes off a 16-byte boundary
        o.copy_(gpu(img))
        assert predict(o, -1, kx, ky, border=b)[0] == "sep_fast_kernel"
        same(cpu(cvb.sepFilter2D(o, -1, kx, ky, borderType=b)), want, "base +4 bytes")
        dbuf = torch.full((H + 4, W + 9), float("nan"), dtype=torch.float32, device="cuda")
        dv = dbuf[2:2 + H, 5:5 + W]
        cvb.sepFilter2D(gpu(img), -1, kx, ky, borderType=b, dst=dv)
        out = cpu(dbuf)
        same(out[2:2 + H, 5:5 + W], want, "dst view")
        guard = np.ones(out.shape, bool); guard[2:2 + H, 5:5 + W] = False
        assert np.isnan(out[guard]).all(), "dst guard touched"
        u = rng.integers(0, 256, (H, W), dtype=np.uint8)
        ub = torch.full((H + 4, W + 40), 0xA5, dtype=torch.uint8, device="cuda")
        uv = ub[1:1 + H, 16:16 + W]
        cvb.sepFilter2D(gpu(u), -1, kx, ky, delta=0.5, borderType=b, dst=uv)
        uo = cpu(ub)
        same(uo[1:1 + H, 16:16 + W], port.sepFilter2D(u, -1, kx, ky, (-1, -1), 0.5, b), "u8 dst view")
        g = np.ones(uo.shape, bool); g[1:1 + H, 16:16 + W] = False
        assert (uo[g] == 0xA5).all(), "u8 dst guard touched"
    batch = rand_f32(rng, 3, 50, 196, 1)
    check_sep(cvb, port, batch, -1, kx, ky, border=REFL, what="batch aligned")
    batch = rand_f32(rng, 3, 50, 197, 1)
    check_sep(cvb, port, batch, -1, kx, ky, border=REFL, what="batch unaligned", expect="sep_fast_kernel")


# ---------------------------------------------------------------------------------------------------------------- walking kernel
@pytest.mark.parametrize("src_kind", ["f32", "u8"])
@pytest.mark.parametrize("nch", [2, 4])
@pytest.mark.parametrize("k", [13, 15, 17, 21, 25, 27, 31])
def test_walking_kernel(cvb, port, rng, k, nch, src_kind):
    """sep_f32_tma_kernel walking nch = 2 and 4 chunks: heights with H mod 128 in {1, 31, 33, 127} (a partial last chunk, a strip that ends
    inside a chunk), every mirroring border at the bottom of a walked strip and BORDER_CONSTANT, float and 8-bit sources.  Narrow frames in
    a batch make the grid deep enough to walk while the port still checks every element of every frame."""
    i = BUCKETS.index(k)
    H = 128 * (2 + i % 3) + (1, 31, 33, 127)[(i + nch) % 4]
    W = 36 if src_kind == "f32" else 48
    kx = rand_taps(rng, k, "rand")
    ky = rand_taps(rng, k, "sym" if (i + nch) % 2 else "asym")
    f = walking_frames(W, H, nch)
    if src_kind == "f32":
        img = rand_f32(rng, f, H, W, 1)
    else:
        img = rng.integers(0, 256, (f, H, W, 1), dtype=np.uint8)
    d = gpu(img)
    assert predict(d, -1, kx, ky) == ("sep_f32_tma_kernel", nch)
    for b in BORDERS:
        check_sep(cvb, port, img, -1, kx, ky, delta=0.125, border=b, what="walk k=%d nch=%d %s %dx%dx%d b=%d" % (k, nch, src_kind, f, H, W, b), dev=d)


def _band_check(cvb, port, img, got, kx, ky, b, rows, what):
    """compare rows [a, z) of one frame: the port filters the source band that feeds them (the image's own border where a band touches it)"""
    H = img.shape[0]
    r = len(ky) // 2
    for a, z in rows:
        a, z = max(a, 0), min(z, H)
        s0, s1 = (0 if a - r <= 0 else a - r), (H if z + r >= H else z + r)
        want = port.sepFilter2D(img[s0:s1], -1, kx, ky, (-1, -1), 0.0, b)
        same(got[a:z], want[a - s0:z - s0], "%s rows %d..%d" % (what, a, z))


@pytest.mark.parametrize("k", [13, 27])
def test_walking_kernel_4k_bands(cvb, port, rng, k):
    """4K frames walking 4 chunks: rows around every strip boundary (128 rows), around the chunk boundaries of the first and last strips,
    and the first and last 40 rows, all columns, every mirroring border"""
    H, W = 2160, 3840
    f = walking_frames(W, H, 4)
    img = rand_f32(rng, f, H, W, 1)
    kx, ky = rand_taps(rng, k, "rand"), rand_taps(rng, k, "sym")
    d = gpu(img)
    assert predict(d, -1, kx, ky) == ("sep_f32_tma_kernel", 4)
    r = k // 2
    rows = [(0, 40), (H - 40, H)] + [(y - r - 2, y + r + 2) for y in range(128, H, 128)] + [(y - 3, y + 3) for y in (32, 64, 96, H - H % 128 + 32)]
    for b in MIRRORS:
        got = cpu(cvb.sepFilter2D(d, -1, kx, ky, borderType=b))
        for fr in (0, f - 1):
            _band_check(cvb, port, img[fr, :, :, 0], got[fr, :, :, 0], kx, ky, b, rows, "4K k=%d b=%d frame %d" % (k, b, fr))


# ---------------------------------------------------------------------------------------------------------------- SIFT / fused DoG
def _sift_sigmas(n_layers=3, sigma=1.6):
    k = 2.0 ** (1.0 / n_layers)
    sig = [sigma]
    for i in range(1, n_layers + 3):
        sp = k ** (i - 1) * sigma
        st = sp * k
        sig.append(math.sqrt(st * st - sp * sp))
    return sig


@pytest.mark.parametrize("shape", [(135, 241), (211, 77), (100, 196), (540, 964), (360, 480)])
def test_sift_levels_are_port_blurs(cvb, port, rng, shape):
    """Every Gaussian level i >= 1 of every octave is port.GaussianBlur(<device level i-1>, sigma_i, REFLECT_101) bit for bit: odd
    octave widths and w*4 % 16 != 0 (sep_fast_kernel with the fused DoG), aligned widths (tile and walking kernels), the small-octave
    kernel; each DoG level is the difference of its two Gaussian levels; the whole pyramid equals the port's sift_pyramid"""
    from oracle.api import unpack_pyramid
    img = rng.integers(0, 256, shape, dtype=np.uint8)
    G, D, dims = cvb.sift_pyramid(gpu(img), 3, 1.6, True)
    gg, gd = unpack_pyramid(cpu(G)[0], cpu(D)[0], dims.reshape(-1), len(dims), 3)
    sig = _sift_sigmas()
    for o in range(len(dims)):
        for i in range(1, 6):
            same(gg[o][i], port.GaussianBlur(gg[o][i - 1], (0, 0), sig[i], sig[i], R101), "%s octave %d level %d" % (shape, o, i))
        for i in range(5):
            same(gd[o][i], gg[o][i + 1] - gg[o][i], "%s dog o=%d i=%d" % (shape, o, i))
    wg, wd = port.sift_pyramid(img, 3, 1.6, True)
    assert len(wg) == len(dims)
    for o in range(len(dims)):
        for i in range(6):
            same(gg[o][i], wg[o][i], "%s pyramid vs port gauss o=%d i=%d" % (shape, o, i))
        for i in range(5):
            same(gd[o][i], wd[o][i], "%s pyramid vs port dog o=%d i=%d" % (shape, o, i))


def test_sift_4k_dog_tile_switch(cvb, port, rng, monkeypatch):
    """4K: the pyramid with the fused-DoG blurs forced onto the plain tile kernel (B200CV_SEP_DOG_TILE) equals the walking one, and the
    first octave's levels are port blurs of their predecessors on row bands"""
    from oracle.api import unpack_pyramid
    img = rng.integers(0, 256, (2160, 3840), dtype=np.uint8)
    G, D, dims = cvb.sift_pyramid(gpu(img), 3, 1.6, True)
    monkeypatch.setenv("B200CV_SEP_DOG_TILE", "1")
    G1, D1, _ = cvb.sift_pyramid(gpu(img), 3, 1.6, True)
    monkeypatch.delenv("B200CV_SEP_DOG_TILE")
    Gh, Dh, G1h, D1h = cpu(G), cpu(D), cpu(G1), cpu(D1)
    same(G1h, Gh, "gauss tile vs walk")
    same(D1h, Dh, "dog tile vs walk")
    del G, D, G1, D1, G1h, D1h
    gg, _ = unpack_pyramid(Gh[0], Dh[0], dims.reshape(-1), len(dims), 3)
    sig = _sift_sigmas()
    H = gg[0][0].shape[0]
    for i in (1, 5):
        ks = int(round(sig[i] * 4 * 2 + 1)) | 1
        from opencv_b200 import getGaussianKernel
        t = getGaussianKernel(ks, sig[i]).astype(np.float32).reshape(-1)
        r = ks // 2
        rows = [(0, 40), (H - 40, H)] + [(y - r - 1, y + r + 1) for y in range(128, H, 512)]
        _band_check(cvb, port, gg[0][i - 1], gg[0][i], t, t, R101, rows, "4K level %d" % i)


# ---------------------------------------------------------------------------------------------------------------- non-finite pixels
def _with_specials(rng, h, w, cn=1):
    img = rand_f32(rng, h, w) if cn == 1 else rand_f32(rng, h, w, cn)
    flat = img.reshape(-1)
    n = flat.size
    pos = rng.choice(n, 9, replace=False)
    flat[pos[:3]] = np.inf
    flat[pos[3:6]] = -np.inf
    flat[pos[6:]] = np.nan
    return img


@pytest.mark.parametrize("kinds", ["sym", "anti"])
@pytest.mark.parametrize("nx,ny", [(7, 7), (13, 13), (19, 19), (23, 23), (29, 29), (3, 7), (7, 3), (5, 3), (3, 5), (9, 27), (31, 17), (11, 11),
                                   (3, 3), (5, 5)])
def test_non_finite_pixels(cvb, port, oracle, rng, nx, ny, kinds):
    """Isolated +inf, -inf and NaN pixels under bucket and non-bucket sizes, on every kernel: the NaN mask and every other value equal
    the port's (and, where it is built, the reference's: same NaN and infinity positions, finite values within its remainder bar).
    The zero taps the reference never evaluates must not turn an infinity into NaN: those that pad a kernel to its bucket, and the zero
    centre of antisymmetric columns and of antisymmetric 3/5-tap rows ("anti": both directions antisymmetric)."""
    if kinds == "anti":
        kx, ky = rand_taps(rng, nx, "asym"), rand_taps(rng, ny, "asym")
    else:
        kx = rand_taps(rng, nx, "sym" if nx <= 5 else "rand")
        ky = rand_taps(rng, ny, "sym")
    for (h, w, cn, layout) in ((70, 388, 1, "aligned"), (61, 201, 1, "fast"), (40, 96, 2, "generic")):
        img = _with_specials(rng, h, w, cn)
        for b in (R101, CONST, REPL):
            got = check_sep(cvb, port, img, -1, kx, ky, border=b, what="non-finite %dx%d %s b=%d" % (nx, ny, layout, b))
            want = oracle.sepFilter2D(img, -1, kx, ky, (-1, -1), 0.0, b)
            assert np.array_equal(np.isnan(got), np.isnan(want)), "NaN mask vs %s" % oracle.kind
            assert np.array_equal(np.isinf(got), np.isinf(want)) and np.array_equal(got[np.isinf(got)], want[np.isinf(want)])
            fin = np.isfinite(want)
            assert np.allclose(got[fin], want[fin], rtol=1e-5, atol=1e-4)
    g = _with_specials(rng, 64, 256)
    for sx, sy in ((2.25, 2.25), (1.0, 3.5), (2.75, 0.9)):
        same(cpu(cvb.GaussianBlur(gpu(g), (0, 0), sx, sy, R101)), port.GaussianBlur(g, (0, 0), sx, sy, R101), "GaussianBlur non-finite %g/%g" % (sx, sy))


@pytest.mark.parametrize("ksize", [1, 3, 5, 7, -1])
def test_non_finite_derivatives(cvb, port, rng, ksize):
    """Sobel and Scharr on float images with inf / NaN pixels: first derivatives have an antisymmetric kernel with a zero centre in
    one direction, which the reference never multiplies"""
    for (h, w) in ((70, 388), (61, 201)):
        img = _with_specials(rng, h, w)
        for dx, dy in ((1, 0), (0, 1)) + (((2, 0), (1, 1)) if ksize > 1 else ()):
            for b in (R101, CONST):
                same(cpu(cvb.Sobel(gpu(img), -1, dx, dy, ksize, 0.37, 1.5, b)), port.Sobel(img, -1, dx, dy, ksize, 0.37, 1.5, b),
                     "Sobel non-finite k=%d d=(%d,%d) %dx%d b=%d" % (ksize, dx, dy, h, w, b))


# ---------------------------------------------------------------------------------------------------------------- dispatch check
def test_predicted_kernel_runs(cvb, rng, tmp_path):
    """predict() against the kernels that actually run (torch.profiler, CUDA activities): tests that mean the tile kernel reach it, and
    the walking kernel's grid has ceil(H / (32 nch)) rows of CTAs for the predicted chunk count nch"""
    import json
    import torch
    from torch.profiler import ProfilerActivity, profile
    f = gpu(rand_f32(rng, 64, 256))
    fu = gpu(rand_f32(rng, 64, 257))
    u = gpu(rng.integers(0, 256, (64, 256), dtype=np.uint8))
    walk = gpu(rand_f32(rng, walking_frames(36, 1025, 4), 1025, 36, 1))
    walk2 = gpu(rand_f32(rng, walking_frames(36, 1025, 2), 1025, 36, 1))
    s7, r7, s19, s13 = rand_taps(rng, 7, "sym"), rand_taps(rng, 7, "rand"), rand_taps(rng, 19, "sym"), rand_taps(rng, 13, "sym")
    cases = [(f, -1, r7, s7, (-1, -1)), (f, -1, s19, s19, (-1, -1)), (f, -1, s13, s13, (-1, -1)), (fu, -1, r7, s7, (-1, -1)),
             (f, -1, r7, r7, (-1, -1)), (f, -1, r7, s7, (2, 3)), (u, -1, r7, s7, (-1, -1)), (u, CV_32F, r7, s7, (-1, -1)),
             (u, CV_16S, r7, s7, (-1, -1)), (pitched(cpu(fu)), -1, r7, s7, (-1, -1)), (walk, -1, s13, s13, (-1, -1)),
             (walk2, -1, s19, s19, (-1, -1)), (f, -1, rand_taps(rng, 3, "sym"), rand_taps(rng, 7, "sym"), (-1, -1))]
    seen = set()
    for src, dd, kx, ky, anc in cases:
        want = predict(src, dd, kx, ky, anc)
        seen.add(want)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(2):       # the profiler now and then loses the first kernel record after it starts: the second call is the one looked at
                cvb.sepFilter2D(src, dd, kx, ky, anc)
                torch.cuda.synchronize()
        trace = tmp_path / "trace.json"
        prof.export_chrome_trace(str(trace))
        kern = [e for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") == "kernel"]
        names = [e["name"] for e in kern]
        hits = sorted((e for e in kern if "sep_" in e["name"]), key=lambda e: e["ts"])[-1:]
        assert len(hits) == 1 and len([n for n in names if "sep_" in n]) <= 2 and want[0] in hits[0]["name"], "predicted %s, ran %s" % (want, names)
        m = C.describe(src)
        gy = hits[0]["args"]["grid"][1]
        if want[0] == "sep_f32_tma_kernel":
            assert gy == -(-m.rows // (32 * want[1])), "predicted nch = %d, grid %s for %d rows" % (want[1], hits[0]["args"]["grid"], m.rows)
    assert {k for k, _ in seen} == {"sep_f32_tile_kernel", "sep_f32_tma_kernel", "sep_fast_kernel", "sep_generic_kernel"}
    assert {n for k, n in seen if k == "sep_f32_tma_kernel"} >= {2, 4}
