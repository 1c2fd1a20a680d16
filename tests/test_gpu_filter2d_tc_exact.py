"""GPU: the tensor-core filter2D kernels held to an exact restatement of their arithmetic (tests/f2d_reference.py).

8-bit (filter2d_tc.cu).  The result is fully defined: host-quantised taps Kq = rint(k 2^sh), three balanced digit planes through exact
integer MMAs, S = S0 + 256 S1 + 65536 S2, then fl(fl(float(S) 2^-sh) + delta) and rint saturation.  All three destination depths must
equal the reference bit for bit.

Float (filter2d_tc_f32.cu).  The kernel accumulates T3 = sum (a_hi k_hi + a_hi k_lo + a_lo k_hi) of the BF16 splits in three FP32
accumulators (A_hi x [B_hi | B_lo] as one MMA, A_lo x B_hi as another) and the epilogue adds fl(fl(fl(hh + lh) + hl) + delta).
  - Exact grid.  Integer data with |a| < 2^b and taps m 2^-g with |m| < 2^c, 2^b 2^c kh kw 1.01 <= 2^24: every product and every partial
    sum, in any order, is a multiple of 2^-g below 2^(24-g), so an FP32 accumulator that keeps 24 bits adds them exactly and the
    result must be fl(T3 + delta) bit for bit.  (b, c) = (4, 9) makes k_lo non-zero, (12, 4) makes a_lo non-zero.
  - Random data.  Each BF16 x BF16 product is exact in FP32 (8-bit significands).  Adding n terms in FP32 with a unit roundoff u costs
    at most (n - 1) u sum|terms| (to first order), combining the three accumulators two more u sum|terms|, and the final add of delta
    u' (|T3| + |delta|) with u' = 2^-24 (round to nearest).  Taking u = 2^-23 allows an accumulator that truncates rather than rounds;
    with one u of room for the second-order terms:
        |got - (T3 + delta)| <= (n + 3) 2^-23 sum|terms| + 2^-24 |delta|.
    And T3 itself is within 3 2^-16 sum|a||k| of the true sum: the split leaves |a - a_hi - a_lo| <= 2^-16 |a| (likewise for k) and
    the dropped a_lo k_lo is at most 2^-16 |a||k|.
Every case checks, through the launch counter, which path ran: the tensor-core path is three launches (Toeplitz operand, padded
source, MMA kernel); a call that falls back makes the direct path's launches and equals its result.
"""
import ctypes

import numpy as np
import pytest
import torch

import f2d_reference as fr
from util import assert_exact, cpu

pytestmark = pytest.mark.gpu

DT = {-1: np.uint8, 3: np.int16, 5: np.float32}
TDT = {np.uint8: torch.uint8, np.int16: torch.int16, np.float32: torch.float32}
TC_LAUNCHES = 3
BORDERS = [fr.BORDER_CONSTANT, fr.BORDER_REPLICATE, fr.BORDER_REFLECT, fr.BORDER_REFLECT_101]
FRAMES = [1, 3]
FLT_MAX = float(np.finfo(np.float32).max)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev(img, pad_left=0):
    """(N, H, W) numpy -> (N, H, W, 1) device tensor; pad_left > 0 makes it a column window of a wider buffer (unaligned rows)"""
    t = torch.from_numpy(np.ascontiguousarray(img[..., None])).cuda()
    if pad_left:
        n, h, w = img.shape
        base = torch.full((n, h, w + pad_left + 3, 1), 255 if img.dtype == np.uint8 else 7, dtype=t.dtype, device="cuda")
        base[:, :, pad_left:pad_left + w] = t
        t = base[:, :, pad_left:pad_left + w]
    return t


def _run(cvb, monkeypatch, src, ddepth, ker, anchor=(-1, -1), delta=0.0, border=4, dst=None, env=()):
    """one filter2D call: (result (N, H, W) as numpy, launches it made)"""
    env = dict(env)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        n0 = cvb.launch_count()
        out = cvb.filter2D(src, ddepth, ker, anchor=anchor, delta=delta, borderType=border, dst=dst)
        torch.cuda.synchronize()
        return cpu(out)[..., 0], cvb.launch_count() - n0
    finally:
        for k in env:
            monkeypatch.delenv(k)


def _direct(cvb, monkeypatch, src, ddepth, ker, anchor=(-1, -1), delta=0.0, border=4):
    return _run(cvb, monkeypatch, src, ddepth, ker, anchor, delta, border, env={"B200CV_FILTER2D_PATH": "direct"})


def _bits(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _u8(cvb, monkeypatch, img, ker, ddepth=-1, anchor=(-1, -1), delta=0.0, border=4, env=(), pad_left=0, what=""):
    """the tensor-core path ran and equals the reference bit for bit"""
    got, n = _run(cvb, monkeypatch, _dev(img, pad_left), ddepth, ker, anchor, delta, border, env=env)
    what = "u8 tc %s %dx%d dd=%d border %d anchor %s %s" % (img.shape, ker.shape[0], ker.shape[1], ddepth, border, anchor, what)
    assert n == TC_LAUNCHES, what + ": the tensor-core path did not run (%d launches)" % n
    assert_exact(got, fr.filter2d_u8_ref(img, ker, DT[ddepth], anchor, delta, border, with_true=False).res, what)


def _falls_back(cvb, monkeypatch, img, ker, ddepth=-1, anchor=(-1, -1), delta=0.0, border=4, env=(), what=""):
    """the call takes the direct path: the same launches and bit for bit the same result as with the direct path forced"""
    src = _dev(img)
    got, n = _run(cvb, monkeypatch, src, ddepth, ker, anchor, delta, border, env=env)
    want, nd = _direct(cvb, monkeypatch, src, ddepth, ker, anchor, delta, border)
    assert n == nd and n != TC_LAUNCHES, what + ": %d launches, direct path %d" % (n, nd)
    assert_exact(_bits(got), _bits(want), what + ": fall-back vs direct")


def _rand_kernel(rng, kh, kw, scale=1.0):
    k = rng.random((kh, kw)) - 0.3
    return (k / np.abs(k).sum() * 2 * scale).astype(np.float32)


def _rand_u8(rng, frames, h, w):
    return rng.integers(0, 256, (frames, h, w), dtype=np.uint8)


# ---- 8-bit ----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("frames", FRAMES)
@pytest.mark.parametrize("ddepth", [-1, 3, 5])
def test_u8_tile_width(cvb, rng, monkeypatch, frames, ddepth):
    """kw 17 (the widest 16-column tile), 18 (the narrowest 32-column tile), 33 (the widest kernel); kh 31 (the tallest) at both widths:
    a 2-deep A ring at NT = 32, 4-deep for small kh.  kh 32 falls back to the direct path; kw 34 is on no device path and says so."""
    img = _rand_u8(rng, frames, 200, 150)
    scale = 64.0 if ddepth == 3 else 1.0
    for kh, kw in ((13, 17), (13, 18), (5, 33), (31, 33), (31, 5), (31, 18)):
        _u8(cvb, monkeypatch, img, _rand_kernel(rng, kh, kw, scale), ddepth, (kw // 3, kh - 2), 1.5)
    _falls_back(cvb, monkeypatch, img, _rand_kernel(rng, 32, 13, scale), ddepth, what="kh 32")
    n0 = cvb.launch_count()
    with pytest.raises(cvb.NotImplementedOnDevice):
        _run(cvb, monkeypatch, _dev(img), ddepth, _rand_kernel(rng, 13, 34))
    assert cvb.launch_count() == n0


@pytest.mark.parametrize("frames", FRAMES)
def test_u8_switch_points(cvb, rng, monkeypatch, frames):
    """8U / 16S: 128 taps direct, 130 (13 x 10) on the tensor cores; 32F: 49 direct, 50 (5 x 10) on; and 32F from 50 to 129 taps"""
    img = _rand_u8(rng, frames, 140, 90)
    for ddepth in (-1, 3):
        _falls_back(cvb, monkeypatch, img, _rand_kernel(rng, 16, 8), ddepth, delta=0.5, what="128 taps dd=%d" % ddepth)
        _u8(cvb, monkeypatch, img, _rand_kernel(rng, 13, 10), ddepth, delta=0.5)
    _falls_back(cvb, monkeypatch, img, _rand_kernel(rng, 7, 7), 5, what="49 taps 32F")
    for kh, kw in ((5, 10), (7, 9), (9, 11), (8, 16), (4, 32), (3, 33)):
        _u8(cvb, monkeypatch, img, _rand_kernel(rng, kh, kw), 5, delta=-0.25)


@pytest.mark.parametrize("frames", FRAMES)
@pytest.mark.parametrize("kw", [15, 19])          # 16- and 32-column tiles
def test_u8_tile_schedule(cvb, rng, monkeypatch, frames, kw):
    """tile counts below, equal to and oddly above the SM count (some warpgroups get no tile), heights 128 k +- 1 and < 128, widths
    NT k +- 1 and < NT"""
    nt, sms = (16 if kw <= 17 else 32), _sms()
    ker = _rand_kernel(rng, 13, kw)
    for h, w in ((128, nt * (sms - 1)), (128, nt * sms), (257, nt * (sms // 3 + 2) - 1), (127, nt + 1), (129, 2 * nt - 1), (255, nt - 5),
                 (100, 3 * nt), (385, 5)):
        _u8(cvb, monkeypatch, _rand_u8(rng, frames, h, w), ker, -1, (-1, -1), 0.0, 4)


@pytest.mark.parametrize("frames", FRAMES)
@pytest.mark.parametrize("ddepth", [-1, 3, 5])
def test_u8_unaligned(cvb, rng, monkeypatch, frames, ddepth):
    """source rows that are not 4-byte aligned (the byte path of pad_u8_kernel; the buffer around the view is 255, so reading it
    changes the answer), and a destination that is a column window of a wider buffer: element stores, guard columns untouched"""
    h, w = 301, 263
    img = _rand_u8(rng, frames, h, w)
    ker = _rand_kernel(rng, 13, 15, 64.0 if ddepth == 3 else 1.0)
    for off in (1, 2, 3):
        _u8(cvb, monkeypatch, img, ker, ddepth, (0, 12), 0.0, 2, pad_left=off, what="source offset %d" % off)
    base = torch.zeros((frames, h, w + 5, 1), dtype=TDT[DT[ddepth]], device="cuda")
    _, n = _run(cvb, monkeypatch, _dev(img), ddepth, ker, (-1, -1), 0.0, 4, dst=base[:, :, 1:w + 1])
    assert n == TC_LAUNCHES
    rest = cpu(base)[..., 0]
    assert_exact(rest[:, :, 1:w + 1], fr.filter2d_u8_ref(img, ker, DT[ddepth], border=4, with_true=False).res, "unaligned destination")
    assert not rest[:, :, 0].any() and not rest[:, :, w + 1:].any(), "stores outside the destination window"


@pytest.mark.parametrize("frames", FRAMES)
def test_u8_borders_anchors(cvb, rng, monkeypatch, frames):
    """borders 0, 1, 2, 4 with the anchor at each corner of the kernel; images smaller than the kernel"""
    kh, kw = 13, 11
    ker = _rand_kernel(rng, kh, kw)
    img = _rand_u8(rng, frames, 70, 50)
    for border in BORDERS:
        for anchor in ((0, 0), (kw - 1, 0), (0, kh - 1), (kw - 1, kh - 1)):
            _u8(cvb, monkeypatch, img, ker, -1, anchor, 0.0, border)
    for h, w in ((1, 1), (1, 23), (19, 1), (7, 40), (30, 6)):
        for border in BORDERS:
            _u8(cvb, monkeypatch, _rand_u8(rng, frames, h, w), ker, 5, (2, 9), 0.0, border)


@pytest.mark.parametrize("frames", FRAMES)
def test_u8_taps(cvb, rng, monkeypatch, frames):
    """rint ties of both signs and taps that quantise to 0; digits at -128 and 127 on an all-255 image (every |S_d| as large as it gets,
    |S| > 2^24 for 32F); results that saturate both ends of 8U and 16S, with large +-delta"""
    img = _rand_u8(rng, frames, 150, 120)
    t = _rand_kernel(rng, 13, 11, 0.3)
    t[0, 0] = 1.0                                           # sh = 21
    t.flat[1:9] = np.array([3, 5, -3, -5, 7, -7, 1, -1], np.float32) * np.float32(2.0 ** -22)
    t.flat[9:12] = np.float32(2.0 ** -23), np.float32(-2.0 ** -24), np.float32(1e-30)
    for ddepth in (-1, 5):
        _u8(cvb, monkeypatch, img, t, ddepth, what="ties")
    white = np.full((frames, 140, 70), 255, np.uint8)
    for q in (127 + 256 * 127 + 65536 * 63, -128 - 256 * 128 - 65536 * 63):
        for kh, kw in ((31, 31), (13, 17)):
            ker = np.full((kh, kw), q * 2.0 ** -22, np.float32)
            assert fr.quantise(ker)[1] == 22
            for ddepth in (-1, 3, 5):
                _u8(cvb, monkeypatch, white, ker, ddepth, delta=0.0, what="digits of %d" % q)
    ker = (rng.random((13, 11)) - 0.5).astype(np.float32)
    for ddepth, delta, scale in ((-1, 120.0, 1.0), (-1, -300.0, 2.0), (-1, 400.0, 0.5), (3, 30000.0, 300.0), (3, -40000.0, 250.0), (5, 1e6, 3.0)):
        res = fr.filter2d_u8_ref(img, ker * np.float32(scale), DT[ddepth], delta=delta, with_true=False).res
        if ddepth != 5:
            info = np.iinfo(DT[ddepth])
            assert (res == info.min).any() and (res == info.max).any(), "the case does not saturate both ends"
        _u8(cvb, monkeypatch, img, (ker * np.float32(scale)).astype(np.float32), ddepth, delta=delta, what="saturation")


@pytest.mark.parametrize("frames", FRAMES)
def test_u8_kernel_scale(cvb, rng, monkeypatch, frames):
    """max|k| near 1e-29 and 1e29 (sh = 118 and -75) run on the tensor cores; below 1e-30, above 1e30 or with a non-finite tap the call
    falls back to the direct path"""
    img = _rand_u8(rng, frames, 140, 90)
    ker = _rand_kernel(rng, 13, 11)
    ker[0, 0] = 1.0
    for s, sh in ((1e-29, 118), (1e29, -75)):
        k = (ker * np.float32(s)).astype(np.float32)
        assert fr.quantise(k)[1] == sh
        _u8(cvb, monkeypatch, img, k, 5, delta=0.0)
    for s in (1e-31, 1e31):
        _falls_back(cvb, monkeypatch, img, (ker * np.float32(s)).astype(np.float32), 5, what="max|k| = %g" % s)
    for bad in (np.nan, np.inf):
        k = ker.copy()
        k[3, 4] = bad
        _falls_back(cvb, monkeypatch, img, k, 5, what="tap %r" % bad)


@pytest.mark.parametrize("frames", FRAMES)
@pytest.mark.parametrize("kh", [1, 2, 3, 4, 5])
def test_u8_few_kernel_rows(cvb, rng, monkeypatch, frames, kh):
    """the tensor-core path forced below its switch point (B200CV_FILTER2D_TC_MIN_TAPS): almost no MMAs per tile"""
    img = _rand_u8(rng, frames, 300, 263)
    for kw in (7, 19):
        _u8(cvb, monkeypatch, img, _rand_kernel(rng, kh, kw), -1, env={"B200CV_FILTER2D_TC_MIN_TAPS": "1"})
        _u8(cvb, monkeypatch, img, _rand_kernel(rng, kh, kw), 5, (0, kh - 1), 2.0, 1, env={"B200CV_FILTER2D_TC_MIN_TAPS": "1"})


# ---- float ------------------------------------------------------------------------------------------------------------------------

GRID = 8          # taps m 2^-8


def _grid_case(rng, frames, h, w, kh, kw, design):
    """integer data below 2^b, taps m 2^-GRID with |m| < 2^c; a_lo (b = 12) or k_lo (c = 9) is non-zero somewhere"""
    b, c = design
    assert 2 ** b * 2 ** c * kh * kw * 1.01 <= 2 ** 24
    img = rng.integers(-(2 ** b - 1), 2 ** b, (frames, h, w)).astype(np.float32)
    m = rng.integers(-(2 ** c - 1), 2 ** c, (kh, kw))
    m[0, 0] = 2 ** c - 1
    img[:, 0, 0] = 2 ** b - 1
    ker = (m * 2.0 ** -GRID).astype(np.float32)
    if b > 8:
        assert (fr.bf16_split(img)[1] != 0).any()
    if c > 8:
        assert (fr.bf16_split(ker)[1] != 0).any()
    return img, ker


def _designs(kh, kw):
    return [d for d in ((4, 9), (12, 4)) if 2 ** d[0] * 2 ** d[1] * kh * kw * 1.01 <= 2 ** 24]


def _f32(cvb, monkeypatch, img, ker, anchor=(-1, -1), delta=0.375, border=4, env=(), dst=None, what=""):
    """exact grid: the tensor-core path ran and equals fl(T3 + delta) bit for bit"""
    got, n = _run(cvb, monkeypatch, _dev(img), -1, ker, anchor, delta, border, dst=dst, env=env)
    what = "f32 tc %s %dx%d border %d anchor %s %s" % (img.shape, ker.shape[0], ker.shape[1], border, anchor, what)
    assert n == TC_LAUNCHES, what + ": the tensor-core path did not run (%d launches)" % n
    want = fr.filter2d_f32_ref(img, ker, anchor, delta, border, grid=GRID, with_true=False).res
    if dst is None:
        assert_exact(_bits(got), _bits(want), what)
    return want


@pytest.mark.parametrize("frames", FRAMES)
@pytest.mark.parametrize("khw", [(14, 1), (14, 2), (14, 17), (14, 18), (14, 33), (33, 17), (31, 31), (33, 33), (14, 10)])
def test_f32_exact_grid_sizes(cvb, rng, monkeypatch, frames, khw):
    """K / 16 = 2 (kw 1, through the hook), 3 (kw 2, 17) and 4 (kw 18, 33); kh 14 and 33"""
    kh, kw = khw
    env = {"B200CV_FILTER2D_TC_MIN_TAPS": "1"} if kh * kw < 130 else {}
    for design in _designs(kh, kw):
        img, ker = _grid_case(rng, frames, 300, 263, kh, kw, design)
        _f32(cvb, monkeypatch, img, ker, (kw // 2, kh // 3), 0.375, 4, env=env, what=str(design))


@pytest.mark.parametrize("frames", FRAMES)
def test_f32_fallback(cvb, rng, monkeypatch, frames):
    """13 kernel rows stay on the direct path; kh 34 or kw 34 is on no device path and says so"""
    img, ker = _grid_case(rng, frames, 120, 90, 13, 11, (4, 9))
    _falls_back(cvb, monkeypatch, img, ker, -1, what="13 x 11 float")
    for kh, kw in ((34, 14), (14, 34)):
        n0 = cvb.launch_count()
        with pytest.raises(cvb.NotImplementedOnDevice):
            _run(cvb, monkeypatch, _dev(img), -1, _rand_kernel(rng, kh, kw))
        assert cvb.launch_count() == n0


@pytest.mark.parametrize("frames", FRAMES)
@pytest.mark.parametrize("kh", [1, 2, 3, 4])
def test_f32_exact_grid_few_rows(cvb, rng, monkeypatch, frames, kh):
    """kernel rows up to the warpgroup lag (FF_LAG = 3) and one past it, through the hook"""
    for kw in (1, 9, 33):
        img, ker = _grid_case(rng, frames, 300, 100, kh, kw, (12, 4))
        _f32(cvb, monkeypatch, img, ker, env={"B200CV_FILTER2D_TC_MIN_TAPS": "1"})


@pytest.mark.parametrize("frames", FRAMES)
def test_f32_exact_grid_schedule(cvb, rng, monkeypatch, frames):
    """heights 255, 256, 257, 511, 513; widths 32 k +- 1 and < 32; strip counts below, equal to and oddly above the SM count"""
    sms = _sms()
    for (h, w), design in (((255, 65), (4, 9)), ((256, 31), (12, 4)), ((257, 97), (4, 9)), ((511, 63), (12, 4)), ((513, 33), (4, 9)),
                           ((256, 32 * (sms - 1)), (12, 4)), ((256, 32 * sms), (4, 9)), ((513, 32 * (sms // 3 + 2) - 1), (12, 4))):
        kh, kw = (15, 15) if design == (12, 4) else (21, 21)
        img, ker = _grid_case(rng, frames, h, w, kh, kw, design)
        _f32(cvb, monkeypatch, img, ker, what="%s %s" % ((h, w), design))


@pytest.mark.parametrize("frames", FRAMES)
def test_f32_exact_grid_borders(cvb, rng, monkeypatch, frames):
    """borders 0, 1, 2, 4 with the anchor at each corner; images smaller than the kernel; a destination that is a column window of a
    wider buffer (element stores, guard columns untouched)"""
    kh, kw = 14, 17
    img, ker = _grid_case(rng, frames, 90, 70, kh, kw, (12, 4))
    for border in BORDERS:
        for anchor in ((0, 0), (kw - 1, 0), (0, kh - 1), (kw - 1, kh - 1)):
            _f32(cvb, monkeypatch, img, ker, anchor, -2.5, border)
    for h, w in ((1, 1), (1, 23), (19, 1), (7, 40), (30, 6)):
        small, ker = _grid_case(rng, frames, h, w, kh, kw, (4, 9))
        for border in BORDERS:
            _f32(cvb, monkeypatch, small, ker, (3, 10), 0.0, border)
    h, w = 301, 263
    img, ker = _grid_case(rng, frames, h, w, 21, 21, (4, 9))
    base = torch.zeros((frames, h, w + 5, 1), dtype=torch.float32, device="cuda")
    want = _f32(cvb, monkeypatch, img, ker, dst=base[:, :, 1:w + 1])
    rest = cpu(base)[..., 0]
    assert_exact(_bits(rest[:, :, 1:w + 1]), _bits(want), "f32 unaligned destination")
    assert not rest[:, :, 0].any() and not rest[:, :, w + 1:].any(), "stores outside the destination window"


def _check_random(got, ref, n, delta, what):
    """the random-data bars of the module docstring"""
    bar = (n + 3) * 2.0 ** -23 * ref.absum + 2.0 ** -24 * abs(delta)
    d = np.abs(got.astype(np.float64) - (ref.T3 + float(np.float32(delta))))
    assert np.isfinite(got).all(), what + ": %d non-finite results" % int((~np.isfinite(got)).sum())
    bad = d > bar
    assert not bad.any(), what + ": %d elements beyond the bar, first at %s (got %r, T3 %r, bar %g)" % (
        int(bad.sum()), tuple(np.argwhere(bad)[0]), got[bad][0], ref.T3[bad][0], bar[bad][0])
    if ref.true is not None:
        slack = n * 2.0 ** -52 * ref.aksum                  # the f64 sums' own rounding
        assert (np.abs(ref.T3 - ref.true) <= 3 * 2.0 ** -16 * ref.aksum + slack).all(), what + ": T3 vs the true sum"


@pytest.mark.parametrize("frames", FRAMES)
@pytest.mark.parametrize("khw", [(14, 10), (15, 15), (31, 31)])
def test_f32_random(cvb, rng, monkeypatch, frames, khw):
    kh, kw = khw
    img = ((rng.random((frames, 261, 97)) - 0.3) * 300).astype(np.float32)
    ker = (rng.standard_normal((kh, kw)) * 0.05).astype(np.float32)
    for border, delta in ((4, 0.25), (0, -1000.0)):
        got, n = _run(cvb, monkeypatch, _dev(img), -1, ker, (-1, -1), delta, border)
        assert n == TC_LAUNCHES
        _check_random(got, fr.filter2d_f32_ref(img, ker, (-1, -1), delta, border), kh * kw, delta, "f32 random %dx%d border %d" % (kh, kw, border))


@pytest.mark.parametrize("frames", FRAMES)
def test_f32_near_flt_max(cvb, rng, monkeypatch, frames):
    """+-FLT_MAX and +-3.39e38 in a few pixels, taps small enough that no sum overflows: every output finite and within the bar.  A finite
    |a| >= 3.3962e38 must not become a BF16 infinity (which would make the sums NaN, also in windows that do not hold the pixel)."""
    kh, kw = 15, 15
    img = ((rng.random((frames, 200, 150)) - 0.3) * 300).astype(np.float32)
    for (y, x), v in (((20, 30), FLT_MAX), ((21, 90), -FLT_MAX), ((120, 31), 3.39e38), ((150, 140), -3.39e38), ((199, 0), FLT_MAX)):
        img[:, y, x] = v
    ker = _rand_kernel(rng, kh, kw, 0.25)              # sum |k| = 0.5
    for border in (4, 0):
        got, n = _run(cvb, monkeypatch, _dev(img), -1, ker, (-1, -1), 0.5, border)
        assert n == TC_LAUNCHES
        _check_random(got, fr.filter2d_f32_ref(img, ker, (-1, -1), 0.5, border), kh * kw, 0.5, "f32 near FLT_MAX border %d" % border)
    # huge taps against small pixels take the Toeplitz operand's split
    img = ((rng.random((frames, 120, 90)) - 0.5) * 0.5).astype(np.float32)
    ker = _rand_kernel(rng, kh, kw)
    ker[3, 4], ker[7, 7] = FLT_MAX, -3.3962e38
    got, n = _run(cvb, monkeypatch, _dev(img), -1, ker, (-1, -1), 0.0, 4)
    assert n == TC_LAUNCHES
    _check_random(got, fr.filter2d_f32_ref(img, ker, (-1, -1), 0.0, 4), kh * kw, 0.0, "f32 near FLT_MAX taps")


# ---- the HAL seam ------------------------------------------------------------------------------------------------------------------

def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("depth", ["u8", "f32"])
def test_hal_filter_roi(cvb, rng, depth):
    """one b200cv_hal_filter call on a ROI of a larger image (the pixels around the ROI are real, the border applies at the parent's
    edges) at 13 x 15 taps: the reference of the parent, cropped -- bit for bit for 8-bit, within the random-data bar for float"""
    L = cvb.lib()
    sz = ctypes.c_size_t
    kh, kw = 15, 13
    ker = _rand_kernel(rng, kh, kw)
    if depth == "u8":
        par, typ = rng.integers(0, 256, (220, 300), dtype=np.uint8), 0
    else:
        par, typ = ((rng.random((220, 300)) - 0.3) * 300).astype(np.float32), 5
    for (x, y, w, h) in ((0, 0, 150, 140), (37, 21, 200, 170), (100, 3, 200, 217)):
        roi = par[y:y + h, x:x + w]
        out = np.zeros((h, w), par.dtype)
        ctx = ctypes.c_void_p()
        assert L.b200cv_hal_filterInit(ctypes.byref(ctx), _p(ker), sz(ker.strides[0]), 5, kw, kh, 300, 220, typ, typ, 4, ctypes.c_double(1.5),
                                       -1, -1, ctypes.c_bool(True), ctypes.c_bool(False)) == 0
        n0 = cvb.launch_count()
        rc = L.b200cv_hal_filter(ctx, _p(roi), sz(par.strides[0]), _p(out), sz(out.strides[0]), w, h, 300, 220, x, y)
        n = cvb.launch_count() - n0
        assert L.b200cv_hal_filterFree(ctx) == 0
        assert rc == 0 and n >= TC_LAUNCHES, "hal filter rc %d, %d launches" % (rc, n)
        what = "hal filter %s ROI %s" % (depth, (x, y, w, h))
        if depth == "u8":
            assert_exact(out, fr.filter2d_u8_ref(par, ker, np.uint8, delta=1.5, border=4, with_true=False).res[y:y + h, x:x + w], what)
        else:
            ref = fr.filter2d_f32_ref(par, ker, delta=1.5, border=4)
            crop = fr.F32Ref(*(a[y:y + h, x:x + w] for a in ref))
            _check_random(out, crop, kh * kw, 1.5, what)
