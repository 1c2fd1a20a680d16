"""CPU: the numpy restatement of the tensor-core filter2D kernels (tests/f2d_reference.py) against the plain-C port
(oracle/port/port_filter.c: port_filter2d), against exact rational arithmetic and against values computed by hand.  The GPU tests of
tests/test_gpu_filter2d_tc_exact.py hold the device to this reference bit for bit, so it is checked here first, on every machine.

The port is a direct float sum at every kernel size.  With 8-bit data and dyadic taps m 2^-g whose partial sums all stay below 2^24
units of 2^-g, every float operation of that sum is exact, and so is the fixed-point sum of the tensor-core kernel (the quantisation
of such taps loses nothing): the two must then agree bit for bit, roundings of the 8U / 16S destination included.  For float data the
same holds where one of a_lo, k_lo is zero and the other operand has at most 16 significant bits, so that the three BF16 products add
up to the true product."""
from fractions import Fraction

import numpy as np
import pytest

import f2d_reference as fr
from util import assert_exact

BORDERS = [fr.BORDER_CONSTANT, fr.BORDER_REPLICATE, fr.BORDER_REFLECT, fr.BORDER_REFLECT_101]
# (H, W): an ordinary image, 1 x 1, one row, one column, fewer rows than the kernel, fewer columns than the kernel
IMAGES = [(37, 45), (1, 1), (1, 23), (19, 1), (7, 40), (30, 6)]
KSIZES = [(13, 11), (9, 17)]         # 143 and 153 taps: the tensor-core regime


def _corners(kh, kw):
    return [(0, 0), (kw - 1, 0), (0, kh - 1), (kw - 1, kh - 1)]


def _dyadic(rng, kh, kw, mmax, g):
    m = rng.integers(-mmax, mmax + 1, (kh, kw))
    m[rng.integers(kh), rng.integers(kw)] = mmax        # max|k| reached, so the quantiser's scale is the one the taps were made for
    return (m * 2.0 ** -g).astype(np.float32)


@pytest.mark.parametrize("ddepth", [-1, 3, 5])
def test_u8_reference_vs_port(port, rng, ddepth):
    """8U -> 8U / 16S / 32F, all four borders, anchors at the kernel's four corners, images smaller than the kernel"""
    dt = {-1: np.uint8, 3: np.int16, 5: np.float32}[ddepth]
    g = 2 if ddepth == 3 else 6                 # 16S: sums up to ~6e5, so both ends saturate
    for kh, kw in KSIZES:
        ker = _dyadic(rng, kh, kw, 64, g)
        assert kh * kw * 64 * 255 < 2 ** 24
        for h, w in IMAGES:
            img = rng.integers(0, 256, (h, w), dtype=np.uint8)
            for border in BORDERS:
                for anchor in _corners(kh, kw):
                    want = port.filter2D(img, ddepth, ker, anchor=anchor, delta=-3.25, borderType=border)
                    got = fr.filter2d_u8_ref(img, ker, dt, anchor, -3.25, border, with_true=False).res
                    assert got.dtype == want.dtype
                    assert_exact(got, want, "f2d_reference u8 dd=%d %dx%d image %s border %d anchor %s" % (ddepth, kh, kw, (h, w), border, anchor))


@pytest.mark.parametrize("design", [(4, 9), (12, 4)])       # (b, c): k_lo != 0, a_lo != 0
def test_f32_reference_vs_port(port, rng, design):
    """float data below 2^b, taps m 2^-6 with |m| < 2^c: T3 equals the true sum, and every float operation of the port is exact"""
    b, c = design
    for kh, kw in KSIZES:
        ker = _dyadic(rng, kh, kw, 2 ** c - 1, 6)
        assert 2 ** b * 2 ** c * kh * kw * 1.01 <= 2 ** 24
        khi, klo = fr.bf16_split(ker)
        for h, w in IMAGES:
            img = rng.integers(0, 2 ** b, (h, w)).astype(np.float32)
            ahi, alo = fr.bf16_split(img)
            assert (klo != 0).any() if c > 8 else (alo != 0).any() or img.size < 4
            for border in BORDERS:
                for anchor in _corners(kh, kw):
                    want = port.filter2D(img, -1, ker, anchor=anchor, delta=0.375, borderType=border)
                    ref = fr.filter2d_f32_ref(img, ker, anchor, 0.375, border, grid=6)
                    assert_exact(ref.T3, ref.true, "T3 vs true")
                    assert_exact(ref.res, want, "f2d_reference f32 %s %dx%d image %s border %d anchor %s" % (design, kh, kw, (h, w), border, anchor))


def test_border_extension():
    """pad() against numpy's own padding modes, including reflections that bounce several times off a short axis"""
    img = np.arange(1, 4, dtype=np.uint8)[None, :] * np.array([[1], [10]], np.uint8)        # 2 x 3
    modes = {fr.BORDER_CONSTANT: "constant", fr.BORDER_REPLICATE: "edge", fr.BORDER_REFLECT: "symmetric", fr.BORDER_REFLECT_101: "reflect"}
    for border, mode in modes.items():
        for kh, kw, ax, ay in ((1, 1, 0, 0), (5, 9, 4, 2), (7, 15, 0, 6), (9, 13, 12, 0)):
            got = fr.pad(img, kh, kw, ax, ay, border)[0]
            want = np.pad(img, ((ay, kh - 1 - ay), (ax, kw - 1 - ax)), mode=mode)
            assert_exact(got, want, "pad border %d %dx%d anchor (%d, %d)" % (border, kh, kw, ax, ay))
    # REFLECT "cba|abc|cba", REFLECT_101 "cb|abc|ba", and one-pixel axes
    assert [fr.border_interpolate(p, 3, fr.BORDER_REFLECT) for p in range(-7, 10)] == [0, 0, 1, 2, 2, 1, 0, 0, 1, 2, 2, 1, 0, 0, 1, 2, 2]
    assert [fr.border_interpolate(p, 3, fr.BORDER_REFLECT_101) for p in range(-5, 8)] == [1, 0, 1, 2, 1, 0, 1, 2, 1, 0, 1, 2, 1]
    assert fr.border_interpolate(-9, 1, fr.BORDER_REFLECT_101) == 0 and fr.border_interpolate(9, 1, fr.BORDER_REFLECT) == 0
    assert fr.border_interpolate(-1, 5, fr.BORDER_CONSTANT) == -1


def _kernels(rng):
    """extreme kernels for the quantiser: max|k| an exact power of two (either sign), the largest tap negative, ties of rint of both
    signs, taps below 2^-(sh+1), and ordinary random ones at scales from 1e-29 to 1e29"""
    k = (rng.random((13, 11)) - 0.5).astype(np.float32)
    yield k
    for top in (1.0, 0.5, -1.0, -0.25, 0.99999994, -0.99999994):
        t = k * np.float32(0.49 * abs(top))
        t[6, 5] = top
        yield t.astype(np.float32)
    t = np.zeros((11, 13), np.float32)
    t[0, 0] = 1.0                                          # sh = 21: k 2^21 lands on .5 for odd multiples of 2^-22
    t.flat[1:9] = np.array([3, 5, -3, -5, 7, -7, 1, -1], np.float32) * np.float32(2.0 ** -22)
    t.flat[9:12] = np.float32(2.0 ** -23), np.float32(-2.0 ** -24), np.float32(1e-30)   # below 2^-(sh+1): quantise to 0
    yield t
    for s in (1e-29, 1e29, 3e-30, 7e29):
        yield (k * np.float32(s)).astype(np.float32)


def test_quantiser(rng):
    for k in _kernels(rng):
        kq, sh = fr.quantise(k)
        mx = max(abs(Fraction(float(x))) for x in k.flat)
        assert Fraction(2) ** (21 - sh) <= mx < Fraction(2) ** (22 - sh), "sh = 22 - e with max|k| = m 2^e, m in [0.5, 1)"
        want = np.array([round(Fraction(float(x)) * Fraction(2) ** sh) for x in k.flat], np.int64).reshape(k.shape)   # round half to even
        assert_exact(kq, want, "Kq vs exact rational rounding (sh=%d)" % sh)
        assert np.abs(kq).max() <= 2 ** 22
        d0, d1, d2 = fr.digits(kq)
        assert_exact(d0 + 256 * d1 + 65536 * d2, kq, "digit recombination")
        for d in (d0, d1, d2):
            assert d.min() >= -128 and d.max() <= 127
    t = list(_kernels(rng))[7]
    kq, sh = fr.quantise(t)
    assert sh == 21 and list(kq.flat[:12]) == [2 ** 21, 2, 2, -2, -2, 4, -4, 0, 0, 0, 0, 0], "rint ties to even of both signs; tiny taps 0"
    assert fr.quantise(np.full((1, 1), 1e-29, np.float32))[1] == 118 and fr.quantise(np.full((1, 1), 1e29, np.float32))[1] == -75


def test_digit_extremes():
    """balanced digits reach both -128 and 127; 2^22 (the largest |Kq|) has digits (0, 0, 64)"""
    kq = np.array([127 + 256 * 127 + 65536 * 63, -128 - 256 * 128 - 65536 * 63, 2 ** 22, -2 ** 22, 128, -129, 255], np.int64)
    d0, d1, d2 = fr.digits(kq)
    assert list(d0) == [127, -128, 0, 0, -128, 127, -1] and list(d1) == [127, -128, 0, 0, 1, -1, 1] and list(d2) == [63, -63, 64, -64, 0, 0, 0]


def test_quantisation_bound(rng):
    """|S 2^-sh - true| <= 2^-(sh+1) sum |P| per element, for random kernels at several scales and all borders"""
    img = rng.integers(0, 256, (2, 29, 41), dtype=np.uint8)
    for k in _kernels(rng):
        for border in BORDERS:
            ref = fr.filter2d_u8_ref(img, k, np.float32, (-1, -1), 0.0, border)
            exact = ref.S.astype(np.float64) * 2.0 ** -ref.sh
            slack = 1e-12 * np.abs(ref.true) + 1e-300                  # the f64 tap-by-tap sum's own rounding
            assert (np.abs(exact - ref.true) <= ref.qbound * (1 + 1e-12) + slack).all(), "quantisation bound, sh=%d border %d" % (ref.sh, border)


def test_bf16_split(rng):
    import torch
    a = np.concatenate([
        (rng.standard_normal(20000) * np.exp(rng.uniform(-80, 80, 20000))).astype(np.float32),
        rng.integers(-2 ** 31, 2 ** 31, 4000, dtype=np.int64).astype(np.int32).view(np.float32),        # random bit patterns
        np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, 1.1754942e-38, fr.BF16_MAX, -fr.BF16_MAX, 3.39e38, -3.39e38, 1.0 + 2 ** -8,
                  1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8)], np.float32)])
    a = a[np.isfinite(a) & (np.abs(a) < 3.3961e38)]
    want = torch.from_numpy(a).to(torch.bfloat16).to(torch.float32).numpy()
    assert_exact(fr.bf16_rn(a).view(np.uint32), want.view(np.uint32), "bf16_rn vs torch (bits)")
    hi, lo = fr.bf16_split(a)
    assert_exact(hi.view(np.uint32), want.view(np.uint32), "bf16_split hi")
    assert_exact(lo.view(np.uint32), torch.from_numpy(a - hi).to(torch.bfloat16).to(torch.float32).numpy().view(np.uint32), "bf16_split lo")
    normal = np.abs(a) >= 2.0 ** -100
    err = np.abs(a[normal].astype(np.float64) - hi[normal] - lo[normal])
    assert (err <= 2.0 ** -16 * np.abs(a[normal].astype(np.float64))).all()
    # beyond the largest BF16: torch rounds to infinity, the split saturates hi and keeps lo finite
    big = np.array([np.finfo(np.float32).max, -np.finfo(np.float32).max, 3.3962e38, -3.3962e38], np.float32)
    assert np.isinf(torch.from_numpy(big).to(torch.bfloat16).to(torch.float32).numpy()).all()
    hi, lo = fr.bf16_split(big)
    assert (np.abs(hi) == fr.BF16_MAX).all() and (np.sign(hi) == np.sign(big)).all() and np.isfinite(lo).all()
    assert (np.abs(big.astype(np.float64) - hi - lo) <= 2.0 ** -16 * np.abs(big.astype(np.float64))).all()


def test_hand_values():
    """an all-255 image with a constant kernel: S = 255 sum Kq at every pixel (every border but CONSTANT), S_d = 255 sum d; a one-hot
    kernel moves the image; the float reference of an all-ones image is the sum of the taps' three-plane products"""
    img = np.full((2, 40, 50), 255, np.uint8)
    k = np.full((13, 11), 1 / 143, np.float32)
    for border in BORDERS[1:]:
        ref = fr.filter2d_u8_ref(img, k, np.float32, (-1, -1), 0.0, border)
        assert (ref.S == 255 * int(ref.Kq.sum())).all()
        for sd, d in zip(ref.Sd, fr.digits(ref.Kq)):
            assert (sd == 255 * int(d.sum())).all()
    ref = fr.filter2d_u8_ref(img, k, np.uint8, (-1, -1), 0.0, fr.BORDER_CONSTANT)
    assert ref.S[0, 6, 5] == 255 * int(ref.Kq.sum()) and ref.S[0, 0, 0] == 255 * int(ref.Kq[6:, 5:].sum())
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (23, 31), dtype=np.uint8)
    k = np.zeros((13, 11), np.float32)
    k[2, 7] = 1.0
    got = fr.filter2d_u8_ref(img, k, np.uint8, (0, 0), 0.0, fr.BORDER_CONSTANT).res
    want = np.zeros_like(img)
    want[:-2, :-7] = img[2:, 7:]
    assert_exact(got, want, "one-hot kernel")
    k = (rng.standard_normal((14, 10)) * 0.1).astype(np.float32)
    hi, lo = fr.bf16_split(k)
    ref = fr.filter2d_f32_ref(np.ones((20, 20), np.float32), k, border=fr.BORDER_REPLICATE)
    assert np.allclose(ref.T3, float(hi.astype(np.float64).sum() + lo.astype(np.float64).sum()), rtol=0, atol=1e-12)
