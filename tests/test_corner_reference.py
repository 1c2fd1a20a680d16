"""CPU: the numpy restatement of harris.cu (tests/corner_reference.py) against exact rational arithmetic, hand-written taps and values,
a plain f64 evaluation, and the plain-C port (oracle/port/port_features.c, built with -ffp-contract=off).  The GPU tests of
tests/test_gpu_corner_exact.py hold the device to this restatement bit for bit, so it is checked here first, on every machine.

The port computes the Sobel with the same operation order as the kernels (tap-order FMA rows for 8-bit and 7-tap float sources,
centre-out 3- and 5-tap float rows, mirrored-rows-first columns; port_filter.c: sep_float), rounds the products to float, sums the box
in f64 row by row from the border-interpolated product image and evaluates the same float response.  Its selection is pinned bit for
bit to the reference's goodFeaturesToTrack (tests/test_oracle.py).  The restatement therefore has to equal it bit for bit, on every
border, block size and image size tried here, and it does: no case needed a bar.
"""
from fractions import Fraction

import numpy as np
import pytest

import corner_reference as cr
from util import assert_exact

BORDERS = [cr.BORDER_CONSTANT, cr.BORDER_REPLICATE, cr.BORDER_REFLECT, cr.BORDER_REFLECT_101]
# an ordinary image, 1 x 1, 2 x N, N x 2, one row, one column, images smaller than the box (bs 31) and than the Sobel
IMAGES = [(37, 45), (1, 1), (2, 9), (9, 2), (1, 17), (23, 1), (5, 40), (40, 6), (3, 3)]


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _round_f32(x):
    """a Fraction rounded to the nearest float32, ties to even (subnormals included, no overflow)"""
    if x == 0:
        return np.float32(0)
    e = abs(x.numerator).bit_length() - abs(x.denominator).bit_length()
    while Fraction(2) ** e > abs(x):
        e -= 1
    while Fraction(2) ** (e + 1) <= abs(x):
        e += 1
    ulp = Fraction(2) ** max(e - 23, -149)
    return np.float32(float(round(x / ulp) * ulp))          # Fraction.__round__: half to even; the product is exact in float


def _img(rng, shape, dt):
    img = rng.integers(0, 256, shape, dtype=np.uint8)
    if dt == np.float32:
        img = (img / np.float32(255) + rng.random(shape, dtype=np.float32) * np.float32(0.01)).astype(np.float32)
    return img


# ---- FMA emulation --------------------------------------------------------------------------------------------------------------

def _fma_cases(rng):
    n = 20000
    a = (rng.standard_normal(n) * np.exp2(rng.integers(-60, 60, n))).astype(np.float32)
    b = (rng.standard_normal(n) * np.exp2(rng.integers(-60, 60, n))).astype(np.float32)
    c = (rng.standard_normal(n) * np.exp2(rng.integers(-120, 120, n))).astype(np.float32)
    yield a, b, c, "random"
    # cancellation: c = -fl(a b) (+- a few ulp), the result is the product's rounding error
    p = (a * b).astype(np.float32)
    yield a, b, (-p + np.where(rng.random(n) < 0.5, 0, np.spacing(p))).astype(np.float32), "cancellation"
    # exact midpoints: (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 is half an ulp above 1 + 2^-11; a far smaller c must decide the rounding
    one = np.float32(1 + 2 ** -12)
    mid = []
    for s in (1, -1):
        for cc in (0.0, 2.0 ** -60, -2.0 ** -60, 2.0 ** -149, -2.0 ** -149, 2.0 ** -23, -2.0 ** -24):
            mid.append((s * one, one, s * cc))
        mid.append((s * np.float32(1 + 2 ** -12), np.float32(1 + 3 * 2 ** -12), 0.0))     # 1 + 2^-10 + 3 2^-24: above the midpoint
        mid.append((s * np.float32(3.0), np.float32(1 + 2 ** -23), s * -3.0))             # 3 2^-23 exactly
    m = np.array(mid, np.float64).astype(np.float32)
    yield m[:, 0], m[:, 1], m[:, 2], "midpoints"
    # subnormal results: products near 2^-140 .. 2^-150 and subnormal addends
    k = 5000
    a = (rng.uniform(1, 2, k) * np.exp2(rng.integers(-80, -60, k))).astype(np.float32)
    b = (rng.uniform(-2, 2, k) * np.exp2(-140.0 - np.log2(a.astype(np.float64)) + rng.integers(-8, 3, k))).astype(np.float32)
    c = (rng.integers(-2 ** 23, 2 ** 23, k) * 2.0 ** -149).astype(np.float32)
    yield a, b, c, "subnormal"


def test_fma32_vs_fractions(rng):
    for a, b, c, what in _fma_cases(rng):
        got = cr.fma32(a, b, c)
        want = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], np.float32)
        nz = want != 0
        assert_exact(_bits(got[nz]), _bits(want[nz]), "fma32 vs Fraction (%s)" % what)
        assert (got[~nz] == 0).all(), "fma32 exact zeros (%s)" % what
        if what == "subnormal":
            assert (np.abs(want[nz]) < np.finfo(np.float32).tiny).sum() > 1000, "the subnormal case reaches subnormal results"
        if what == "midpoints":
            plain = (a.astype(np.float64) * b + c).astype(np.float32)
            assert (plain != got).any(), "the midpoint case includes a triple that a double rounding gets wrong"


# ---- taps ---------------------------------------------------------------------------------------------------------------------

def _scaled(v, den):
    return (np.array(v, np.float32) * np.float32(1.0 / den)).astype(np.float32)


@pytest.mark.parametrize("u8", [True, False])
def test_taps(u8):
    """every ksize at both depths against hand-written binomial taps; the scale goes into the smoothing kernel, and 1-tap kernels sit in
    the middle of 3"""
    d = 255 if u8 else 1
    hand = {
        1: ([-1, 0, 1], [1], 1),
        3: ([-1, 0, 1], [1, 2, 1], 4),
        5: ([-1, -2, 0, 2, 1], [1, 4, 6, 4, 1], 16),
        7: ([-1, -4, -5, 0, 5, 4, 1], [1, 6, 15, 20, 15, 6, 1], 64),
    }
    for ksize, (deriv, smooth, norm) in hand.items():
        for bs in (1, 2, 3, 7, 31):
            t = cr.corner_taps(ksize, bs, u8)
            den = norm * bs * d
            sm = _scaled(smooth, den)
            if ksize == 1:
                sm = np.array([0, sm[0], 0], np.float32)
            assert t.ks == max(3, ksize)
            assert_exact(_bits(t.dxk_x), _bits(np.array(deriv, np.float32)), "Dx row taps ksize %d" % ksize)
            assert_exact(_bits(t.dyk_y), _bits(np.array(deriv, np.float32)), "Dy column taps ksize %d" % ksize)
            assert_exact(_bits(t.dxk_y), _bits(sm), "Dx column taps ksize %d bs %d u8 %s" % (ksize, bs, u8))
            assert_exact(_bits(t.dyk_x), _bits(sm), "Dy row taps ksize %d bs %d u8 %s" % (ksize, bs, u8))
    # the scale is rounded to float once, then multiplied in float: 1 / (4 3 255) is not a power of two
    fs = np.float32(1.0 / (4 * 3 * 255))
    assert cr.corner_taps(3, 3, True).dxk_y[1] == np.float32(np.float32(2) * fs)
    assert cr.corner_scale(7, 31, True) == 1.0 / (64.0 * 31 * 255)


# ---- response against the port --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", [np.uint8, np.float32])
@pytest.mark.parametrize("ksize", [1, 3, 5, 7])
def test_response_vs_port(port, rng, dt, ksize):
    """bit for bit: Harris and min eigenvalue, all four borders, bs 1 - 31, images down to 1 x 1 and smaller than the box"""
    spikes = rng.random((30, 41), dtype=np.float32)
    spikes[3::9, 4::11] = np.float32(2.0 ** 30)            # box sums whose float value depends on the order of the f64 additions
    for img in [_img(rng, shape, dt) for shape in IMAGES] + ([spikes] if dt == np.float32 else []):
        shape = img.shape
        for bs in (1, 2, 3, 4, 5, 7, 30, 31):
            for border in BORDERS:
                what = "%s %s ksize %d bs %d border %d" % (np.dtype(dt).name, shape, ksize, bs, border)
                assert_exact(_bits(cr.corner_harris(img, bs, ksize, 0.04, border)), _bits(port.cornerHarris(img, bs, ksize, 0.04, border)),
                             "cornerHarris " + what)
                assert_exact(_bits(cr.corner_min_eigen_val(img, bs, ksize, border)), _bits(port.cornerMinEigenVal(img, bs, ksize, border)),
                             "cornerMinEigenVal " + what)


def test_response_batch(rng):
    """a batch is its frames, each on its own"""
    img = _img(rng, (3, 21, 34), np.uint8)
    got = cr.corner_response(img, 3, 3, cr.BORDER_REFLECT, 1).res
    for f in range(3):
        assert_exact(_bits(got[f]), _bits(cr.corner_min_eigen_val(img[f], 3, 3, cr.BORDER_REFLECT)), "frame %d" % f)


# ---- selection against the port --------------------------------------------------------------------------------------------------

def _selection_images(rng):
    yield "noise", rng.integers(0, 256, (60, 80), dtype=np.uint8)
    yield "tiled 8x8", np.tile(rng.integers(0, 256, (8, 8), dtype=np.uint8), (9, 12))           # interior responses tie exactly
    yield "tiled 4x4 binary", np.tile(rng.integers(0, 2, (4, 4), dtype=np.uint8) * 255, (20, 20))
    yield "smooth", np.kron(rng.integers(0, 256, (10, 12)), np.ones((7, 7))).astype(np.uint8)


@pytest.mark.parametrize("harris", [True, False])
def test_selection_vs_port(port, rng, harris):
    """gftt_select on the restated map = the port's goodFeaturesToTrack: positions, order and qualities; ties, min_distance 0 / 1 / 5 /
    10.5, max_corners 0 (unlimited), a few, and more than there are candidates"""
    for name, img in _selection_images(rng):
        resp = cr.corner_response(img, 3, 3, cr.BORDER_REFLECT_101, 0 if harris else 1).res
        ncand = len(cr.gftt_candidates(resp, 0.01)[0])
        assert ncand > 20
        if name.startswith("tiled"):
            assert len(np.unique(cr.gftt_candidates(resp, 0.01)[0])) < ncand // 10, "ties"
        for md in (0, 1, 5, 10.5):
            for mc in (0, 7, ncand + 5):
                for q in (0.01, 0.3):
                    gp, gq = cr.gftt_select(resp, mc, q, md)
                    wp, wq = port.goodFeaturesToTrack(img, mc, q, md, 3, 3, harris, 0.04)
                    what = "%s harris %s md %g mc %d q %g" % (name, harris, md, mc, q)
                    assert_exact(gp, wp, "corners " + what)
                    assert_exact(_bits(gq), _bits(wq), "qualities " + what)


def test_selection_rules():
    """hand-made maps: the threshold is strict, the 3x3 test is not, equal values go larger address first, the frame is excluded, a
    corner at exactly min_distance is accepted"""
    r = np.zeros((7, 9), np.float32)
    r[2, 2] = r[2, 3] = 4.0            # equal neighbours: both pass the non-strict test
    r[4, 6] = 2.0
    r[5, 1] = 0.04                     # = float32(4 * 0.01): not above the threshold
    r[0, 4] = 9.0                      # the maximum, on the frame: never a corner, but it sets the threshold
    pts, q = cr.gftt_select(r, 0, 0.01 * 4 / 9, 0)
    assert np.float32(9.0 * (0.01 * 4 / 9)) == np.float32(0.04)
    assert pts.tolist() == [[3, 2], [2, 2], [6, 4]] and q.tolist() == [4.0, 4.0, 2.0]
    pts, _ = cr.gftt_select(r, 0, 0.01 * 4 / 9, 1)          # (2, 2) is 1 away from (3, 2): rejected (1 < 1 is false: accepted)
    assert pts.tolist() == [[3, 2], [2, 2], [6, 4]]
    pts, _ = cr.gftt_select(r, 0, 0.01 * 4 / 9, 1.5)
    assert pts.tolist() == [[3, 2], [6, 4]]
    pts, _ = cr.gftt_select(r, 2, 0.01 * 4 / 9, 0)
    assert len(pts) == 2
    for m in (np.zeros((6, 6), np.float32), np.full((6, 6), -1, np.float32), np.ones((2, 9), np.float32)):
        assert len(cr.gftt_select(m, 0, 0.01, 0)[0]) == 0


# ---- hand-computed values and the f64 evaluation -------------------------------------------------------------------------------

def test_hand_values():
    """one bright pixel on zeros, ksize 3, bs 2 (scale 1/8): around it dx = +-0.25 beside and +-0.125 on the diagonals, dy likewise; the
    2 x 2 box at the pixel (anchor 1) holds A = C = 5/64, B = 1/64, so Harris = 24/4096 - k (10/64)^2 and minEig = 5/64 - 1/64"""
    img = np.zeros((5, 5), np.float32)
    img[2, 2] = 1.0
    ref = cr.corner_response(img, 2, 3, cr.BORDER_REFLECT_101, 0, 0.04)
    assert ref.dx[2, 1] == 0.25 and ref.dx[2, 3] == -0.25 and ref.dx[1, 1] == 0.125 and ref.dx[1, 2] == 0 and ref.dx[2, 2] == 0
    assert ref.dy[1, 2] == 0.25 and ref.dy[3, 2] == -0.25 and ref.dy[1, 1] == 0.125
    assert [s[2, 2] for s in ref.sums] == [5 / 64, 1 / 64, 5 / 64]
    assert ref.res[2, 2] == np.float32(24 / 4096) - np.float32(0.04) * np.float32(100 / 4096)
    assert cr.corner_min_eigen_val(img, 2, 3)[2, 2] == np.float32(1 / 16)
    # 8-bit: the same pixel at 255 gives the same derivatives (the scale carries 1/255)
    u8 = (img * 255).astype(np.uint8)
    assert_exact(_bits(cr.corner_harris(u8, 2, 3)), _bits(ref.res), "8-bit pixel at 255")
    # a ramp along x: dx = 2 / bs inside (the scale holds 1 / bs, exact for bs a power of two), dy = 0, A = bs^2 (2 / bs)^2 = 4;
    # Harris = -16 k and minEig = 0 away from the border
    ramp = np.tile(np.arange(12, dtype=np.float32), (10, 1))
    for bs in (2, 4):
        h = cr.corner_harris(ramp, bs, 3, 0.04)
        assert (h[3:-3, 3:-3] == -(np.float32(0.04) * np.float32(16))).all()
        assert (cr.corner_min_eigen_val(ramp, bs, 3)[3:-3, 3:-3] == 0).all()
    # constant images: no gradient anywhere, except where BORDER_CONSTANT brings in zeros
    for border in BORDERS[1:]:
        assert (cr.corner_harris(np.full((9, 11), 200, np.uint8), 3, 5, 0.04, border) == 0).all()
    assert (cr.corner_harris(np.full((9, 11), 200, np.uint8), 3, 5, 0.04, cr.BORDER_CONSTANT) != 0).any()


@pytest.mark.parametrize("ksize", [1, 3, 5, 7])
def test_f64_sanity(rng, ksize):
    """float data of four integer levels and bs a power of two: every scale is a power of two, so the float Sobel, the products and the
    f64 box sums are exact, and the independent f64 evaluation must give the same box sums; the responses then differ only by the
    response step's roundings, within the bound derived in corner_reference"""
    for bs in (1, 2, 4, 8, 16):
        for border in BORDERS:
            img = rng.integers(0, 4, (2, 40, 50)).astype(np.float32)
            for op in (0, 1):
                ref = cr.corner_response(img, bs, ksize, border, op, 0.04)
                r64, s64 = cr.corner_response_f64(img, bs, ksize, border, op, 0.04)
                what = "ksize %d bs %d border %d op %d" % (ksize, bs, border, op)
                for a, b in zip(ref.sums, s64):
                    assert_exact(a, b, "box sums vs f64 " + what)
                d = np.abs(ref.res.astype(np.float64) - r64)
                lim = cr.response_bound(s64, op, 0.04)
                assert (d <= lim).all(), "%s: |R32 - R64| %g above the bound %g" % (what, d.max(), lim[np.unravel_index(d.argmax(), d.shape)])
                assert np.abs(r64).max() > 0 or (bs == 1 and op == 1), "a 1 x 1 box has rank 1: its min eigenvalue is 0"
