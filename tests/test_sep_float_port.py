"""The C port's float separable filter (oracle/port/port_filter.c, sep_float) against an independent float64 correlation.

tests/test_gpu_sep_float_exact.py ties the CUDA kernels to the port bit for bit, so a formula wrong in both (tap order, anchor, border
index) would pass there.  Here the port's f32 -> f32 and 8U -> 32F sepFilter2D must stay within a rounding bound of an exact f64
correlation written from the definition, with its own border code.

The bound.  With u = 2^-24 and gamma_n = n u / (1 - n u):
  rows     an FMA chain of n terms from 0 (or the centre-out order of the 3/5-tap rows: at most one more rounding per pair) gives
           |S^ - S| <= gamma_(nx+1) sum_i |kx_i x_i|                                                    =: E(row)
  columns  the mirrored pairs are added (one rounding) before the FMA chain, the scalar order rounds each product then adds; either way
           |y^ - y(S^)| <= gamma_(ny+2) (|delta| + sum_j |ky_j S^_j|), and the row errors pass through linearly:
  total    |y^ - y| <= gamma_(ny+2) (|delta| + sum_j |ky_j| |S^_j|) + sum_j |ky_j| E(row j)
A wrong tap order or anchor moves a result by a whole tap times a pixel difference, far above this.

The port's equality with the reference's SIMD body is held in test_oracle.py
(test_port_float_separable_filters_follow_the_reference_operation_order).
"""
import numpy as np
import pytest

U = 2.0 ** -24
CONST, REPL, REFL, WRAP, R101 = 0, 1, 2, 3, 4


def gamma(n):
    return n * U / (1 - n * U)


def border_index(p, n, border):
    """cv::borderInterpolate, written from its definition; -1 = outside (BORDER_CONSTANT)"""
    if 0 <= p < n:
        return p
    if border == CONST:
        return -1
    if border == REPL:
        return 0 if p < 0 else n - 1
    if border == WRAP:
        return p % n
    if n == 1:
        return 0
    while not 0 <= p < n:       # REFLECT: fedcba|abcdefgh ; REFLECT_101: gfedcb|abcdefgh
        p = -p - 1 + (border == R101) if p < 0 else 2 * n - 1 - p - (border == R101)
    return p


def corr1d(a, k, anchor, border, axis):
    """float64 correlation along axis: out[i] = sum_t k[t] a[i + t - anchor], plus sum_t |k[t] a[...]|"""
    a = np.moveaxis(a, axis, 0)
    n = a.shape[0]
    out = np.zeros(a.shape, np.float64)
    mag = np.zeros(a.shape, np.float64)
    for t, kt in enumerate(np.asarray(k, np.float64)):
        idx = np.array([border_index(i + t - anchor, n, border) for i in range(n)])
        v = np.where((idx >= 0)[(slice(None),) + (None,) * (a.ndim - 1)], a[np.maximum(idx, 0)], 0.0)
        out += kt * v
        mag += np.abs(kt * v)
    return np.moveaxis(out, 0, axis), np.moveaxis(mag, 0, axis)


def f64_bound(src, kx, ky, anchor, delta, border):
    """exact result and the rounding bound of the docstring"""
    nx, ny = len(kx), len(ky)
    ax = nx // 2 if anchor[0] < 0 else anchor[0]
    ay = ny // 2 if anchor[1] < 0 else anchor[1]
    x = src.astype(np.float64)
    S, Smag = corr1d(x, kx, ax, border, 1)
    Erow = gamma(nx + 1) * Smag
    y, _ = corr1d(S, ky, ay, border, 0)
    y += delta
    # |ky_j| |S^_j| <= |ky_j| (|S_j| + E_j)
    absS, _ = corr1d(np.abs(S) + Erow, np.abs(ky), ay, border, 0)
    prop, _ = corr1d(Erow, np.abs(ky), ay, border, 0)
    bound = gamma(ny + 2) * (abs(delta) + absS) + prop
    return y, bound * (1 + 1e-12) + 1e-300


def taps(rng, n, kind):
    k = rng.random(n) - 0.3
    if kind == "sym":
        k = k + k[::-1]
    elif kind == "asym":
        k = k - k[::-1]
    return (k / np.abs(k).sum()).astype(np.float32)


CASES = [((3, 3), ("sym", "sym"), (-1, -1)), ((5, 5), ("asym", "sym"), (-1, -1)), ((3, 5), ("sym", "asym"), (-1, -1)),
         ((7, 3), ("rand", "sym"), (-1, -1)), ((19, 23), ("rand", "sym"), (-1, -1)), ((31, 29), ("sym", "asym"), (-1, -1)),
         ((4, 6), ("rand", "rand"), (-1, -1)), ((6, 3), ("rand", "sym"), (1, -1)), ((5, 7), ("rand", "rand"), (0, 6)),
         ((33, 9), ("rand", "sym"), (3, 2)), ((1, 7), ("sym", "sym"), (-1, -1)), ((9, 1), ("rand", "sym"), (-1, -1)),
         ((2, 2), ("rand", "rand"), (1, 0))]


@pytest.mark.parametrize("border", [CONST, REPL, REFL, WRAP, R101])
@pytest.mark.parametrize("ks,kinds,anchor", CASES)
def test_port_within_f64_bound(port, rng, ks, kinds, anchor, border):
    nx, ny = ks
    kx, ky = taps(rng, nx, kinds[0]), taps(rng, ny, kinds[1])
    e = rng.integers(-6, 9, (23, 1)).astype(np.float64)
    for src in (((rng.random((23, 41)) - 0.3) * 2.0 ** e).astype(np.float32), rng.integers(0, 256, (23, 41), dtype=np.uint8),
                ((rng.random((4, 3)) - 0.5) * 8).astype(np.float32)):
        for delta in (0.0, 1.375):
            got = port.sepFilter2D(src, 5, kx, ky, anchor, delta, border).astype(np.float64)
            want, bound = f64_bound(src, kx, ky, anchor, delta, border)
            bad = np.abs(got - want) > bound
            assert not bad.any(), "%s %dx%d %s a=%s b=%d delta=%g: %d elements beyond the bound, first %s (got %r want %r bound %g)" % (
                src.dtype, nx, ny, kinds, anchor, border, delta, bad.sum(), tuple(np.argwhere(bad)[0]), got[bad][0], want[bad][0], bound[bad][0])


def test_bound_catches_a_wrong_anchor(port, rng):
    """the bound is tight enough to see one tap off: an anchor moved by one fails it"""
    kx, ky = taps(rng, 5, "rand"), taps(rng, 5, "sym")
    src = (rng.random((23, 41)) * 10).astype(np.float32)
    got = port.sepFilter2D(src, 5, kx, ky, (2, -1), 0.0, R101).astype(np.float64)
    want, bound = f64_bound(src, kx, ky, (1, -1), 0.0, R101)
    assert (np.abs(got - want) > bound).mean() > 0.9


@pytest.mark.parametrize("nx,ny", [(3, 3), (5, 3), (3, 7), (19, 19), (23, 9), (29, 29), (7, 13), (4, 6)])
@pytest.mark.parametrize("special", [np.inf, -np.inf, np.nan])
def test_port_non_finite_footprint(port, rng, nx, ny, special):
    """An inf or NaN pixel reaches exactly the outputs whose window holds it with a non-zero tap: the kernel's own footprint, not
    the footprint of the bucket the device pads the kernel to"""
    kx = (rng.random(nx) + 0.1).astype(np.float32)
    ky = (rng.random(ny) + 0.1).astype(np.float32)
    if nx in (3, 5):
        kx = ((kx + kx[::-1]) / 2).astype(np.float32)         # the centre-out small-row order
    ky = ((ky + ky[::-1]) / 2).astype(np.float32)
    src = (rng.random((60, 70)) - 0.5).astype(np.float32)
    py, px = 30, 33
    src[py, px] = special
    for b in (CONST, R101):
        out = port.sepFilter2D(src, -1, kx, ky, (-1, -1), 0.0, b)
        ax, ay = nx // 2, ny // 2
        fp = np.zeros(out.shape, bool)
        fp[py - (ny - 1 - ay):py + ay + 1, px - (nx - 1 - ax):px + ax + 1] = True
        bad = ~np.isfinite(out)
        assert np.array_equal(bad, fp), "%dx%d %r b=%d: non-finite outputs %s, footprint %s" % (
            nx, ny, special, b, np.argwhere(bad)[[0, -1]].tolist(), np.argwhere(fp)[[0, -1]].tolist())
        if np.isinf(special):        # positive taps: the sign survives
            assert np.all(out[fp] == special)
