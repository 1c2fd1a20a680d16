"""A plain numpy restatement of harris.cu: cornerHarris / cornerMinEigenVal (the response map) and goodFeaturesToTrack's corner
selection, for the exact corner tests.  Test infrastructure only: numpy and scipy, no device code.

Response.  Every float operation of the kernels is spelled out (__fmul_rn, __fadd_rn, explicit fmaf, __fsqrt_rn) and the box sums
are f64 in a stated order, so the result is fully defined and this module reproduces it bit for bit:
  - taps (sobel_taps, sepfilter.cu): binomial smoothing (1 + z)^(n - 1) and derivative (1 + z)^(n - 2) (z - 1); ksize 1 uses 3 taps
    along the derivative and 1 across.  scale = 1 / ((1 << (ksize - 1)) bs (255 for 8U)) in double, rounded to float and multiplied
    in float32 into the smoothing kernel (kx for Dy, ky for Dx).  1-tap kernels are embedded centred in ks taps (corner_response);
  - row pass on the border-extended source: 8U sources and 7-tap float sources in tap order with FMA from 0; 3- and 5-tap float
    sources centre-out, Dx = (r[m+1] - r[m-1]) k[m+1] then fma(r[m+2] - r[m-2], k[m+2], .), Dy = fma(r[m], k[m], (r[m-1] + r[m+1])
    k[m+1]) then fma(r[m-2] + r[m+2], k[m+2], .);
  - column pass, mirrored rows first: Dx = fma(k[m], centre, 0) then fma(k[m+j], down + up, .); Dy from 0 with fma(k[m+j], down - up, .);
  - products dx dx, dx dy, dy dy rounded to float32;
  - the box filter's border applies to the PRODUCT image: an out-of-image position takes the products of the border-interpolated
    position, or 0 for BORDER_CONSTANT;
  - box sums in f64: each box row left to right from 0, then the rows top to bottom;
  - response: fa, fb, fc = float(sums); Harris (fa fc - fb fb) - k ((fa + fc) (fa + fc)) without FMA, k as float; min eigenvalue
    (ha + hc) - sqrt(fb fb + (ha - hc)^2) with ha = fa 0.5, hc = fc 0.5, every step in float32.

numpy has no float32 FMA: fma32 computes it exactly (see there).

Selection (gftt_select).  max of the map in float32; thr = float32(float64(max) quality); TOZERO thresholding with a strict >; the
non-strict 3x3 maximum test on the thresholded map (v != 0, 1-pixel frame excluded); sort by value descending, equal values larger
row-major address first; greedy acceptance on a lrint(min_distance) cell grid over +-1 cells with float dx dx + dy dy < md^2 (only when
min_distance >= 1); stop at max_corners (0 = unlimited).

Sanity bound (corner_response_f64).  A plain f64 evaluation of the same Sobel -> box -> response from independently derived taps
(scipy.ndimage).  Where the float Sobel, the products and the f64 box sums are exact (float data of a few integer levels and a
power-of-two bs, so that every scale is a power of two), the two agree on the box sums exactly and differ only in the response step.
With A, B, C the exact box sums (A, C >= 0, B^2 <= AC by Cauchy-Schwarz) and u = 2^-24, to first order:
  Harris  fa fc carries 2u from the conversions and u from its product, fb fb likewise 3u, the subtraction u (of |AC| + B^2);
          (fa + fc) carries 2u (A, C >= 0, so the conversions and the add are relative to A + C), its square 5u, times k 6u; the
          final subtraction u of |AC| + B^2 + k (A + C)^2.  Total 5u |AC| + 5u B^2 + 7u k (A + C)^2 <= 7u (|AC| + B^2 + k (A + C)^2);
          c = 8 leaves a u for second-order terms:  |R32 - R64| <= 8u (|AC| + B^2 + k (A + C)^2).
  MinEig  X = B^2 + (ha - hc)^2 <= (A + C)^2 / 4, so sqrt(X) <= (A + C) / 2.  The absolute error of X is at most 3u B^2 (fb fb) +
          2u |t| (A + C) / 2 + 2u t^2 (t = ha - hc from rounded halves, its square) + u X (the add); through sqrt (error / 2 sqrt(X),
          plus u sqrt(X) for its rounding) that is <= 4u sqrt(X) + u (A + C) / 2 <= 2.5u (A + C); ha + hc carries 2u (A + C) / 2 and
          the final subtraction u (A + C) / 2.  Total 4u (A + C); with a u of room:  |R32 - R64| <= 5u (A + C).
Images are (H, W) or a batch (N, H, W); results have the image's shape.
"""
from collections import namedtuple

import numpy as np
from scipy import ndimage

from f2d_reference import (BORDER_CONSTANT, BORDER_REFLECT, BORDER_REFLECT_101, BORDER_REPLICATE,  # noqa: F401
                           border_interpolate, pad)

U = 2.0 ** -24
HARRIS_C, MINEIG_C = 8, 5


# ---- float32 FMA ----------------------------------------------------------------------------------------------------------------

def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays, exactly (one rounding to nearest even):
      1. p = f64(a) f64(b) is exact (24 + 24 significant bits);
      2. s = p + f64(c) rounded, e = the exact error of that addition (TwoSum);
      3. if e != 0 and s has an even last mantissa bit, s steps one ulp towards e: s is then p + c rounded to odd at 53 bits;
      4. round s to float32.
    Rounding to odd at 53 bits and then once to nearest at 24 bits (53 >= 24 + 2) gives the correctly rounded result, subnormal
    float32 results included (they have fewer than 24 bits).  The f64 sum can neither overflow nor lose bits to f64 underflow:
    |p| < 2^257, and a non-zero |p| >= 2^-298."""
    a = np.asarray(a, np.float32).astype(np.float64)
    b = np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    even = (np.asarray(s).view(np.int64) & 1) == 0
    fix = (e != 0) & even
    s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


# ---- taps --------------------------------------------------------------------------------------------------------------------------

def _binomial(n, d):
    """(1 + z)^(n - d - 1) (z - 1)^d, low power first (sobel_kernel_1d); n = 1: [1]"""
    p = np.array([1], np.int64)
    if n > 1:
        for _ in range(n - d - 1):
            p = np.convolve(p, [1, 1])
        for _ in range(d):
            p = np.convolve(p, [-1, 1])
    return p


def sobel_taps(dx, dy, ksize, scale):
    """(kx, ky) float32 of sobel_taps for ksize 1/3/5/7: the scale rounded to float and multiplied in float32 into the smoothing kernel"""
    nx = 3 if ksize == 1 and dx > 0 else ksize
    ny = 3 if ksize == 1 and dy > 0 else ksize
    kx = _binomial(nx, dx).astype(np.float32)
    ky = _binomial(ny, dy).astype(np.float32)
    if scale != 1:
        fs = np.float32(scale)
        if dx == 0:
            kx = (kx * fs).astype(np.float32)
        else:
            ky = (ky * fs).astype(np.float32)
    return kx, ky


def corner_scale(ksize, bs, u8):
    """1 / ((1 << (ksize - 1)) bs (255 for 8U)), in double (corner.cpp:247-252)"""
    s = float(1 << (ksize - 1)) * bs
    if u8:
        s *= 255.0
    return 1.0 / s


# dxk_x, dxk_y: Dx = row pass with dxk_x, column pass with dxk_y;  dyk_x, dyk_y likewise;  ks taps per direction
Taps = namedtuple("Taps", "dxk_x dxk_y dyk_x dyk_y ks")


def corner_taps(ksize, bs, u8):
    """the four kernels of HarrisParams, each embedded centred in ks = max length taps (ksize 1: 3)"""
    sc = corner_scale(ksize, bs, u8)
    xkx, xky = sobel_taps(1, 0, ksize, sc)
    ykx, yky = sobel_taps(0, 1, ksize, sc)
    ks = max(len(xkx), len(xky), len(ykx), len(yky))

    def put(v):
        out = np.zeros(ks, np.float32)
        o = (ks - len(v)) // 2
        out[o:o + len(v)] = v
        return out
    return Taps(put(xkx), put(xky), put(ykx), put(yky), ks)


# ---- response ----------------------------------------------------------------------------------------------------------------------

def _batch(img):
    img = np.asarray(img)
    assert img.dtype in (np.uint8, np.float32), img.dtype
    return img[None] if img.ndim == 2 else img


def derivatives(img, ksize, bs, border):
    """(dx, dy) float32 (N, H, W) at the in-image positions: the kernels' row and column passes on the border-extended source"""
    imgs = _batch(img)
    u8 = imgs.dtype == np.uint8
    t = corner_taps(ksize, bs, u8)
    ks, m = t.ks, t.ks // 2
    n, h, w = imgs.shape
    p = pad(imgs, ks, ks, m, m, border).astype(np.float32)         # (N, H + ks - 1, W + ks - 1)
    col = [p[:, :, i:i + w] for i in range(ks)]                     # tap i of the row pass
    if not u8 and ks <= 5:
        rx = (col[m + 1] - col[m - 1]) * t.dxk_x[m + 1]
        ry = fma32(col[m], t.dyk_x[m], (col[m - 1] + col[m + 1]) * t.dyk_x[m + 1])
        if ks == 5:
            rx = fma32(col[m + 2] - col[m - 2], t.dxk_x[m + 2], rx)
            ry = fma32(col[m - 2] + col[m + 2], t.dyk_x[m + 2], ry)
    else:
        rx = np.zeros((n, h + ks - 1, w), np.float32)
        ry = np.zeros_like(rx)
        for i in range(ks):
            rx = fma32(col[i], t.dxk_x[i], rx)
            ry = fma32(col[i], t.dyk_x[i], ry)
    row = lambda a, j: a[:, j:j + h]                                 # noqa: E731  (row j of the column pass)
    dx = fma32(t.dxk_y[m], row(rx, m), np.float32(0))
    dy = np.zeros((n, h, w), np.float32)
    for j in range(1, m + 1):
        dx = fma32(t.dxk_y[m + j], row(rx, m + j) + row(rx, m - j), dx)
        dy = fma32(t.dyk_y[m + j], row(ry, m + j) - row(ry, m - j), dy)
    return dx, dy


def _extend_products(q, bs, border):
    """(N, H + bs - 1, W + bs - 1): the product image under the box filter's border, anchor bs / 2"""
    h, w = q.shape[1:]
    ba = bs // 2
    ys = np.array([border_interpolate(y - ba, h, border) for y in range(h + bs - 1)])
    xs = np.array([border_interpolate(x - ba, w, border) for x in range(w + bs - 1)])
    e = q[:, np.maximum(ys, 0)][:, :, np.maximum(xs, 0)]
    e[:, ys < 0] = 0
    e[:, :, xs < 0] = 0
    return e


def box_sums(prods, bs, border):
    """the f64 box sums of the products (float32 (N, H, W) each): every box row left to right from 0, then the rows top to bottom"""
    out = []
    for q in prods:
        h, w = q.shape[1:]
        e = _extend_products(q, bs, border).astype(np.float64)
        s = np.zeros(q.shape, np.float64)
        for j in range(bs):
            r = np.zeros(q.shape, np.float64)
            for i in range(bs):
                r += e[:, j:j + h, i:i + w]
            s += r
        out.append(s)
    return tuple(out)


def response32(sa, sb, sc, op, k=0.0):
    """the response step: op 0 Harris, 1 min eigenvalue"""
    fa, fb, fc = (np.asarray(x).astype(np.float32) for x in (sa, sb, sc))
    if op == 0:
        acbb = fa * fc - fb * fb
        ac = fa + fc
        return acbb - np.float32(k) * (ac * ac)
    ha, hc = fa * np.float32(0.5), fc * np.float32(0.5)
    t = ha - hc
    t = fb * fb + t * t
    return (ha + hc) - np.sqrt(t)


# res      the response map, float32, the kernels' result bit for bit
# dx, dy   the scaled derivatives;  sums  the f64 box sums (A, B, C) of dx dx, dx dy, dy dy
CornerRef = namedtuple("CornerRef", "res dx dy sums")


def corner_response(img, bs, ksize, border=BORDER_REFLECT_101, op=0, k=0.04):
    imgs = _batch(img)
    assert 1 <= bs <= 31 and ksize in (1, 3, 5, 7) and border in (0, 1, 2, 4)
    dx, dy = derivatives(imgs, ksize, bs, border)
    sums = box_sums((dx * dx, dx * dy, dy * dy), bs, border)
    res = response32(*sums, op, k)
    sh = (lambda x: x[0]) if np.asarray(img).ndim == 2 else (lambda x: x)
    return CornerRef(sh(res), sh(dx), sh(dy), tuple(sh(s) for s in sums))


def corner_harris(img, bs, ksize, k=0.04, border=BORDER_REFLECT_101):
    return corner_response(img, bs, ksize, border, 0, k).res


def corner_min_eigen_val(img, bs, ksize=3, border=BORDER_REFLECT_101):
    return corner_response(img, bs, ksize, border, 1).res


# ---- plain f64 evaluation (sanity bound only) ----------------------------------------------------------------------------------

_MODE = {BORDER_CONSTANT: "constant", BORDER_REPLICATE: "nearest", BORDER_REFLECT: "reflect", BORDER_REFLECT_101: "mirror"}


def corner_response_f64(img, bs, ksize, border=BORDER_REFLECT_101, op=0, k=0.04):
    """(response, (A, B, C)) in f64 from scipy.ndimage with taps derived here from binomial coefficients (not from sobel_taps): a Sobel
    of size n is the smoothing row C(n-1, i) and the difference of C(n-2, i).  Images must be at least as large as the kernels (scipy
    extends a short axis differently from cv::borderInterpolate)."""
    from math import comb
    imgs = _batch(img).astype(np.float64)
    u8 = np.asarray(img).dtype == np.uint8
    n = 3 if ksize == 1 else ksize
    smooth = np.array([comb(ksize - 1, i) for i in range(ksize)], np.float64)
    deriv = np.array([comb(n - 2, i - 1) - comb(n - 2, i) if 0 < i < n - 1 else (1.0 if i == n - 1 else -1.0) for i in range(n)], np.float64)
    scale = 1.0 / ((1 << (ksize - 1)) * bs * (255.0 if u8 else 1.0))
    mode = _MODE[border]
    out, sums = [], []
    for f in imgs:
        dx = ndimage.correlate1d(ndimage.correlate1d(f, deriv, axis=1, mode=mode), smooth * scale, axis=0, mode=mode)
        dy = ndimage.correlate1d(ndimage.correlate1d(f, smooth * scale, axis=1, mode=mode), deriv, axis=0, mode=mode)
        box = np.ones((bs, bs))
        a, b, c = (ndimage.correlate(q, box, mode=mode) for q in (dx * dx, dx * dy, dy * dy))
        out.append(a * c - b * b - k * (a + c) ** 2 if op == 0 else (a + c) / 2 - np.sqrt(b * b + ((a - c) / 2) ** 2))
        sums.append((a, b, c))
    sh = (lambda x: x[0]) if np.asarray(img).ndim == 2 else (lambda x: np.stack(x))
    return sh(out), tuple(sh([s[i] for s in sums]) for i in range(3))


def response_bound(sums, op, k=0.04):
    """the per-element bar |R32 - R64| of the module docstring, from the exact box sums (A, B, C)"""
    a, b, c = (np.asarray(x, np.float64) for x in sums)
    if op == 0:
        return HARRIS_C * U * (np.abs(a * c) + b * b + k * (a + c) ** 2)
    return MINEIG_C * U * (a + c)


# ---- goodFeaturesToTrack selection ---------------------------------------------------------------------------------------------

def gftt_threshold(resp, quality):
    """(max, thr): the map's maximum in float32 and thr = float32(float64(max) quality)"""
    mx = np.float32(np.asarray(resp, np.float32).max())
    return mx, np.float32(float(mx) * quality)


def gftt_candidates(resp, quality):
    """(values float32, positions y W + x int64) of the local maxima above the threshold, in the selection's order: value descending,
    equal values larger row-major address first"""
    r = np.asarray(resp, np.float32)
    h, w = r.shape
    _, thr = gftt_threshold(r, quality)
    t = np.where(r > thr, r, np.float32(0))
    if h < 3 or w < 3:
        return np.zeros(0, np.float32), np.zeros(0, np.int64)
    c = t[1:-1, 1:-1]
    m = c.copy()
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            m = np.maximum(m, t[1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx])
    ys, xs = np.nonzero((c != 0) & ~(m > c))
    vals = c[ys, xs]
    pos = (ys + 1).astype(np.int64) * w + (xs + 1)
    order = np.lexsort((pos, vals))[::-1]
    return vals[order], pos[order]


def gftt_select(resp, max_corners, quality, min_distance):
    """(corners (n, 2) float32 (x, y), qualities (n,) float32) of goodFeaturesToTrack on the response map resp (H, W)"""
    h, w = np.asarray(resp).shape
    vals, pos = gftt_candidates(resp, quality)
    pts, q = [], []
    if min_distance >= 1:
        cell = int(round(min_distance))                          # lrint: half to even, as Python's round
        gw, gh = (w + cell - 1) // cell, (h + cell - 1) // cell
        grid = {}
        md2 = min_distance * min_distance
        for v, p in zip(vals.tolist(), pos.tolist()):
            y, x = divmod(p, w)
            cx, cy = x // cell, y // cell
            keep = True
            for yy in range(max(0, cy - 1), min(gh - 1, cy + 1) + 1):
                for xx in range(max(0, cx - 1), min(gw - 1, cx + 1) + 1):
                    for ax, ay in grid.get((yy, xx), ()):
                        ddx, ddy = np.float32(x) - ax, np.float32(y) - ay
                        if float(ddx * ddx + ddy * ddy) < md2:
                            keep = False
                            break
                    if not keep:
                        break
                if not keep:
                    break
            if not keep:
                continue
            grid.setdefault((cy, cx), []).append((np.float32(x), np.float32(y)))
            pts.append((x, y))
            q.append(v)
            if max_corners > 0 and len(pts) == max_corners:
                break
    else:
        n = len(vals) if max_corners <= 0 else min(max_corners, len(vals))
        for v, p in zip(vals[:n].tolist(), pos[:n].tolist()):
            y, x = divmod(p, w)
            pts.append((x, y))
            q.append(v)
    return np.array(pts, np.float32).reshape(-1, 2), np.array(q, np.float32)
