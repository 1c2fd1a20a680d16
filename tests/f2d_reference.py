"""A plain numpy restatement of the two tensor-core filter2D kernels, filter2d_tc.cu (8-bit source) and filter2d_tc_f32.cu (float
source), for the exact filter2D tests.  Test infrastructure only: numpy and scipy, no device code.

8-bit.  The kernel's result is fully defined by its arithmetic, and this module reproduces it bit for bit:
  - the taps are quantised on the host against max|k|: frexp(max|k|) = m 2^e, sh = 22 - e, Kq = rint(k 2^sh) (half to even);
  - Kq is split into three balanced base-256 digits d0, d1, d2 in [-128, 127] (Kq = d0 + 256 d1 + 65536 d2);
  - the integer MMAs give the exact digit-plane sums S_d = sum_{v,u} d(Kq[v, u]) P[y+v, x+u], and S = S0 + 256 S1 + 65536 S2;
  - the epilogue computes fl(fl(float(S) 2^-sh) + delta) in float32 (float(S) is one rounding to nearest, __ll2float_rn; the scale is
    a power of two) and saturates with rint (half to even) for 8U and 16S destinations.
P is the border-extended image (cv::borderInterpolate, common.cuh).

Float.  Every operand a is split as hi = bf16_rn(a), lo = bf16_rn(a - hi), rounding to nearest even on the float32 bits; a finite a
that would round to a BF16 infinity takes hi = the largest finite BF16 of its sign (so lo stays finite).  The kernel accumulates
  T3 = sum (a_hi k_hi + a_hi k_lo + a_lo k_hi)
in FP32 and adds delta; this module gives T3 exactly (or in f64 for random data), the per-element sum of the absolute values of those
three terms (which scales any float32 accumulation error), and the true f64 correlation sum a k.

NaN or inf in the image is outside this model: the tensor-core kernels multiply every padded pixel of a tile's strip by the Toeplitz
zero taps too, so a non-finite pixel spreads to up to 32 + kw - 1 columns of its rows (the reference's own DFT path spreads it further).

Images are (H, W) or a batch (N, H, W); kernels are (kh, kw) float32.  Results have the image's shape.
"""
from collections import namedtuple

import numpy as np
from scipy import signal

BORDER_CONSTANT, BORDER_REPLICATE, BORDER_REFLECT, BORDER_WRAP, BORDER_REFLECT_101 = range(5)
BF16_MAX = float(np.uint32(0x7F7F0000).view(np.float32))       # the largest finite BF16, 3.3895e38


def border_interpolate(p, n, border):
    """cv::borderInterpolate for one coordinate p of an axis of length n; -1 for BORDER_CONSTANT outside the axis"""
    if 0 <= p < n:
        return p
    if border == BORDER_REPLICATE:
        return 0 if p < 0 else n - 1
    if border in (BORDER_REFLECT, BORDER_REFLECT_101):
        delta = 1 if border == BORDER_REFLECT_101 else 0
        if n == 1:
            return 0
        while not 0 <= p < n:                  # bounces as often as needed when the axis is shorter than the kernel
            p = -p - 1 + delta if p < 0 else n - 1 - (p - n) - delta
        return p
    if border == BORDER_WRAP:
        return p % n
    return -1


def pad(img, kh, kw, ax, ay, border):
    """the border-extended image P, (N, H + kh - 1, W + kw - 1) in the image's dtype: P[y, x] = img(border(y - ay), border(x - ax))"""
    img = np.asarray(img)
    imgs = img[None] if img.ndim == 2 else img
    h, w = imgs.shape[1:]
    ys = np.array([border_interpolate(y - ay, h, border) for y in range(h + kh - 1)])
    xs = np.array([border_interpolate(x - ax, w, border) for x in range(w + kw - 1)])
    p = imgs[:, np.maximum(ys, 0)][:, :, np.maximum(xs, 0)]
    p[:, ys < 0] = 0
    p[:, :, xs < 0] = 0
    return p


def _anchor(kh, kw, anchor):
    ax, ay = anchor
    return (kw // 2 if ax < 0 else ax), (kh // 2 if ay < 0 else ay)


def _int_correlate(p, k):
    """exact valid correlation of integer planes p (N, Hp, Wp) and k (kh, kw), int64.  An f64 FFT; every element must land within 1/4
    of an integer (checked), which it does by a wide margin at the magnitudes used here."""
    out = []
    for f in p:
        x = signal.correlate(f.astype(np.float64), k.astype(np.float64), mode="valid", method="fft")
        r = np.rint(x)
        err = float(np.abs(x - r).max()) if x.size else 0.0
        assert err < 0.25, "f2d_reference: the f64 FFT is %g away from an integer" % err
        out.append(r.astype(np.int64))
    return np.stack(out)


def _f64_correlate(p, k):
    """valid correlation in f64, tap by tap (kh kw shifted slices)"""
    kh, kw = k.shape
    oh, ow = p.shape[1] - kh + 1, p.shape[2] - kw + 1
    r = np.zeros((p.shape[0], oh, ow))
    for v in range(kh):
        for u in range(kw):
            if k[v, u] != 0:
                r += float(k[v, u]) * p[:, v:v + oh, u:u + ow]
    return r


def _shape_like(x, img):
    return x[0] if np.asarray(img).ndim == 2 else x


# ---- 8-bit: filter2d_tc.cu ------------------------------------------------------------------------------------------------------

def quantise(k):
    """(Kq int64, sh) exactly as filter2d_u8_tensor: sh = 22 - e with frexp((double)max|k|) = m 2^e, Kq = lrint(ldexp((double)k, sh))"""
    k = np.asarray(k, np.float32)
    mx = float(np.abs(k).max())
    _, e = np.frexp(mx)
    sh = 22 - int(e)
    return np.rint(np.ldexp(k.astype(np.float64), sh)).astype(np.int64), sh


def digits(kq):
    """the three balanced base-256 digits of fc_toeplitz_kernel: kq = d0 + 256 d1 + 65536 d2, d0 and d1 in [-128, 127]"""
    q = np.asarray(kq, np.int64)
    d0 = ((q + 128) & 255) - 128
    q = (q - d0) >> 8
    d1 = ((q + 128) & 255) - 128
    d2 = (q - d1) >> 8
    return d0, d1, d2


# res    result in the destination's dtype (uint8, int16 or float32)
# S      the exact int64 correlation of Kq with P;  Sd  its three digit-plane sums (S = Sd[0] + 256 Sd[1] + 65536 Sd[2])
# true   the f64 correlation of the float taps with P (without delta)
# qbound 2^-(sh+1) sum |P| over the window: |S 2^-sh - true| <= qbound (each tap moves by at most 2^-(sh+1))
# Kq, sh the quantised taps
U8Ref = namedtuple("U8Ref", "res S Sd true qbound Kq sh")


def filter2d_u8_ref(img, k, ddepth=np.uint8, anchor=(-1, -1), delta=0.0, border=BORDER_REFLECT_101, with_true=True):
    """filter2d_tc.cu on an 8-bit image; ddepth is np.uint8, np.int16 or np.float32.  with_true=False skips the f64 correlation
    (kh kw passes over the image) when only the bit-exact result is wanted."""
    img = np.asarray(img)
    assert img.dtype == np.uint8
    k = np.asarray(k, np.float32)
    kh, kw = k.shape
    ax, ay = _anchor(kh, kw, anchor)
    p = pad(img, kh, kw, ax, ay, border)
    kq, sh = quantise(k)
    sd = [_int_correlate(p, d) for d in digits(kq)]
    s = sd[0] + 256 * sd[1] + 65536 * sd[2]
    assert np.abs(s).max(initial=0) < 2 ** 53
    v = s.astype(np.float64).astype(np.float32)                          # __ll2float_rn: one rounding to nearest even
    v = v * np.float32(np.ldexp(1.0, -sh))                               # exact power of two
    v = v + np.float32(delta)
    if ddepth == np.float32:
        res = v
    else:
        lo, hi = (0, 255) if ddepth == np.uint8 else (-32768, 32767)
        res = np.clip(np.rint(v.astype(np.float64)), lo, hi).astype(ddepth)
    true = _f64_correlate(p.astype(np.float64), k.astype(np.float64)) if with_true else None
    pin = p.astype(np.int64)
    qbound = np.ldexp(_int_correlate(pin, np.ones((kh, kw), np.int64)).astype(np.float64), -(sh + 1))
    out = (res, s, tuple(sd), true, qbound)
    out = tuple(None if x is None else (tuple(_shape_like(y, img) for y in x) if isinstance(x, tuple) else _shape_like(x, img)) for x in out)
    return U8Ref(*out, kq, sh)


# ---- float: filter2d_tc_f32.cu ------------------------------------------------------------------------------------------------

def bf16_rn(a):
    """float32 -> the nearest BF16 (ties to even) on the float32 bits, returned as float32; overflow gives inf (as __float2bfloat16_rn)"""
    b = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def bf16_split(a):
    """(hi, lo) of ff_pad_split_kernel / ff_toeplitz_kernel: hi = bf16_rn(a), saturated to +-BF16_MAX for a finite a that would round to
    infinity; lo = bf16_rn(a - hi) (a - hi is exact in float32)"""
    a = np.asarray(a, np.float32)
    hi = bf16_rn(a)
    sat = np.isinf(hi) & np.isfinite(a)
    hi = np.where(sat, np.copysign(np.float32(BF16_MAX), a), hi).astype(np.float32)
    lo = bf16_rn((a - hi).astype(np.float32))
    return hi, lo


# res    fl(T3 + delta), float32: the kernel's result where its FP32 accumulation of T3 is exact
# T3     sum (a_hi k_hi + a_hi k_lo + a_lo k_hi): exact (grid=g) or in f64
# absum  sum |a_hi k_hi| + |a_hi k_lo| + |a_lo k_hi| per element
# true   sum a k in f64;  aksum  sum |a| |k|
F32Ref = namedtuple("F32Ref", "res T3 absum true aksum")


def filter2d_f32_ref(img, k, anchor=(-1, -1), delta=0.0, border=BORDER_REFLECT_101, grid=None, with_true=True):
    """filter2d_tc_f32.cu on a float32 image.  grid=g: the image's BF16 planes are integers and the taps' planes multiples of 2^-g, so
    T3 2^g is an integer correlation, computed exactly (checked); otherwise T3 and the sums are f64 (tap by tap).  with_true=False
    skips true and aksum."""
    img = np.asarray(img, np.float32)
    k = np.asarray(k, np.float32)
    kh, kw = k.shape
    ax, ay = _anchor(kh, kw, anchor)
    p = pad(img, kh, kw, ax, ay, border)
    ahi, alo = bf16_split(p)
    khi, klo = bf16_split(k)
    if grid is not None:
        sc = np.ldexp(1.0, grid)
        ints = [x.astype(np.float64) for x in (ahi, alo)] + [x.astype(np.float64) * sc for x in (khi, klo)]
        assert all((x == np.rint(x)).all() for x in ints), "f2d_reference: the data are not on the 2^-%d grid" % grid
        ai, li, ki, kli = [np.rint(x).astype(np.int64) for x in ints]
        t3 = (_int_correlate(ai, ki + kli) + _int_correlate(li, ki)).astype(np.float64) / sc
        absum = (_int_correlate(np.abs(ai), np.abs(ki) + np.abs(kli)) + _int_correlate(np.abs(li), np.abs(ki))).astype(np.float64) / sc
    else:
        ah, al = ahi.astype(np.float64), alo.astype(np.float64)
        kh64, kl64 = khi.astype(np.float64), klo.astype(np.float64)
        t3 = _f64_correlate(ah, kh64 + kl64) + _f64_correlate(al, kh64)
        absum = _f64_correlate(np.abs(ah), np.abs(kh64) + np.abs(kl64)) + _f64_correlate(np.abs(al), np.abs(kh64))
    true = aksum = None
    if with_true:
        p64 = p.astype(np.float64)
        true = _shape_like(_f64_correlate(p64, k.astype(np.float64)), img)
        aksum = _shape_like(_f64_correlate(np.abs(p64), np.abs(k.astype(np.float64))), img)
    res = (t3 + float(np.float32(delta))).astype(np.float32)             # one rounding: exact (grid) sum plus delta, then to float32
    return F32Ref(*(_shape_like(x, img) for x in (res, t3, absum)), true, aksum)
