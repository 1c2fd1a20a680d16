"""A plain float64 / int64 restatement of cv::matchTemplate without a mask (all six methods, 8-bit and float32 images), for the exact
matchTemplate tests.  Test infrastructure only: numpy and scipy, no device code.

For 8-bit data every input of the normalisation is an integer: the correlation numerator R, the window sums S = sum I and Q = sum I^2
and the template's sums.  What remains is the short f64 formula of common_matchTemplate (templmatch.cpp:906-1029, restated in
oracle/port/port_features.c: port_match_template), applied to (double)(float)R.  This module evaluates that formula elementwise in
the same order, and reports beside each result the magnitudes that bound how far another f64 evaluation of it (one with FMA
contraction) can drift; tests/test_gpu_match_template_exact.py derives its bars from them.

Images are (H, W) or a batch (N, H, W); templates are (h, w).  Results are float32, (H-h+1, W-w+1) or (N, H-h+1, W-w+1).
"""
from collections import namedtuple

import numpy as np
from scipy import signal

SQDIFF, SQDIFF_NORMED, CCORR, CCORR_NORMED, CCOEFF, CCOEFF_NORMED = range(6)
FLT_EPSILON = 1.1920928955078125e-07
DBL_EPSILON = 2.220446049250313e-16

# res    float32 result
# big    per element, the largest magnitude of an f64 term of the numerator formula (R, S*mean, Q, templSum2), in numerator units
# t      per element, the normaliser sqrt(max(Q - S^2/n, 0)) * templNorm of the normed methods (0 where the threshold zeroes it);
#        1 for the other methods
# d2     per element, max(Q - S^2/n, 0) (normed methods), or 1
# wnd2   per element, Q (normed methods), or 0: the largest term of d2
# kappa  the template's condition number for its norm: (sum T^2 / n) / var(T) for the CCOEFF methods, 1 otherwise
# clamp  per element, True where the normed result came from the 1.125 clamp (t <= |num| < 1.125 t), not from num / t
MTRef = namedtuple("MTRef", "method res big t d2 wnd2 kappa clamp")


def _frames(img):
    img = np.asarray(img)
    return (img[None], True) if img.ndim == 2 else (img, False)


def ccorr_exact(img, templ):
    """the exact correlation R[y, x] = sum_{v,u} T[v, u] * I[y+v, x+u] of 8-bit data, int64.  An f64 FFT gives every element to well
    within 1/4 of an integer at these sizes; the rounding is checked, so a result that is not clearly an integer fails here, loudly."""
    img = np.asarray(img)
    templ = np.asarray(templ)
    assert img.dtype == np.uint8 and templ.dtype == np.uint8
    imgs, single = _frames(img)
    t64 = templ.astype(np.float64)
    out = []
    for f in imgs:
        x = signal.correlate(f.astype(np.float64), t64, mode="valid", method="fft")
        r = np.rint(x)
        err = float(np.abs(x - r).max())
        assert err < 0.25, "ccorr_exact: the f64 FFT is %g away from an integer" % err
        out.append(r.astype(np.int64))
    out = np.stack(out)
    return out[0] if single else out


def ccorr_f64(img, templ):
    """the correlation of float data accumulated in float64 term by term, and beside it A = sum_{v,u} |T[v, u]| * |I[y+v, x+u]|: the
    scale of the rounding error of any float32 evaluation.  The f64 sum itself is within n * 2^-53 * A of the exact value."""
    imgs, single = _frames(np.asarray(img, np.float64))
    templ = np.asarray(templ, np.float64)
    h, w = templ.shape
    oh, ow = imgs.shape[1] - h + 1, imgs.shape[2] - w + 1
    r = np.zeros((imgs.shape[0], oh, ow))
    a = np.zeros_like(r)
    ai = np.abs(imgs)
    for v in range(h):
        for u in range(w):
            tv = templ[v, u]
            if tv != 0:
                r += tv * imgs[:, v:v + oh, u:u + ow]
                a += abs(tv) * ai[:, v:v + oh, u:u + ow]
    return (r[0], a[0]) if single else (r, a)


def window_sums(img, w, h):
    """per window of w x h: (S, Q) = (sum I, sum I^2), from int64 integral images for 8-bit data (exact) and f64 ones otherwise"""
    imgs, single = _frames(img)
    dt = np.int64 if imgs.dtype == np.uint8 else np.float64
    x = imgs.astype(dt)
    out = []
    for p in (x, x * x):
        ii = np.zeros((p.shape[0], p.shape[1] + 1, p.shape[2] + 1), dt)
        ii[:, 1:, 1:] = p.cumsum(1).cumsum(2)
        out.append(ii[:, h:, w:] - ii[:, :-h, w:] - ii[:, h:, :-w] + ii[:, :-h, :-w])
    return (out[0][0], out[1][0]) if single else tuple(out)


def template_stats(templ, method):
    """(mean, templNorm, templSum2, invArea, flat, kappa) as common_matchTemplate derives them from the template's mean and
    standard deviation (meanStdDev semantics)"""
    templ = np.asarray(templ)
    n = templ.size
    t = templ.astype(np.int64 if templ.dtype == np.uint8 else np.float64)
    ts, tq = float(t.sum()), float((t * t).sum())
    scale = 1.0 / n
    mean = ts * scale
    var = max(tq * scale - mean * mean, 0.0)
    sdv = np.sqrt(var)
    templ_norm = sdv * sdv
    inv_area = 1.0 / (float(templ.shape[0]) * templ.shape[1])
    num_type = 0 if method in (CCORR, CCORR_NORMED) else 1 if method in (CCOEFF, CCOEFF_NORMED) else 2
    flat = templ_norm < DBL_EPSILON and method == CCOEFF_NORMED
    kappa = (tq * scale) / var if num_type == 1 and var > 0 else 1.0
    templ_sum2 = templ_norm + mean * mean
    if num_type != 1:
        mean = 0.0
        templ_norm = templ_sum2
    templ_sum2 /= inv_area
    templ_norm = np.sqrt(templ_norm) / np.sqrt(inv_area)
    return mean, templ_norm, templ_sum2, inv_area, flat, kappa


def match_template_ref(img, templ, method, r=None):
    """cv::matchTemplate(img, templ, method) without a mask, elementwise in f64 as port_match_template evaluates it; returns an MTRef.
    r: the numerator if already computed (ccorr_exact / ccorr_f64), so that several methods share one correlation."""
    img = np.asarray(img)
    templ = np.asarray(templ)
    h, w = templ.shape
    if r is not None:
        r = np.asarray(r, np.float64)
    elif img.dtype == np.uint8:
        r = ccorr_exact(img, templ).astype(np.float64)
    else:
        r = ccorr_f64(img, templ)[0]
    num = r.astype(np.float32).astype(np.float64)       # both the library and the reference round the numerator to float first
    ones = np.ones_like(num)
    if method == CCORR:
        return MTRef(method, num.astype(np.float32), np.abs(num), ones, ones, 0 * ones, 1.0, ones < 0)
    mean, templ_norm, templ_sum2, inv_area, flat, kappa = template_stats(templ, method)
    if flat:
        return MTRef(method, ones.astype(np.float32), 0 * ones, ones, ones, 0 * ones, 1.0, ones < 0)
    num_type = 0 if method in (CCORR, CCORR_NORMED) else 1 if method in (CCOEFF, CCOEFF_NORMED) else 2
    normed = method in (SQDIFF_NORMED, CCORR_NORMED, CCOEFF_NORMED)
    s, q = window_sums(img, w, h)
    s = s.astype(np.float64)
    q = q.astype(np.float64)
    big = np.abs(num)
    wnd_mean2 = np.zeros_like(num)
    wnd_sum2 = np.zeros_like(num)
    if num_type == 1:
        big = np.maximum(big, np.abs(s * mean))
        wnd_mean2 = s * s
        num = num - s * mean
        wnd_mean2 = wnd_mean2 * inv_area
    if normed or num_type == 2:
        wnd_sum2 = wnd_sum2 + q
        if num_type == 2:
            big = np.maximum(np.maximum(2 * big, q), templ_sum2)
            num = np.maximum(q - 2 * num + templ_sum2, 0.0)
    if not normed:
        return MTRef(method, num.astype(np.float32), big, ones, ones, 0 * ones, kappa, ones < 0)
    d2 = np.maximum(wnd_sum2 - wnd_mean2, 0.0)
    t = np.where(d2 <= np.minimum(0.5, 10 * FLT_EPSILON * wnd_sum2), 0.0, np.sqrt(d2) * templ_norm)
    a = np.abs(num)
    inside = a < t
    clamp = ~inside & (a < t * 1.125)
    with np.errstate(divide="ignore", invalid="ignore"):
        res = np.where(inside, num / np.where(t > 0, t, 1.0), np.where(clamp, np.where(num > 0, 1.0, -1.0), 0.0 if method != SQDIFF_NORMED else 1.0))
    return MTRef(method, res.astype(np.float32), big, t, d2, wnd_sum2, kappa, clamp)


def allowance(ref, dnum=0.0, ulps=8):
    """per element bound on |other - ref.res| for another evaluation of the same formula, whose numerator R is within dnum of the one
    this module rounded to float (0 for 8-bit data) and whose f64 operations may round each term up to `ulps` units of 2^-53 of its
    magnitude differently (FMA contraction, summation order); derived in tests/test_gpu_match_template_exact.py.  Includes the final
    rounding to float32.  Zero allowance before that rounding where the normed methods' threshold gives t = 0 (the result is then a
    constant that no rounding of the terms changes)."""
    normed = ref.method in (SQDIFF_NORMED, CCORR_NORMED, CCOEFF_NORMED)
    if ref.method in (SQDIFF, SQDIFF_NORMED):
        dnum = 2 * dnum                              # R enters as Q - 2 R + templSum2
    pos = ref.t > 0
    tt = np.where(pos, ref.t, 1.0)
    e = dnum / tt + ulps * 2.0 ** -53 * ref.big / tt
    if normed:
        r = np.abs(ref.res.astype(np.float64))
        e = e + ulps * 2.0 ** -53 * r * (1 + ref.wnd2 / np.where(ref.d2 > 0, ref.d2, 1.0) + ref.kappa)
        e = np.where(pos, e, 0.0)
    return e + np.spacing((np.abs(ref.res.astype(np.float64)) + e).astype(np.float32)).astype(np.float64)
