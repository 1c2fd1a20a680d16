"""Plain numpy restatement of cv::Canny (imgproc/src/canny.cpp:823-1003) -- the checker for opencv_b200's Canny kernels.

It shares no algorithm with the CUDA code: the 16S Sobel / Scharr is a direct integer correlation, and the hysteresis is the reference's
own stack flood fill from the strong pixels (canny.cpp:647-678, :914-927), not union-find.  `hysteresis_labels` (scipy's connected-
component labelling) gives the same set faster and is only used for large frames, after the tests have held it equal to the flood fill.

Also here: `RefCanny`, ctypes access to the compiled reference's two cv::Canny overloads (oracle/_ref/libcannyref*.so, built by
tools/build_canny_ref.py where the reference is available).
"""
import ctypes
import math
import os

import numpy as np

INT_MIN = -(1 << 31)
TG22 = 13573
L2_BIT = 1 << 31


class CannyArgError(ValueError):
    """cv::Canny raises cv::Exception (the device API returns B200CV_ERR_BAD_ARG)"""


def wrap32(v):
    """int32 wrap-around of an integer array / scalar, as the reference's int arithmetic does on x86-64"""
    return ((np.asarray(v, np.int64) + (1 << 31)) % (1 << 32)) - (1 << 31)


def cv_floor_x86(v):
    """cvFloor(double) of the x86-64 build: (int)floor(v) through cvttsd2si -- NaN and values outside the int range give INT_MIN"""
    v = float(v)
    if not (-2147483648.0 <= v < 2147483648.0):
        return INT_MIN
    return int(math.floor(v))


def user_args(t1, t2, aperture, l2):
    """canny.cpp:838-856: the CV_CANNY_L2_GRADIENT bit, the aperture check, /16 for aperture 7, the low/high swap.
    Note that aperture -1 carries bit 31 itself, so Scharr without L2gradient is refused (the bit turns it into 0x7fffffff)."""
    ap = int(wrap32(aperture))
    l2 = bool(l2)
    if not l2 and (ap & L2_BIT) == L2_BIT:
        ap = int(wrap32((ap & 0xFFFFFFFF) & ~L2_BIT))
        l2 = True
    if (ap & 1) == 0 or (ap != -1 and (ap < 3 or ap > 7)):
        raise CannyArgError("aperture size should be odd between 3 and 7")
    lo, hi = float(t1), float(t2)
    if ap == 7:
        lo, hi = lo / 16.0, hi / 16.0
    if lo > hi:
        lo, hi = hi, lo
    return lo, hi, ap, l2


def int_thresholds(lo, hi, l2):
    """canny.cpp:884-893"""
    if l2:
        lo, hi = min(32767.0, lo), min(32767.0, hi)
        if lo > 0:
            lo *= lo
        if hi > 0:
            hi *= hi
    return cv_floor_x86(lo), cv_floor_x86(hi)


def deriv_taps(ksize):
    """(smoothing, derivative) integer taps of getDerivKernels (deriv.cpp:38-105); ksize -1 = Scharr"""
    return {-1: ([3, 10, 3], [-1, 0, 1]), 3: ([1, 2, 1], [-1, 0, 1]), 5: ([1, 4, 6, 4, 1], [-1, -2, 0, 2, 1]),
            7: ([1, 6, 15, 20, 15, 6, 1], [-1, -4, -5, 0, 5, 4, 1])}[ksize]


def _rhe_div16(s):
    """round-half-even of s / 16 for integer s (cvRound of the exact float sum * (1/16))"""
    q, r = s >> 4, s & 15
    return q + ((r > 8) | ((r == 8) & ((q & 1) == 1)))


def sobel16(img, ksize):
    """Sobel(img, CV_16S, 1, 0) and (0, 1) with BORDER_REPLICATE, scale 1/16 for ksize 7 (canny.cpp:372-379).
    img: (H, W) or (H, W, cn) uint8.  Returns dx, dy as int64 arrays of shape (H, W, cn)."""
    a = np.asarray(img)
    if a.ndim == 2:
        a = a[:, :, None]
    h, w, cn = a.shape
    sm, dk = deriv_taps(ksize)
    r = len(sm) // 2
    p = np.pad(a.astype(np.int64), ((r, r), (r, r), (0, 0)), mode="edge")
    dx = np.zeros((h, w, cn), np.int64)
    dy = np.zeros((h, w, cn), np.int64)
    for i in range(2 * r + 1):
        for j in range(2 * r + 1):
            win = p[i:i + h, j:j + w]
            if sm[i] * dk[j]:
                dx += sm[i] * dk[j] * win
            if dk[i] * sm[j]:
                dy += dk[i] * sm[j] * win
    if ksize == 7:
        dx, dy = _rhe_div16(dx), _rhe_div16(dy)
    return dx, dy


def magnitude_select(dx, dy, l2):
    """per-channel L1 / L2 magnitude in int32, then the channel with the largest one (first channel on ties, canny.cpp:486-495).
    L1 takes |-32768| = 32768, as the reference's scalar loop does; its SIMD loop (canny.cpp:456-466) gets -32768 for it, so for a
    Canny(dx, dy) input holding -32768 the reference's L1 answer depends on the pixel's position in the row.  8-bit images never get there."""
    dx = np.asarray(dx, np.int64)
    dy = np.asarray(dy, np.int64)
    if dx.ndim == 2:
        dx, dy = dx[:, :, None], dy[:, :, None]
    mag = wrap32(dx * dx + dy * dy) if l2 else np.abs(dx) + np.abs(dy)
    k = np.argmax(mag, axis=2)[:, :, None]           # argmax keeps the first maximum
    take = lambda a: np.take_along_axis(a, k, axis=2)[:, :, 0]
    return take(mag), take(dx), take(dy)


def nms_classes(mag, dx, dy, low, high):
    """non-maximum suppression (canny.cpp:596-640): 0 = not a candidate, 1 = weak, 2 = strong.  Magnitude outside the image is 0."""
    h, w = mag.shape
    P = np.zeros((h + 2, w + 2), np.int64)
    P[1:-1, 1:-1] = mag
    m = P[1:-1, 1:-1]
    left, right, up, down = P[1:-1, :-2], P[1:-1, 2:], P[:-2, 1:-1], P[2:, 1:-1]
    x = np.abs(dx)
    y = np.abs(dy) << 15
    tg22x = x * TG22
    tg67x = wrap32(tg22x + (x << 16))
    s = np.where((dx ^ dy) < 0, -1, 1)
    yy, xx = np.mgrid[0:h, 0:w]
    diag_up = P[yy, xx + 1 - s]                      # mag[up][x - s]
    diag_down = P[yy + 2, xx + 1 + s]                # mag[down][x + s]
    keep = np.where(y < tg22x, (m > left) & (m >= right),
                    np.where(y > tg67x, (m > up) & (m >= down), (m > diag_up) & (m > diag_down)))
    keep &= m > low
    return np.where(keep, np.where(m > high, 2, 1), 0).astype(np.uint8)


def hysteresis_stack(cls):
    """the reference's flood fill: push every strong pixel, pop, mark 8-neighbour candidates and push them (canny.cpp:914-927)"""
    h, w = cls.shape
    mp = np.ones((h + 2, w + 2), np.uint8)           # 1 = never an edge (border ring and non-candidates)
    inner = mp[1:-1, 1:-1]
    inner[cls == 1] = 0
    inner[cls == 2] = 2
    flat = mp.reshape(-1)
    step = w + 2
    stack = list(np.flatnonzero(flat == 2))
    offs = (-step - 1, -step, -step + 1, -1, 1, step - 1, step, step + 1)
    while stack:
        m = stack.pop()
        for o in offs:
            if flat[m + o] == 0:
                flat[m + o] = 2
                stack.append(m + o)
    return np.where(mp[1:-1, 1:-1] == 2, 255, 0).astype(np.uint8)


def hysteresis_labels(cls):
    """the same edge set through scipy's 8-connected labelling (for large frames)"""
    from scipy import ndimage
    lab, n = ndimage.label(cls > 0, structure=np.ones((3, 3), np.int32))
    good = np.zeros(n + 1, bool)
    good[np.unique(lab[cls == 2])] = True
    good[0] = False
    return np.where(good[lab], 255, 0).astype(np.uint8)


def hysteresis(cls):
    return hysteresis_stack(cls) if cls.size <= 300_000 else hysteresis_labels(cls)


def canny(img, threshold1, threshold2, aperture=3, l2=False):
    """cv::Canny(image, edges, threshold1, threshold2, apertureSize, L2gradient) on an 8-bit (H, W[, cn]) array"""
    lo, hi, ap, l2 = user_args(threshold1, threshold2, aperture, l2)
    return canny_prepared(img, lo, hi, ap, l2)


def canny_prepared(img, lo, hi, ap, l2):
    """from the arguments cv_hal_canny receives (canny.cpp:864)"""
    low, high = int_thresholds(lo, hi, l2)
    dx, dy = sobel16(img, ap)
    m, sx, sy = magnitude_select(dx, dy, l2)
    return hysteresis(nms_classes(m, sx, sy, low, high))


def canny_derivs(dx, dy, threshold1, threshold2, l2=False):
    """cv::Canny(dx, dy, edges, threshold1, threshold2, L2gradient) on int16 (H, W[, cn]) arrays (canny.cpp:933-1003)"""
    lo, hi = float(threshold1), float(threshold2)
    if lo > hi:
        lo, hi = hi, lo
    low, high = int_thresholds(lo, hi, l2)
    m, sx, sy = magnitude_select(np.asarray(dx, np.int64), np.asarray(dy, np.int64), l2)
    return hysteresis(nms_classes(m, sx, sy, low, high))


# ---- the compiled reference ---------------------------------------------------------------------------------------------------------
REF_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")


def ref_available(kind="ref"):
    return os.path.exists(os.path.join(REF_DIR, "libcannyref.so" if kind == "ref" else "libcannyref_hal.so"))


class RefCanny:
    """cv::Canny of the compiled reference: kind "ref" (its own code) or "ref_hal" (its HAL routed to b200cv_hal_canny)"""

    def __init__(self, kind="ref"):
        self.kind = kind
        self.lib = ctypes.CDLL(os.path.join(REF_DIR, "libcannyref.so" if kind == "ref" else "libcannyref_hal.so"))

    def Canny(self, img, threshold1, threshold2, aperture=3, l2=False):
        """edges, or None when the reference refuses the arguments"""
        img = np.ascontiguousarray(img)
        h, w = img.shape[:2]
        cn = 1 if img.ndim == 2 else img.shape[2]
        dst = np.zeros((h, w), np.uint8)
        rc = self.lib.ref_canny(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(img.strides[0]), w, h, cn, dst.ctypes.data_as(ctypes.c_void_p),
                                ctypes.c_size_t(dst.strides[0]), ctypes.c_double(threshold1), ctypes.c_double(threshold2), ctypes.c_int(int(wrap32(aperture))),
                                int(bool(l2)))
        assert rc in (0, -1), rc
        return dst if rc == 0 else None

    def CannyDerivs(self, dx, dy, threshold1, threshold2, l2=False):
        dx = np.ascontiguousarray(dx, np.int16)
        dy = np.ascontiguousarray(dy, np.int16)
        h, w = dx.shape[:2]
        cn = 1 if dx.ndim == 2 else dx.shape[2]
        dst = np.zeros((h, w), np.uint8)
        rc = self.lib.ref_canny_derivs(dx.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(dx.strides[0]), dy.ctypes.data_as(ctypes.c_void_p),
                                       ctypes.c_size_t(dy.strides[0]), w, h, cn, dst.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(dst.strides[0]),
                                       ctypes.c_double(threshold1), ctypes.c_double(threshold2), int(bool(l2)))
        assert rc in (0, -1), rc
        return dst if rc == 0 else None


# ---- seeded inputs shared by the golden file, its writer and the tests -----------------------------------------------------------------
def test_image(seed, h, w, cn):
    """smooth structure plus noise: blocks, ramps and a disc, so every NMS direction and both thresholds are exercised"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = 90 + 60 * np.sin(xx / (3.0 + seed % 5)) * np.cos(yy / (4.0 + seed % 3))
    base += np.where((xx // 7 + yy // 5) % 2 == 0, 40, -40)
    base += np.where((xx - w / 2) ** 2 + (yy - h / 2) ** 2 < (min(h, w) / 3) ** 2, 50, 0)
    out = np.empty((h, w, cn), np.uint8)
    for c in range(cn):
        out[:, :, c] = np.clip(base * (1 - 0.2 * c) + rng.normal(0, 12, (h, w)), 0, 255).astype(np.uint8)
    return out[:, :, 0] if cn == 1 else out
