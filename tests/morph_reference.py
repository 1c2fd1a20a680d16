"""A numpy restatement of cv::erode / cv::dilate / cv::morphologyEx (morph.dispatch.cpp in the reference) for 8U, 16U, 16S and 32F images.

Each pass pads its input by the border rule (cv::borderInterpolate, or the border value for CONSTANT) and takes the min or max over the
element's offsets.  resolve() applies the argument rules of morphOp and morphologyEx:
  1. iterations == 0, or a 1x1 element (even a zero one), copies;
  2. cv::erode / cv::dilate with an empty element use a (1+2it)^2 rectangle anchored at (it, it), once; morphologyEx uses 3x3;
  3. an all-ones element with iterations > 1 grows to ksize + (it-1)(ksize-1), its anchor to anchor * it, and runs once;
  4. any other element runs max(it, 1) passes, each reading the previous pass's output;
  5. OPEN / CLOSE chain them, GRADIENT / TOPHAT / BLACKHAT subtract with saturation (a plain float subtract for 32F);
  6. the default CONSTANT value is the depth's maximum (FLT_MAX for 32F) for erode and its minimum (-FLT_MAX) for dilate; an explicit value
     is saturate_cast per channel (cvRound half to even, INT_MIN outside int32, then clamped).
excluded() marks the 32F outputs whose windows hold a NaN or a -0.0: the reference's choice there depends on the column (minps / maxps
in its vector body, std::min / std::max in its tail), so they are left out of every comparison.
"""
import sys

import numpy as np

MORPH_ERODE, MORPH_DILATE, MORPH_OPEN, MORPH_CLOSE, MORPH_GRADIENT, MORPH_TOPHAT, MORPH_BLACKHAT, MORPH_HITMISS = range(8)
BORDER_CONSTANT, BORDER_REPLICATE, BORDER_REFLECT, BORDER_WRAP, BORDER_REFLECT_101, BORDER_ISOLATED = 0, 1, 2, 3, 4, 16
DBL_MAX = sys.float_info.max
FLT_MAX = float(np.finfo(np.float32).max)
LIMITS = {np.dtype(np.uint8): (0, 255), np.dtype(np.uint16): (0, 65535), np.dtype(np.int16): (-32768, 32767)}


class Refused(Exception):
    """the reference asserts on these arguments"""


def border_interpolate(p, n, border):
    """cv::borderInterpolate; -1 for CONSTANT outside [0, n)"""
    if 0 <= p < n:
        return p
    if border == BORDER_REPLICATE:
        return 0 if p < 0 else n - 1
    if border in (BORDER_REFLECT, BORDER_REFLECT_101):
        if n == 1:
            return 0
        delta = 1 if border == BORDER_REFLECT_101 else 0
        while not 0 <= p < n:
            p = -p - 1 + delta if p < 0 else n - 1 - (p - n) - delta
        return p
    return -1


def resolve(entry, op, kernel, anchor, iterations):
    """(mask, ax, ay, passes) of each erode / dilate in the call.  entry 'erode' / 'dilate' / 'mex' (morphologyEx); kernel None or an
    empty array is the empty element"""
    empty = kernel is None or np.asarray(kernel).size == 0
    if empty and entry == "mex":
        kernel, empty = np.ones((3, 3), np.uint8), False
    m = None if empty else (np.asarray(kernel) != 0).astype(np.uint8)
    kh, kw = (3, 3) if empty else m.shape
    ax = kw // 2 if anchor[0] == -1 else anchor[0]
    ay = kh // 2 if anchor[1] == -1 else anchor[1]
    if not (0 <= ax < kw and 0 <= ay < kh):
        raise Refused("anchor outside the element")
    if iterations == 0 or (not empty and kw * kh == 1):
        return np.ones((1, 1), np.uint8), 0, 0, 1
    if empty:
        if iterations < 0:
            raise Refused("empty element with negative iterations")
        n = 1 + 2 * iterations
        return np.ones((n, n), np.uint8), iterations, iterations, 1
    if not m.any():
        raise Refused("element without a non-zero entry")
    if m.all():
        if iterations > 1:
            gw, gh = kw + (iterations - 1) * (kw - 1), kh + (iterations - 1) * (kh - 1)
            return np.ones((gh, gw), np.uint8), ax * iterations, ay * iterations, 1
        return m, ax, ay, 1
    return m, ax, ay, max(iterations, 1)


def cv_round(v):
    r = np.rint(v)
    return int(r) if -2147483648.0 <= r <= 2147483647.0 else -2147483648


def border_values(dtype, cn, is_max, border_value):
    """the CONSTANT value of each channel, in the image's dtype"""
    dtype = np.dtype(dtype)
    if border_value is None or all(v == DBL_MAX for v in border_value):
        if dtype == np.float32:
            v = -FLT_MAX if is_max else FLT_MAX
        else:
            lo, hi = LIMITS[dtype]
            v = lo if is_max else hi
        return np.full(cn, v, dtype)
    if dtype == np.float32:
        with np.errstate(over="ignore"):
            return np.array([np.float32(border_value[c]) for c in range(cn)], np.float32)
    lo, hi = LIMITS[dtype]
    return np.array([min(max(cv_round(border_value[c]), lo), hi) for c in range(cn)], dtype)


def morph_once(img, mask, ax, ay, reduce, border, bv):
    """one pass over (H, W, C): min / max (reduce) over the element's offsets of the padded image"""
    H, W, C = img.shape
    kh, kw = mask.shape
    border &= ~BORDER_ISOLATED
    ry = [border_interpolate(y, H, border) for y in range(-ay, H + kh - 1 - ay)]
    rx = [border_interpolate(x, W, border) for x in range(-ax, W + kw - 1 - ax)]
    iy, ix = np.array(ry), np.array(rx)
    pad = np.empty((len(ry), len(rx), C), img.dtype)
    pad[...] = bv
    vy, vx = iy >= 0, ix >= 0
    pad[np.ix_(vy, vx)] = img[np.ix_(iy[vy], ix[vx])]
    if mask.all():                         # a rectangle: rows, then columns (the same min / max, fewer operations)
        rows = pad[:, 0:W]
        for j in range(1, kw):
            rows = reduce(rows, pad[:, j:j + W])
        out = rows[0:H]
        for i in range(1, kh):
            out = reduce(out, rows[i:i + H])
        return np.ascontiguousarray(out)
    out = None
    for i, j in zip(*np.nonzero(mask)):
        v = pad[i:i + H, j:j + W]
        out = v.copy() if out is None else reduce(out, v)
    return out


def saturating_sub(a, b):
    if a.dtype == np.float32:
        with np.errstate(invalid="ignore"):          # inf - inf is NaN, as in the reference
            return a - b
    lo, hi = LIMITS[a.dtype]
    return np.clip(a.astype(np.int64) - b.astype(np.int64), lo, hi).astype(a.dtype)


def _apply(img, entry, op, kernel, anchor, iterations, border, border_value, indicator):
    mask, ax, ay, passes = resolve(entry, op, kernel, anchor, iterations)
    C = img.shape[2]

    def chain(x, is_max):
        if indicator:
            bv, red = np.zeros(C, np.uint8), np.maximum
        else:
            bv, red = border_values(img.dtype, C, is_max, border_value), (np.maximum if is_max else np.minimum)
        for _ in range(passes):
            x = morph_once(x, mask, ax, ay, red, border, bv)
        return x

    sub = (lambda a, b: a | b) if indicator else saturating_sub
    if op == MORPH_ERODE:
        return chain(img, False)
    if op == MORPH_DILATE:
        return chain(img, True)
    if op == MORPH_OPEN:
        return chain(chain(img, False), True)
    if op == MORPH_CLOSE:
        return chain(chain(img, True), False)
    if op == MORPH_GRADIENT:
        return sub(chain(img, True), chain(img, False))
    if op == MORPH_TOPHAT:
        return sub(img, chain(chain(img, False), True))
    if op == MORPH_BLACKHAT:
        return sub(chain(chain(img, True), False), img)
    raise Refused("unknown operation")


def _hwc(img):
    return img[:, :, None] if img.ndim == 2 else img


def morphology(img, entry, op, kernel=None, anchor=(-1, -1), iterations=1, border=BORDER_CONSTANT, border_value=None):
    """the reference's answer, with the shape of img; raises Refused where the reference asserts"""
    return _apply(_hwc(img), entry, op, kernel, anchor, iterations, border, border_value, False).reshape(img.shape)


def excluded(img, entry, op, kernel=None, anchor=(-1, -1), iterations=1, border=BORDER_CONSTANT, border_value=None):
    """bool mask of the outputs that depend on a NaN or a -0.0 of a 32F source (all False for other depths)"""
    if img.dtype != np.float32:
        return np.zeros(img.shape, bool)
    special = (np.isnan(img) | ((img == 0) & np.signbit(img))).astype(np.uint8)
    return _apply(_hwc(special), entry, op, kernel, anchor, iterations, border, border_value, True).reshape(img.shape) != 0

