"""One table of cv::erode / cv::dilate / cv::morphologyEx cases, aimed at the reference's argument rules (tests/morph_reference.py) and
at the places where the device's kernels change (opencv_b200/csrc/morph.cu):

  rules     copies (iterations 0, 1x1 elements, a zero 1x1), the two empty-element rules, grown rectangles (rule 3, anchors scaled),
            repeated passes of other elements (and negative iterations: one pass), every compound op, default and explicit border values
            (saturating ones among them), 32F images with +-inf (and all +inf), NaN and -0.0 (the latter two left out of the comparison)
  kernels   rectangles on both sides of the fused / van Herk switch (32 on each axis), for erode / dilate and every compound op, crosses, ellipses and random masks up to the 63x63
            cap, anchors at every corner, elements wider or taller than the image, 1 to 4 channels at every depth
  sizes     1x1 up to 2160x3840, one very wide (1 x 20000) and one very tall (20000 x 1)
  refusals  the reference's assertions (anchor outside, negative iterations with an empty element, an element with no non-zero entry);
            the device's own refusals (HITMISS, 64F, WRAP, larger non-rectangular elements) are in tests/test_gpu_morphology.py

Every case is plain data; its pixels come from PCG64 seeded by the SHA-256 of its image id, so every machine builds the same bytes.
The reference's answers come from oracle/_ref/libmorphref.so (tests/cpp/morph_ref_shim.cpp, built by tools/build_morph_ref.py).
"""
import ctypes
import hashlib
import os
from collections import namedtuple

import numpy as np

import morph_reference as mr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libmorphref.so")
DTYPES = {"8U": np.uint8, "16U": np.uint16, "16S": np.int16, "32F": np.float32}
CV_DEPTH = {"8U": 0, "16U": 2, "16S": 3, "32F": 5}

# a call: (entry, op, element, anchor, iterations, border, border value); element: None (empty) or (shape, w, h[, seed])
Call = namedtuple("Call", "entry op elem anchor it border bv")
Case = namedtuple("Case", "id image shape depth cn fill calls")       # calls: {name: Call}

E, D, X = "erode", "dilate", "mex"
C0, REP, REF, R101, ISO = 0, 1, 2, 4, 16


def element(spec):
    """the element's byte mask, or None for the empty element"""
    if spec is None:
        return None
    kind, w, h = spec[:3]
    if kind == "rect":
        return np.ones((h, w), np.uint8)
    if kind == "zero":
        return np.zeros((h, w), np.uint8)
    if kind == "far":                # only the last entry: with anchor (0, 0) the window leaves the image before the row ends
        m = np.zeros((h, w), np.uint8)
        m[-1, -1] = 1
        return m
    if kind in ("cross", "ellipse"):
        import opencv_b200
        return opencv_b200.getStructuringElement({"cross": 1, "ellipse": 2}[kind], (w, h))
    if kind == "random":             # a random mask with at least one non-zero entry
        g = np.random.Generator(np.random.PCG64(spec[3]))
        m = (g.random((h, w)) < 0.45).astype(np.uint8)
        m[g.integers(0, h), g.integers(0, w)] = 1
        if m.all():
            m[0, 0] = 0
        return m
    raise ValueError(kind)


def _basic_calls():
    """the calls every image of the sweep gets: both entry points, every compound op, rectangles on both sides of the switch"""
    return {
        "e3": Call(E, 0, ("rect", 3, 3), (-1, -1), 1, C0, None),
        "d3rep": Call(D, 1, ("rect", 3, 3), (-1, -1), 1, REP, None),
        "e5ell101": Call(E, 0, ("ellipse", 5, 5), (-1, -1), 1, R101, None),
        "d15": Call(D, 1, ("rect", 15, 15), (-1, -1), 1, REF, None),
        "e33x5": Call(E, 0, ("rect", 33, 5), (-1, -1), 1, C0, None),
        "open5ell": Call(X, 2, ("ellipse", 5, 5), (-1, -1), 1, C0, None),
        "close3x2": Call(X, 3, ("cross", 3, 3), (-1, -1), 2, REP, None),
        "grad3": Call(X, 4, ("rect", 3, 3), (-1, -1), 1, C0, None),
        "top7": Call(X, 5, ("ellipse", 7, 7), (-1, -1), 1, R101, None),
        "black3x3it": Call(X, 6, ("rect", 3, 3), (-1, -1), 3, C0, None),
    }


def _rule_calls():
    """one or more rows for each argument rule and kernel switch, on small images"""
    c = {}
    c["it0"] = Call(E, 0, ("ellipse", 5, 5), (-1, -1), 0, C0, None)
    c["one"] = Call(D, 1, ("rect", 1, 1), (-1, -1), 5, C0, None)
    c["zero1x1"] = Call(E, 0, ("zero", 1, 1), (-1, -1), 1, C0, None)
    c["grad_it0"] = Call(X, 4, ("rect", 3, 3), (-1, -1), 0, C0, None)
    c["empty_e1"] = Call(E, 0, None, (-1, -1), 1, C0, None)
    c["empty_d3"] = Call(D, 1, None, (2, 0), 3, REP, None)        # the anchor is checked against 3x3, then replaced by (it, it)
    c["empty_mex_e2"] = Call(X, 0, None, (0, 2), 2, REF, None)   # morphologyEx: 3x3 grown by rule 3 with anchor (0, 4)
    c["empty_mex_neg"] = Call(X, 1, None, (-1, -1), -2, C0, None)
    c["rect_it3_corner"] = Call(E, 0, ("rect", 3, 4), (2, 3), 3, C0, None)
    c["rect_it4_tl"] = Call(D, 1, ("rect", 5, 3), (0, 0), 4, R101, None)
    c["rect_it10"] = Call(E, 0, ("rect", 3, 3), (-1, -1), 10, REP, None)
    c["rect_neg"] = Call(D, 1, ("rect", 3, 3), (-1, -1), -3, C0, None)
    c["cross_it3"] = Call(E, 0, ("cross", 5, 5), (-1, -1), 3, C0, None)
    c["ell_it2_br"] = Call(D, 1, ("ellipse", 7, 5), (6, 4), 2, REF, None)
    c["rand_neg"] = Call(E, 0, ("random", 6, 4, 1), (-1, -1), -1, C0, None)
    c["open_rand_it2"] = Call(X, 2, ("random", 5, 7, 2), (1, 5), 2, R101, None)
    c["close_ell_it2"] = Call(X, 3, ("ellipse", 9, 9), (-1, -1), 2, C0, None)
    c["grad_ell"] = Call(X, 4, ("ellipse", 5, 5), (-1, -1), 1, REP, None)
    c["top_rect_it3"] = Call(X, 5, ("rect", 3, 3), (-1, -1), 3, REF | ISO, None)
    c["black_cross"] = Call(X, 6, ("cross", 5, 3), (0, 1), 1, C0, None)
    c["grad_far"] = Call(X, 4, ("far", 40, 1), (0, 0), 1, C0, None)      # dilate 0 - erode MAX on the right: the subtraction saturates
    c["e32"] = Call(E, 0, ("rect", 32, 32), (-1, -1), 1, C0, None)
    c["d33"] = Call(D, 1, ("rect", 33, 33), (-1, -1), 1, REP, None)
    c["e32x33"] = Call(E, 0, ("rect", 32, 33), (31, 0), 1, R101, None)
    c["d1x100"] = Call(D, 1, ("rect", 1, 100), (0, 99), 1, C0, None)
    c["e101x1"] = Call(E, 0, ("rect", 101, 1), (100, 0), 1, REF, None)
    c["ell31"] = Call(E, 0, ("ellipse", 31, 31), (-1, -1), 1, C0, None)
    c["ell63"] = Call(D, 1, ("ellipse", 63, 63), (-1, -1), 1, REP, None)
    c["rand63x9"] = Call(E, 0, ("random", 63, 9, 3), (62, 8), 1, C0, None)
    c["rand9x63"] = Call(D, 1, ("random", 9, 63, 4), (0, 0), 1, R101, None)
    c["cross63"] = Call(E, 0, ("cross", 63, 63), (0, 62), 1, REF, None)
    c["bv_e"] = Call(E, 0, ("rect", 3, 3), (-1, -1), 1, C0, (300.0, -5.0, 70000.5, 2.5))
    c["bv_d"] = Call(D, 1, ("ellipse", 5, 5), (-1, -1), 1, C0, (-1e10, 1e10, 40000.0, -40000.0))
    c["bv_dflt_mixed"] = Call(E, 0, ("rect", 3, 3), (-1, -1), 1, C0, (mr.DBL_MAX, mr.DBL_MAX, mr.DBL_MAX, 0.0))
    c["bv_e_iso"] = Call(E, 0, ("cross", 3, 3), (-1, -1), 1, C0 | ISO, (3.5, 1e300, -7.25, 0.0))
    c["bad_anchor"] = Call(E, 0, ("rect", 3, 3), (3, 0), 1, C0, None)
    c["bad_anchor_empty"] = Call(D, 1, None, (3, 3), 2, C0, None)
    c["bad_anchor_neg"] = Call(X, 2, ("rect", 3, 3), (-2, 1), 1, C0, None)
    c["bad_empty_neg"] = Call(E, 0, None, (-1, -1), -1, C0, None)
    return c


def _van_herk_calls():
    """compound ops whose rectangles run the two-launch van Herk path: the fused subtraction in both operand orders (saturating where
    an explicit border value pushes open above src or close below it), and OPEN / CLOSE chaining two van Herk passes"""
    return {
        "vh_top41": Call(X, 5, ("rect", 41, 41), (-1, -1), 1, C0, None),
        "vh_top41_bv": Call(X, 5, ("rect", 41, 41), (-1, -1), 1, C0, (1e6, 1e6, 1e6, 1e6)),
        "vh_black3x40": Call(X, 6, ("rect", 3, 40), (-1, -1), 1, REP, None),
        "vh_black40x3_bv": Call(X, 6, ("rect", 40, 3), (0, 2), 1, C0, (-1e6, -1e6, -1e6, -1e6)),
        "vh_grad_it20": Call(X, 4, ("rect", 3, 3), (-1, -1), 20, R101, None),
        "vh_open33": Call(X, 2, ("rect", 33, 33), (-1, -1), 1, REF, None),
        "vh_close33": Call(X, 3, ("rect", 33, 33), (32, 0), 1, C0, None),
    }


BASIC = _basic_calls()
RULES = _rule_calls()
VAN_HERK = _van_herk_calls()
# the reference indexes an empty coordinate list for these (no defined answer): refused by the restatement, never run on the reference
UNDEFINED = {"zero3x3": Call(E, 0, ("zero", 3, 3), (-1, -1), 1, C0, None), "zero5x1_open": Call(X, 2, ("zero", 5, 1), (-1, -1), 1, C0, None)}
ALL_CALLS = dict(BASIC, **RULES, **VAN_HERK)


def _cases():
    out = []

    def add(shape, depth, cn, fill, calls):
        img = "%dx%d-%s-c%d-%s" % (shape[0], shape[1], depth, cn, fill)
        out.append(Case(img, img, shape, depth, cn, fill, calls))

    sweep = {k: BASIC[k] for k in BASIC}
    for depth in DTYPES:
        for cn in (1, 2, 3, 4):
            add((37, 45), depth, cn, "random", sweep)
            add((29, 70), depth, cn, "random", dict(RULES))
    for depth in DTYPES:
        for shape in [(1, 1), (1, 9), (9, 1), (2, 3), (7, 5)]:
            add(shape, depth, 1, "random", sweep)
        add((40, 131), depth, 3, "blobs", sweep)
    add((61, 77), "32F", 1, "inf", dict(sweep, **{k: RULES[k] for k in ("bv_e", "bv_d", "ell31", "d33", "rect_it10")}))
    add((9, 13), "32F", 1, "allinf", sweep)                                # erode's default border: FLT_MAX, not +inf
    add((61, 77), "32F", 2, "special", dict(sweep, **{k: RULES[k] for k in ("ell31", "open_rand_it2", "close_ell_it2", "d33")}))
    add((1, 20000), "8U", 1, "random", {k: BASIC[k] for k in ("e3", "d15", "e33x5", "grad3")})
    add((20000, 1), "16U", 1, "random", {k: BASIC[k] for k in ("e3", "d15", "top7")})
    add((70, 96), "8U", 1, "blobs", VAN_HERK)
    add((70, 96), "16U", 2, "random", VAN_HERK)
    add((70, 96), "16S", 3, "random", VAN_HERK)
    add((70, 96), "32F", 1, "inf", VAN_HERK)
    add((2160, 3840), "8U", 1, "blobs", {"e3": BASIC["e3"], "grad3": BASIC["grad3"], "e5ell101": BASIC["e5ell101"],
                                          "rect_it10": RULES["rect_it10"]})
    add((2160, 3840), "32F", 1, "random", {"d3rep": BASIC["d3rep"], "open5ell": BASIC["open5ell"]})
    return out


def rng_of(image_id):
    return np.random.Generator(np.random.PCG64(int.from_bytes(hashlib.sha256(image_id.encode()).digest()[:8], "little")))


def image_of(case):
    """the case's source, (H, W) for one channel and (H, W, C) otherwise"""
    H, W = case.shape
    shape = (H, W) if case.cn == 1 else (H, W, case.cn)
    g = rng_of(case.image)
    dt = np.dtype(DTYPES[case.depth])
    if dt == np.float32:
        img = (g.standard_normal(shape) * 1000).astype(np.float32)
    else:
        info = np.iinfo(dt)
        img = g.integers(info.min, int(info.max) + 1, shape, dtype=dt)
    if case.fill == "blobs":       # binary-looking content: a thresholded smooth field, as morphology usually sees
        coarse = g.random((H // 16 + 2, W // 16 + 2))
        field = np.kron(coarse, np.ones((16, 16)))[:H, :W]
        on = field > 0.5
        hi = 1.0 if dt == np.float32 else np.iinfo(dt).max
        img = np.where(on if case.cn == 1 else on[:, :, None], np.array(hi, dt), img // 4 if dt != np.float32 else img / 4).astype(dt)
    elif case.fill == "allinf":
        img[...] = np.inf
    elif case.fill == "inf":
        img[g.random(shape) < 0.02] = np.inf
        img[g.random(shape) < 0.02] = -np.inf
        img[g.random(shape) < 0.02] = np.finfo(np.float32).max
    elif case.fill == "special":
        img[g.random(shape) < 0.01] = np.nan
        img[g.random(shape) < 0.01] = -0.0
        img[g.random(shape) < 0.01] = 0.0
        img[g.random(shape) < 0.01] = np.inf
    return img


CASES = _cases()
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)


def restated(img, call):
    """(result, excluded) from tests/morph_reference.py; raises morph_reference.Refused"""
    args = (call.entry, call.op, element(call.elem), call.anchor, call.it, call.border, call.bv)
    return mr.morphology(img, *args), mr.excluded(img, *args)


_fn = {}


def ref_available():
    return os.path.exists(REF_LIB)


def _lib():
    if "m" not in _fn:
        L = ctypes.CDLL(REF_LIB)
        L.ref_morphology.restype = ctypes.c_int
        L.ref_morphology.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_double)]
        L.ref_structuring_element.restype = ctypes.c_int
        L.ref_structuring_element.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p]
        _fn["m"] = L
    return _fn["m"]


def reference(img, depth, call):
    """the reference's answer with the shape of img, or None where it refused"""
    img = np.ascontiguousarray(img)
    H, W = img.shape[:2]
    cn = 1 if img.ndim == 2 else img.shape[2]
    out = np.zeros_like(img)
    k = element(call.elem)
    kw, kh = (0, 0) if k is None else (k.shape[1], k.shape[0])
    kb = None if k is None else np.ascontiguousarray(k)
    bv = (ctypes.c_double * 4)(*(call.bv if call.bv is not None else (mr.DBL_MAX,) * 4))
    rc = _lib().ref_morphology(CV_DEPTH[depth] + ((cn - 1) << 3), img.ctypes.data, img.strides[0], out.ctypes.data, out.strides[0], W, H,
                               0 if call.entry in (E, D) else 1, call.op, None if kb is None else kb.ctypes.data, kw, kh,
                               call.anchor[0], call.anchor[1], call.it, call.border, bv)
    return out if rc == 0 else None


def ref_structuring_element(shape, w, h, anchor=(-1, -1)):
    out = np.zeros((h, w), np.uint8)
    rc = _lib().ref_structuring_element(shape, w, h, anchor[0], anchor[1], out.ctypes.data)
    return out if rc == 0 else None


def digest(result, excl):
    """SHA-256 of the result with the excluded elements zeroed; "refused" for None"""
    if result is None:
        return "refused"
    r = np.ascontiguousarray(result).copy()
    r[excl] = 0
    return hashlib.sha256(r.tobytes()).hexdigest()


# getStructuringElement rows: (shape, w, h, anchor)
STRUCTURING = [(s, w, h, (-1, -1)) for s in (0, 1, 2) for w in range(1, 16) for h in range(1, 16)] + \
    [(s, w, h, (-1, -1)) for s in (1, 2) for w, h in ((31, 31), (63, 63), (63, 9), (20, 64), (101, 37))] + \
    [(1, 7, 5, (0, 0)), (1, 7, 5, (6, 4)), (2, 7, 5, (6, 4)), (1, 5, 5, (5, 0)), (2, 4, 4, (-2, 1))]
