"""The case table of warpAffine / warpPerspective shared by tests/test_warp_port.py (the C port against the reference, CPU) and
tests/test_gpu_warp_exact.py (every warp kernel against the port, GPU).  Plain data and seeded inputs: no GPU, no oracle.

Everything a result depends on is reproducible bit for bit on any machine: matrices are literals or products of literals (no
sin / cos, no matrix inverse), pixels come from numpy's PCG64 seeded by the case id.  tests/golden/warp_ref.json relies on that.

What the table aims at (opencv_b200/csrc/warp.cu):
  bw*     projective column blocks.  The reference evaluates M (x_block, y, 1) once per block line and adds M0 x1 inside the block, so
          every coordinate's rounding depends on bw0 = min(1024 / min(16, dh), dw): heights 1..17 give thirteen widths other than 64,
          most of which cut a 128-column tile and a thread's 4-pixel group; widths around 43 cross the `blocks_ok` switch.
  fp*     affine minification 1 .. 7: the staged footprint crosses 96 KB, first for the 128x32 tile, then for the 64x16 one.
  t64*    every (type, channels, LINEAR | CUBIC) instantiation of warp_tile_kernel at four maps (8-bit: forced, B200CV_WARP_PATH=tile64).
  al*     sources whose pitch is a multiple of 16 (vector loads), constant borders with equal (vector fill) and distinct values, maps
          that leave whole staged vectors outside on all four sides, destination widths 4k .. 4k+3 (32-bit stores and their tail).
  bt*     batches of three frames.
  dg*     degenerate sources and destinations, saturating coordinates, singular matrices, W == 0, INTER_AREA, BORDER_ISOLATED.
"""
import collections
import hashlib

import numpy as np

NEAREST, LINEAR, CUBIC, AREA = 0, 1, 2, 3
INVERSE = 16
CONST, REPL, REFL, WRAP, R101, ISOLATED = 0, 1, 2, 3, 4, 16
BORDERS = (CONST, REPL, REFL, WRAP, R101)
INTERPS = (NEAREST, LINEAR, CUBIC)
INAME = {NEAREST: "nn", LINEAR: "lin", CUBIC: "cub", AREA: "area"}
BNAME = {CONST: "const", REPL: "repl", REFL: "refl", WRAP: "wrap", R101: "r101"}
BV4 = (10.0, 20.0, 30.0, 40.0)
BV1 = (7.0, 7.0, 7.0, 7.0)

# op: "affine" | "perspective"; src = (h, w); dtype "u8" | "f32"; dsize = (dw, dh); M: 6 or 9 numbers, row-major; frames: 1 or a batch
Case = collections.namedtuple("Case", "id group op src dtype cn dsize M flags border bval frames")

# ---- matrices -------------------------------------------------------------------------------------------------------------------
# A homography with real perspective (W runs from 1 to 1.8 over 1100 columns), destination -> source.
H_STRONG = (0.25, 0.30, 3.0, 0.02, 1.10, 2.0, 7e-4, 3e-3, 1.0)
# Its inverse to 12 digits, written out: the form the library inverts itself (no WARP_INVERSE_MAP).
H_STRONG_FWD = (4.1160314534, -1.09484931713, -10.1583957259, -0.0699800594454, 0.932691222394, -1.65544226645,
                -0.00267128183905, -0.00203167914519, 1.01207720381)
# Block-relative evaluation differs from absolute evaluation only in the last bit of X0 + M0 x1 and W0 + M6 x1, and that reaches a
# result only where the quotient sits on a rounding tie.  H_TIES puts destination row 0 there: with g = M6, row 0 of the matrix is
# 2.5 (g, ., 1) and row 1 is 161/64 (g, ., 1), so for y = 0 the exact source point is (2.5, 2.515625) at every x: a tie of rint for
# NEAREST in X, and of rint(32 Y) = rint(80.5) for LINEAR / CUBIC in Y.  The computed quotient lands within an ulp or two of the
# tie, on the side its rounding errors choose.  Over the 1100 columns of row 0, evaluation relative to blocks of 64 and absolute
# evaluation choose differently at 288 columns for NEAREST and 209 for LINEAR; blocks of 64 and blocks of 204 (dh = 5) at 315 and
# 206 (test_warp_port.py::test_row0_of_h_ties_tells_block_widths_apart recomputes this).  Rows below 0 are ordinary.
_G = 7e-4
H_TIES = (2.5 * _G, 0.31, 2.5, 161.0 / 64.0 * _G, 1.07, 161.0 / 64.0, _G, 3e-3, 1.0)

_C4, _S4 = 0.9976, 0.0698           # about 4 degrees


def _aff(scale, tx, ty):
    return (scale * _C4, scale * _S4, tx, -(scale * _S4), scale * _C4, ty)


TYPES3 = (("u8", 1), ("u8", 3), ("f32", 1))
TYPES6 = (("u8", 1), ("u8", 3), ("u8", 4), ("f32", 1), ("f32", 3), ("f32", 4))


def _tn(dtype, cn):
    return "%sc%d" % (dtype, cn)


def _cases():
    out = []

    def add(group, name, op, src, dtype, cn, dsize, M, flags, border, bval=BV4, frames=1):
        out.append(Case("%s-%s" % (group, name), group, op, src, dtype, cn, dsize, tuple(float(v) for v in M), flags, border,
                        tuple(float(v) for v in bval), frames))

    # ---- projective column blocks: bw0 = 1024, 512, 341, 204, 146, 113, 93, 78, 68, 64, 64 at the heights below ----
    n = 0
    for dh in (1, 2, 3, 5, 7, 9, 11, 13, 15, 16, 17):
        for dw in (700, 1100):
            for it in INTERPS:
                for dtype, cn in TYPES3:
                    n += 1
                    add("bwh", "h%d-w%d-%s-%s-strong" % (dh, dw, _tn(dtype, cn), INAME[it]), "perspective", (40, 160), dtype, cn, (dw, dh),
                        H_STRONG, it | INVERSE, BORDERS[n % 5])
                    if cn == 1:
                        add("bwh", "h%d-w%d-%s-%s-ties" % (dh, dw, _tn(dtype, cn), INAME[it]), "perspective", (40, 160), dtype, cn, (dw, dh),
                            H_TIES, it | INVERSE, BORDERS[(n + 2) % 5])
                add("bwh", "h%d-w%d-u8c3-%s-forward" % (dh, dw, INAME[it]), "perspective", (40, 160), "u8", 3, (dw, dh), H_STRONG_FWD, it, REPL)
    # widths 1 .. 129 at height 40 (bw0 = dw below 64): 42 | 43 is the `blocks_ok` switch, 64 and 128 the single-tile sizes
    for dw in (1, 31, 42, 43, 63, 64, 65, 127, 128, 129):
        for it in INTERPS:
            for dtype, cn in TYPES3:
                n += 1
                add("bww", "w%d-%s-%s-strong" % (dw, _tn(dtype, cn), INAME[it]), "perspective", (40, 160), dtype, cn, (dw, 40), H_STRONG,
                    it | INVERSE, BORDERS[n % 5])
                if cn == 1:
                    add("bww", "w%d-%s-%s-ties" % (dw, _tn(dtype, cn), INAME[it]), "perspective", (40, 160), dtype, cn, (dw, 40), H_TIES,
                        it | INVERSE, BORDERS[(n + 2) % 5])
            add("bww", "w%d-u8c3-%s-forward" % (dw, INAME[it]), "perspective", (40, 160), "u8", 3, (dw, 40), H_STRONG_FWD, it, REPL)

    # ---- affine minification against the 96 KB (98304 bytes) of staged footprint ----
    # footprint(case, 128, 32) / footprint(case, 64, 16) in bytes, LINEAR (CUBIC is 1-5 % larger), and the kernel predict() names:
    #   scale      1.0            2.0            2.5             3.0             4.0             5.0              5.5              7.0
    #   8UC1   7744/2688 q   25536/7568 q   38272/11024 q   53568/15120 q   91840/24928 q  139664/37168 t  167696/44400 t  267152/69440 t
    #   8UC3  21824/7296 q   73920/21328 q 111488/31376 t  156736/43344 t  270272/72160 t  412496/108272 d 495952/129648 d 792400/203840 d
    #   8UC4  28864/9600 q   98112/28208 q 148096/41552 t  208320/57456 t  359488/95776 t  548912/143824 d        d                d
    #   32FC1     -/9600 t       -/28208 t      -/41552 t       -/57456 t       -/95776 t       -/143824 d        d                d
    #   32FC3     -/28032 t      -/83248 t      -/122960 d      d               d               d                 d                d
    #   32FC4     -/37248 t      -/110768 d     d               d               d               d                 d                d
    #   q = warp_tile4_kernel (128x32), t = warp_tile_kernel (64x16), d = warp_kernel (direct).  8UC4 CUBIC at 2.0 is 100448: already t.
    # test_gpu_warp_exact.py::test_predicted_kernel_runs checks these against the kernels that run.
    for sc in (1.0, 2.0, 2.5, 3.0, 4.0, 5.0, 5.5, 7.0):
        for dtype, cn in TYPES6:
            for it in INTERPS:
                add("fp", "x%g-%s-%s" % (sc, _tn(dtype, cn), INAME[it]), "affine", (300, 400), dtype, cn, (160, 48), _aff(sc, 3.3, 2.7),
                    it | INVERSE, R101)

    # ---- every instantiation of the 64x16 kernel at four maps ----
    maps = (("frac", (1, 0, 0.37, 0, 1, 0.61), REPL), ("rot", (0.8, 0.6, -20.0, -0.6, 0.8, 40.0), CONST),
            ("flip", (-1, 0, 149.25, 0, -1, 99.5), R101), ("shift", (1, 0, -7.53125, 0, 1, 5.28125), WRAP))
    for dtype, cn in TYPES6:
        for it in (LINEAR, CUBIC):
            for mname, M, border in maps:
                add("t64", "%s-%s-%s" % (mname, _tn(dtype, cn), INAME[it]), "affine", (100, 150), dtype, cn, (150, 70), M, it | INVERSE, border)

    # ---- alignment: 16-byte pitches, constant fill, destination widths ----
    MA = (_C4, _S4, -35.3, -_S4, _C4, -12.6)        # the 230 x 110 destination overhangs the 160 x 64 source on all four sides
    for sw in (160, 256):
        for dtype, cn in (("u8", 1), ("u8", 3), ("u8", 4), ("f32", 1)):
            for it in INTERPS:
                for bn, bv in (("same", BV1), ("distinct", BV4)):
                    add("al", "s%d-%s-%s-%s" % (sw, _tn(dtype, cn), INAME[it], bn), "affine", (64, sw), dtype, cn, (230 + (sw - 160), 110), MA,
                        it | INVERSE, CONST, bv)
    for dw in (228, 229, 231):
        for cn in (1, 3, 4):
            for it in INTERPS:
                add("al", "d%d-u8c%d-%s" % (dw, cn, INAME[it]), "affine", (64, 160), "u8", cn, (dw, 110), MA, it | INVERSE, CONST, BV4)
    for dw in (129, 130, 131, 132):                    # the same through the projective tables
        for it in INTERPS:
            add("al", "d%d-u8c3-%s-persp" % (dw, INAME[it]), "perspective", (40, 160), "u8", 3, (dw, 37), H_STRONG, it | INVERSE, CONST, BV1)

    # ---- batches of three frames ----
    for dtype, cn in TYPES3:
        for it in INTERPS:
            add("bt", "affine-%s-%s" % (_tn(dtype, cn), INAME[it]), "affine", (60, 90), dtype, cn, (150, 50), (0.8, 0.6, -20.0, -0.6, 0.8, 40.0),
                it | INVERSE, R101, frames=3)
            add("bt", "persp-%s-%s" % (_tn(dtype, cn), INAME[it]), "perspective", (40, 160), dtype, cn, (300, 13), H_STRONG, it | INVERSE, CONST,
                frames=3)

    # ---- degenerate and extreme ----
    MD = (0.31, 0.05, -2.4, -0.04, 0.29, -1.9)
    HD = (0.31, 0.05, -2.4, -0.04, 0.29, -1.9, 2e-3, -1e-3, 1.0)
    for src in ((1, 1), (1, 9), (9, 1), (2, 2), (3, 40), (40, 3)):
        for border in BORDERS:
            for it in INTERPS:
                nm = "s%dx%d-%s-%s" % (src[0], src[1], BNAME[border], INAME[it])
                add("dg", nm + "-u8c3", "affine", src, "u8", 3, (40, 24), MD, it | INVERSE, border)
                add("dg", nm + "-f32c1", "affine", src, "f32", 1, (40, 24), MD, it | INVERSE, border)
                add("dg", nm + "-u8c1-persp", "perspective", src, "u8", 1, (40, 24), HD, it | INVERSE, border)
    for it in INTERPS:
        for dtype, cn in (("u8", 1), ("u8", 3), ("f32", 3)):
            add("dg", "d1x1-affine-%s-%s" % (_tn(dtype, cn), INAME[it]), "affine", (20, 30), dtype, cn, (1, 1), (1, 0, 4.4, 0, 1, 3.3), it | INVERSE, REFL)
            add("dg", "d1x1-persp-%s-%s" % (_tn(dtype, cn), INAME[it]), "perspective", (20, 30), dtype, cn, (1, 1), H_STRONG, it | INVERSE, REFL)
    # translations far beyond the 16-bit coordinates the maps saturate to
    for tx, ty in ((33000, 0), (-33000, 0), (0, 70000), (0, -70000), (-70000, 33000)):
        for border in BORDERS:
            for it in INTERPS:
                nm = "t%d,%d-%s-%s" % (tx, ty, BNAME[border], INAME[it])
                add("dg", nm + "-u8c1", "affine", (20, 30), "u8", 1, (40, 16), (1, 0, tx + 0.25, 0, 1, ty + 0.5), it | INVERSE, border)
                if border in (CONST, WRAP):
                    add("dg", nm + "-f32c1-persp", "perspective", (20, 30), "f32", 1, (40, 16), (1, 0, tx + 0.25, 0, 1, ty + 0.5, 0, 0, 1),
                        it | INVERSE, border)
    for it in INTERPS:
        for dtype, cn in (("u8", 3), ("f32", 1)):
            t = "%s-%s" % (_tn(dtype, cn), INAME[it])
            add("dg", "x1000-inverse-" + t, "affine", (20, 30), dtype, cn, (40, 16), (1000, 0, 0, 0, 1000, 0), it | INVERSE, WRAP)
            add("dg", "x1000-forward-" + t, "affine", (20, 30), dtype, cn, (40, 16), (1000, 0, 0, 0, 1000, 0), it, REFL)
            add("dg", "singular-persp-" + t, "perspective", (20, 30), dtype, cn, (40, 16), (1, 2, 3, 2, 4, 6, 0, 0, 1), it, CONST)
            add("dg", "singular-affine-" + t, "affine", (20, 30), dtype, cn, (40, 16), (1, 2, 3, 2, 4, 6), it, CONST)
            # W = 1 - x/8 - y/4 is exactly 0 at (8, 0), (6, 1), (4, 2), (2, 3), (0, 4) and changes sign across that line
            add("dg", "w0-" + t, "perspective", (20, 30), dtype, cn, (40, 16), (1, 0, 0, 0, 1, 0, -0.125, -0.25, 1), it | INVERSE, REPL)
            add("dg", "isolated-" + t, "affine", (20, 30), dtype, cn, (40, 16), MD, it | INVERSE, R101 | ISOLATED)
            add("dg", "isolated-persp-" + t, "perspective", (20, 30), dtype, cn, (40, 16), HD, it | INVERSE, CONST | ISOLATED)
    for dtype, cn in TYPES6:
        add("dg", "area-affine-" + _tn(dtype, cn), "affine", (60, 90), dtype, cn, (150, 50), (0.8, 0.6, -20.0, -0.6, 0.8, 40.0), AREA | INVERSE, REFL)
        add("dg", "area-persp-" + _tn(dtype, cn), "perspective", (40, 160), dtype, cn, (150, 20), H_STRONG, AREA | INVERSE, REFL)
    return out


CASES = _cases()
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)


# ---- inputs -------------------------------------------------------------------------------------------------------------------
def frames_of(case):
    """the case's source frames, a list of (h, w) or (h, w, cn) arrays; float data is non-integer so that rounding shows"""
    rng = np.random.default_rng(int.from_bytes(hashlib.sha256(case.id.encode()).digest()[:8], "little"))
    h, w = case.src
    out = []
    for _ in range(case.frames):
        a = rng.integers(0, 256, (h, w) if case.cn == 1 else (h, w, case.cn), dtype=np.uint8)
        out.append(a if case.dtype == "u8" else (a.astype(np.float32) + np.float32(0.37)) * np.float32(0.731))
    return out


def remap_case(dtype, cn):
    """cv::remap with a CV_16SC2 map and no fraction map: the input and destination size of the check both suites make"""
    return Case("remap-fixed-%sc%d" % (dtype, cn), "remap", "remap", (50, 70), dtype, cn, (44, 30), (), NEAREST, 0, BV4, 1)


def fixed_maps(h=30, w=44):
    """integer source coordinates, a third of them outside a 70 x 50 source"""
    yy, xx = np.mgrid[0:h, 0:w]
    return np.stack([xx * 2 - 9 + yy % 3, yy * 3 - 7 + xx % 2], -1).astype(np.int16)


def run(oracle, case, img):
    """the case through an oracle.api.Oracle (port or reference).  The reference does not accept BORDER_ISOLATED in a warp (its
    borderInterpolate refuses the value as soon as a pixel needs the border); the library and the port ignore the bit, as the
    filters do, so the reference's answer for such a case is its answer without the bit."""
    fn = oracle.warpAffine if case.op == "affine" else oracle.warpPerspective
    border = case.border & ~ISOLATED if oracle.kind == "ref" else case.border
    return fn(img, matrix(case), case.dsize, case.flags, border, case.bval)


def matrix(case):
    return np.array(case.M, np.float64).reshape(2 if case.op == "affine" else 3, 3)


def digest(arrays):
    """SHA-256 over the bytes of the results of a case's frames (-0 folded into +0), its first 64 bits in hex"""
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(("%s%s" % (a.dtype.str, a.shape)).encode())
        h.update((a + 0 if a.dtype == np.float32 else a).tobytes())
    return h.hexdigest()[:16]


# ---- the dispatch of launch_warp_i restated: which kernel a case runs on ----------------------------------------------------------
WT_W, WT_H, WQ_W, WQ_H, WQ_NB, SMEM_MAX = 64, 16, 128, 32, 4, 96 * 1024


def inverse_matrix(case):
    """the destination -> source matrix the kernels get: cv::warpAffine / cv::warpPerspective invert M unless WARP_INVERSE_MAP is set"""
    m = list(case.M) + ([0.0, 0.0, 1.0] if case.op == "affine" else [])
    if case.flags & INVERSE:
        return m
    if case.op == "affine":
        D = m[0] * m[4] - m[1] * m[3]
        D = 1.0 / D if D != 0 else 0.0
        a11, a22 = m[4] * D, m[0] * D
        m[0], m[1], m[3], m[4] = a11, m[1] * -D, m[3] * -D, a22
        b1 = -m[0] * m[2] - m[1] * m[5]
        b2 = -m[3] * m[2] - m[4] * m[5]
        m[2], m[5] = b1, b2
        return m
    det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6])
    if det == 0:
        return [0.0] * 9
    d = 1.0 / det
    return [(m[4] * m[8] - m[5] * m[7]) * d, (m[2] * m[7] - m[1] * m[8]) * d, (m[1] * m[5] - m[2] * m[4]) * d,
            (m[5] * m[6] - m[3] * m[8]) * d, (m[0] * m[8] - m[2] * m[6]) * d, (m[2] * m[3] - m[0] * m[5]) * d,
            (m[3] * m[7] - m[4] * m[6]) * d, (m[1] * m[6] - m[0] * m[7]) * d, (m[0] * m[4] - m[1] * m[3]) * d]


def block_width(case):
    """WarpPerspectiveInvoker's column block"""
    dw, dh = case.dsize
    return min(1024 // min(16, dh), dw)


def tile_footprint(case, x0, y0, TW, TH):
    """warp.cu:tile_footprint: the host's estimate of the bytes one TW x TH tile stages; -1: do not stage"""
    M, persp = inverse_matrix(case), case.op == "perspective"
    dw, dh = case.dsize
    es = case.cn * (1 if case.dtype == "u8" else 4)
    taps = {NEAREST: 1, LINEAR: 2, CUBIC: 4, AREA: 2}[case.flags & 7]
    X, Y = [], []
    for k in range(4):
        x = float(min(x0 + TW, dw) - 1 if k & 1 else x0)
        y = float(min(y0 + TH, dh) - 1 if k & 2 else y0)
        W = M[6] * x + M[7] * y + M[8] if persp else 1.0
        if not abs(W) > 1e-12:
            return -1
        u, v = (M[0] * x + M[1] * y + M[2]) / W, (M[3] * x + M[4] * y + M[5]) / W
        if not (abs(u) < 1e6 and abs(v) < 1e6):
            return -1
        X.append(u); Y.append(v)
    bw = (int(max(X) - min(X)) + taps + 3 + 15 + 15) & ~15
    bh = int(max(Y) - min(Y)) + taps + 3
    return ((bw * es // 16) | 1) * 16 * bh


def footprint(case, TW, TH):
    """the largest estimate over the tiles launch_warp_i samples (one for an affine map, up to 9 x 9 for a projective one)"""
    dw, dh = case.dsize
    tx, ty = -(-dw // TW), -(-dh // TH)
    nsx, nsy = (min(tx, 9), min(ty, 9)) if case.op == "perspective" else (1, 1)
    need = 0
    for j in range(nsy):
        for i in range(nsx):
            bx = i * (tx - 1) // (nsx - 1) if nsx > 1 else 0
            by = j * (ty - 1) // (nsy - 1) if nsy > 1 else 0
            fp = tile_footprint(case, bx * TW, by * TH, TW, TH)
            if fp < 0:
                return -1
            need = max(need, fp)
    return need


def predict(case, path=None):
    """the kernel launch_warp_i picks for the case; path: the value of B200CV_WARP_PATH"""
    u8, it = case.dtype == "u8", case.flags & 7
    it = LINEAR if it == AREA else it
    bw0 = block_width(case)
    blocks_ok = case.op == "affine" or (WQ_W + bw0 - 1) // bw0 + 1 <= WQ_NB
    if u8 and it == NEAREST and blocks_ok and path != "direct":
        return "warp_nn4_kernel"
    need = footprint(case, WT_W, WT_H)
    if it == NEAREST or need < 0 or need > SMEM_MAX or path == "direct":
        return "warp_kernel"
    if u8 and blocks_ok and path != "tile64" and 0 < footprint(case, WQ_W, WQ_H) <= SMEM_MAX:
        return "warp_tile4_kernel"
    return "warp_tile_kernel"
