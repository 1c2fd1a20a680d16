"""The case table of cv::resize shared by tests/test_resize_port.py (the C port against the reference, CPU) and
tests/test_gpu_resize_exact_edges.py (every resize kernel against the port, GPU).  Plain data and seeded inputs: no GPU, no oracle.

Everything a result depends on is reproducible bit for bit on any machine: sizes and factors are literals, pixels come from numpy's
PCG64 seeded by the case id.  tests/golden/resize_ref.json relies on that.

What the table aims at (opencv_b200/csrc/resize*.cu; predict() restates the dispatch of resize_impl, launch_rs and launch_lanczos_sep):
  sx   resize_sep_u8_kernel's tile columns: destination widths DW k - 1, DW k, DW k + 1 (DW = 256 LINEAR, 128 CUBIC), enlargements that
       end in `last_col` columns, source widths that put a column's words exactly on the row end of the H pass's fast path
       (A + NT CN + 7 == row_bytes) or one step past it, every residue of dw cn mod 8 for the CUBIC body / tail switch, on random
       data and on rounding ties.
  sy   its row blocks: vertical factors at which launch_rs picks each of DH = 64 .. 4, the last factor at which DH = 4 fits and the
       first at which nothing does (the per-pixel fallback), destination heights DH k +- 1.
  pp   the per-pixel LINEAR / CUBIC kernels: the six 8-bit instantiations through the fallback (word loads on and off, `last_col`,
       ragged 8-row blocks, the CUBIC vec_limit tail), the six float ones at every residue of dw cn mod 4.
  am   INTER_AREA with an enlarging axis (bilinear with area-mode weights), tiled and through the fallback.
  nn   NEAREST: resize_nn_kernel<1, 3, 4, 12, 16> with 32-bit stores on and off, the walking kernel's 32-row blocks, coordinates
       within an ulp of an integer.
  a2   the exact 2x2 kernels (8-bit: 32-bit loads / stores on and off; float: the SIMD body's (a+b)+(c+d) against the scalar
       ((a+b)+c)+d on data of mixed magnitudes), reached through LINEAR, AREA and LINEAR_EXACT.
  ai   integer-factor INTER_AREA: windows of area % 4 = 0 .. 3 (the float sums' groups of four), an 8-bit window sum above 2^24.
  ag   fractional INTER_AREA: partial pixels just under and over the 1e-3 threshold, a last cell shorter than the scale by an ulp,
       1 x 1 and 1 x N destinations.
  ex   NEAREST_EXACT at every pixel size, LINEAR_EXACT's three tap kinds and 1- and 2-pixel sources, a 32767-column source.
  lz   LANCZOS4: each DH of the tiled 8-bit kernel and the first factor that falls back, 64-column tile edges, float body / tail,
       checkerboards that saturate both ways.
  fx   explicit scales (cv::resize(src, dst, Size(), fx, fy)): the sampling scale is fx, fy, not dsize / ssize.
  bt   batches of three frames, one per kernel family.
  dg   degenerate sizes: 1 x 1, one row, one column, equal sizes (a copy), a 65535-row source.
  nf   float data with +-inf, NaN, -0.0, subnormals and +-3e38 beside small values.
REFUSALS lists the calls the library declines (NOT_IMPLEMENTED, destination untouched).
"""
import collections
import hashlib
import math

import numpy as np

NEAREST, LINEAR, CUBIC, AREA, LANCZOS4, LINEAR_EXACT, NEAREST_EXACT = 0, 1, 2, 3, 4, 5, 6
INAME = {NEAREST: "nn", LINEAR: "lin", CUBIC: "cub", AREA: "area", LANCZOS4: "lz4", LINEAR_EXACT: "linx", NEAREST_EXACT: "nnx"}
TYPES6 = (("u8", 1), ("u8", 3), ("u8", 4), ("f32", 1), ("f32", 3), ("f32", 4))

# src = (h, w); dsize = (dw, dh); fxfy: None or (fx, fy) -- then dsize is (round(w fx), round(h fy)); data: how pixels are drawn
Case = collections.namedtuple("Case", "id group src dtype cn dsize interp fxfy frames data")


def _tn(dtype, cn):
    return "%sc%d" % (dtype, cn)


def _cases():
    out = []

    def add(group, name, src, dtype, cn, dsize, interp, fxfy=None, frames=1, data="rand"):
        if fxfy is not None:
            dsize = (int(round(src[1] * fxfy[0])), int(round(src[0] * fxfy[1])))      # saturate_cast<int>: half to even, like round()
        out.append(Case("%s-%s" % (group, name), group, tuple(src), dtype, cn, tuple(dsize), interp, fxfy, frames, data))

    LC = (LINEAR, CUBIC)

    # ---- sx: tile columns of resize_sep_u8_kernel (DW = 256 LINEAR, 128 CUBIC) ----
    for it in LC:
        DW = 256 if it == LINEAR else 128
        for cn in (1, 3, 4):
            for dw in (5, DW - 1, DW, DW + 1, 2 * DW - 1, 2 * DW, 2 * DW + 1):
                add("sx", "w%d-u8c%d-%s" % (dw, cn, INAME[it]), (20, 300), "u8", cn, (dw, 17), it)
            add("sx", "last-u8c%d-%s" % (cn, INAME[it]), (21, 50), "u8", cn, (173, 30), it)      # enlarging: the last columns are `last_col`
    # H pass fast / edge switch: margin = A + NT CN + 7 - row_bytes of a column whose taps are interior.  Margins are congruent mod CN,
    # so the closest a fast column can come to the row end is m0 = 0 (CN 1), -2 (CN 3), -1 (CN 4).  "on": some column has margin m0
    # (fast, its last word the row's last); "past": some column has m0 + CN (edge path) and none m0.  Found by hpass_margins() below.
    for it, cn, on, past in ((LINEAR, 1, 26, 30), (LINEAR, 3, 26, 30), (LINEAR, 4, 30, 26), (CUBIC, 1, 30, 26), (CUBIC, 3, 26, 32), (CUBIC, 4, 26, 30)):
        add("sx", "edge-on-u8c%d-%s" % (cn, INAME[it]), (19, 40), "u8", cn, (on, 23), it)
        add("sx", "edge-past-u8c%d-%s" % (cn, INAME[it]), (19, 40), "u8", cn, (past, 23), it)
    for cn in (1, 3):                                  # CUBIC vec_limit = floor8(dw cn): every residue of dw cn mod 8
        for dw in range(200, 208):
            add("sx", "res%d-w%d-u8c%d-cub" % (dw * cn % 8, dw, cn), (22, 150), "u8", cn, (dw, 19), CUBIC)
    # the same residues on rounding ties, where the body (float, half to even) and the tail ((sum + 2^21) >> 22, half up) disagree:
    # columns 2:1 (tap fraction 0.5: -192, 1216, 1216, -192), rows 1:1 (fraction 0: 0, 2048, 0, 0), even source columns v = 1 mod 4 and
    # odd ones 0, so every result is exactly v / 2 with an even integer part
    for cn in (1, 3):
        for dw in range(200, 208):
            add("sx", "tie%d-w%d-u8c%d-cub" % (dw * cn % 8, dw, cn), (9, 2 * dw), "u8", cn, (dw, 9), CUBIC, data="ties")

    # ---- sy: row blocks.  dh = 97; the smallest source height at which launch_rs picks each DH, the last with DH = 4, the first with
    # none (per-pixel fallback) -- found by scanning sh with predict() (test_resize_port.py::test_row_block_edges recomputes them) ----
    SY = {(1, LINEAR): (20, 113, 152, 236, 318, 494, 1070, 2491), (1, CUBIC): (20, 111, 148, 230, 310, 479, 1040, 2427),
          (3, LINEAR): (20, 36, 50, 73, 100, 156, 334, 777), (3, CUBIC): (20, 35, 48, 67, 89, 144, 306, 712),
          (4, LINEAR): (20, 27, 36, 55, 73, 112, 237, 551), (4, CUBIC): (20, 26, 34, 49, 65, 100, 209, 487)}
    for (cn, it), shs in SY.items():
        for DH, sh in zip((64, 48, 32, 24, 16, 8, 4), shs):
            add("sy", "dh%d-sh%d-u8c%d-%s" % (DH, sh, cn, INAME[it]), (sh, 40), "u8", cn, (37, 97), it)
        add("sy", "last4-sh%d-u8c%d-%s" % (shs[-1], cn, INAME[it]), (shs[-1], 40), "u8", cn, (37, 97), it)
        add("sy", "fallback-sh%d-u8c%d-%s" % (shs[-1] + 1, cn, INAME[it]), (shs[-1] + 1, 40), "u8", cn, (37, 97), it)
    for dh in (127, 128, 129):                          # DH = 64 blocks (enlarging), destination heights 2 DH - 1 .. 2 DH + 1
        add("sy", "dh64-h%d-u8c1-lin" % dh, (30, 33), "u8", 1, (41, dh), LINEAR)
        add("sy", "dh64-h%d-u8c3-cub" % dh, (30, 33), "u8", 3, (41, dh), CUBIC)
    for dh in (31, 32, 33):                             # DH = 16 (8UC1 LINEAR, factor 4) and 8 (8UC3 CUBIC, factor 3): 2 and 4 blocks +- 1 row
        add("sy", "dh16-h%d-u8c1-lin" % dh, (4 * dh, 33), "u8", 1, (41, dh), LINEAR)
        add("sy", "dh8-h%d-u8c3-cub" % dh, (3 * dh, 33), "u8", 3, (41, dh), CUBIC)

    # ---- pp: the per-pixel kernels.  8-bit: dh = 13 (one full and one ragged 8-row block) at a factor past the fallback edge;
    # sw = 64 (4-byte rows: word loads) and 63 (cn 1, 3: byte loads), dw = 150 (enlarging: `last_col`) and 45 (dw cn mod 8 = 5, 7, 4) ----
    for cn, fsh in ((1, 28), (3, 9), (4, 7)):
        for it in LC:
            for sw in (64, 63):
                for dw in (150, 45):
                    add("pp", "sw%d-w%d-u8c%d-%s" % (sw, dw, cn, INAME[it]), (13 * fsh, sw), "u8", cn, (dw, 13), it)
    for cn in (1, 3, 4):                                # float: every residue of dw cn mod 4 (cn 4: always 0)
        for it in LC:
            for dw in ((40, 41, 42, 43) if cn != 4 else (41,)):
                add("pp", "w%d-f32c%d-%s" % (dw, cn, INAME[it]), (31, 29), "f32", cn, (dw, 45), it, data="mixed")
                add("pp", "shrink-w%d-f32c%d-%s" % (dw, cn, INAME[it]), (61, 97), "f32", cn, (dw, 21), it)

    # ---- am: INTER_AREA with an enlarging axis ----
    for dtype, cn in (("u8", 3), ("f32", 3), ("u8", 1), ("f32", 4)):
        add("am", "xup-%s" % _tn(dtype, cn), (60, 30), dtype, cn, (70, 25), AREA)
        add("am", "yup-%s" % _tn(dtype, cn), (30, 60), dtype, cn, (25, 70), AREA)
    add("am", "xup-ydown30-u8c3", (900, 20), "u8", 3, (50, 30), AREA)           # y factor 30: no DH fits, the per-pixel kernel
    add("am", "xup-ydown40-u8c1", (1600, 20), "u8", 1, (50, 40), AREA)

    # ---- nn: NEAREST ----
    for dtype, cn in (("u8", 1), ("u8", 3), ("u8", 4), ("f32", 3), ("f32", 4)):
        for dw in (40, 41, 42, 43):
            add("nn", "w%d-%s" % (dw, _tn(dtype, cn)), (50, 61), dtype, cn, (dw, 30), NEAREST)
    for cn in (1, 3, 4):                               # the walking kernel: 32-row blocks; rows repeated 2x, 3x, 64/45x
        for dh in (63, 64, 65):
            for rep, sh in (("x2", (dh + 1) // 2), ("x3", (dh + 2) // 3), ("x1.4", dh * 45 // 64)):
                add("nn", "walk-h%d-%s-u8c%d" % (dh, rep, cn), (sh, 37), "u8", cn, (40, dh), NEAREST)
    # sw = 4 -> dw = 196: x (1 / 49) lies within an ulp of 1, 2, 3 at x = 49, 98, 147 without being exact (found by an fp64 search)
    for dtype, cn in (("u8", 3), ("f32", 1)):
        add("nn", "ulp-%s" % _tn(dtype, cn), (4, 4), dtype, cn, (196, 196), NEAREST)
        add("nn", "ulp-down-%s" % _tn(dtype, cn), (196, 196), dtype, cn, (4, 4), NEAREST)

    # ---- a2: exact 2 x 2 ----
    for cn in (1, 3, 4):
        for dw in (40, 41, 42, 43):
            add("a2", "w%d-u8c%d" % (dw, cn), (2 * 11, 2 * dw), "u8", cn, (dw, 11), AREA)
            add("a2", "w%d-f32c%d" % (dw, cn), (2 * 11, 2 * dw), "f32", cn, (dw, 11), AREA, data="mixed")
    for it in (LINEAR, AREA, LINEAR_EXACT):
        add("a2", "route-%s-u8c3" % INAME[it], (30, 82), "u8", 3, (41, 15), it)
        add("a2", "route-%s-f32c1" % INAME[it], (30, 82), "f32", 1, (41, 15), it, data="mixed")

    # ---- ai: integer-factor INTER_AREA ----
    for isx, isy in ((2, 4), (3, 3), (2, 3), (1, 3), (3, 1)):
        for dtype, cn in TYPES6:
            add("ai", "%dx%d-a%d-%s" % (isx, isy, isx * isy % 4, _tn(dtype, cn)), (7 * isy, 9 * isx), dtype, cn, (9, 7), AREA, data="mixed" if dtype == "f32" else "rand")
    add("ai", "sum2e24-u8c1", (300, 600), "u8", 1, (2, 1), AREA, data="high")       # 300 x 300 window, sums up to 2.3e7 > 2^24

    # ---- ag: fractional INTER_AREA ----
    # 2001 -> 1001: partial pixels of 1/1001 < 1e-3 are dropped; 1997 -> 999: 1/999 > 1e-3 are kept
    for dtype in ("u8", "f32"):
        add("ag", "below-%sc1" % dtype, (6, 2001), dtype, 1, (1001, 3), AREA)
        add("ag", "above-%sc1" % dtype, (6, 1997), dtype, 1, (999, 3), AREA)
        add("ag", "below-y-%sc1" % dtype, (2001, 6), dtype, 1, (3, 1001), AREA)
        # 5 -> 3 and 8 -> 5: the last cell, min(scale, ssize - fsx1), is shorter than the scale by an ulp (fp64 search)
        add("ag", "short-%sc3" % dtype, (8, 5), dtype, 3, (3, 5), AREA)
        add("ag", "d1x1-%sc3" % dtype, (7, 5), dtype, 3, (1, 1), AREA)
        add("ag", "d1xN-%sc1" % dtype, (50, 9), dtype, 1, (1, 13), AREA)
        add("ag", "dNx1-%sc4" % dtype, (9, 50), dtype, 4, (13, 1), AREA)
        add("ag", "frac-%sc3" % dtype, (77, 101), dtype, 3, (29, 31), AREA)

    # ---- ex: exact resizers ----
    for dtype, cn in (("u8", 1), ("u8", 3), ("u8", 4), ("f32", 1), ("f32", 3), ("f32", 4)):      # pixel sizes 1, 3, 4, 4, 12, 16
        add("ex", "nnx-up-%s" % _tn(dtype, cn), (30, 45), dtype, cn, (77, 61), NEAREST_EXACT)
        add("ex", "nnx-down-%s" % _tn(dtype, cn), (61, 77), dtype, cn, (30, 45), NEAREST_EXACT)
    for cn in (1, 3, 4):
        add("ex", "linx-up-u8c%d" % cn, (20, 30), "u8", cn, (67, 51), LINEAR_EXACT)      # left copies, interior, right copies
        add("ex", "linx-down-u8c%d" % cn, (51, 67), "u8", cn, (30, 20), LINEAR_EXACT)
        add("ex", "linx-s1x1-u8c%d" % cn, (1, 1), "u8", cn, (5, 4), LINEAR_EXACT)
        add("ex", "linx-s2x2-u8c%d" % cn, (2, 2), "u8", cn, (7, 5), LINEAR_EXACT)
    add("ex", "nnx-sw32767-u8c1", (2, 32767), "u8", 1, (100, 3), NEAREST_EXACT)

    # ---- lz: LANCZOS4.  dh = 37: the smallest source height giving each DH of resize_lanczos4_sep_kernel, and the first with none ----
    LZ = {1: (10, 202, 417, 889, 2073), 3: (10, 61, 124, 265, 618), 4: (10, 45, 90, 191, 445)}
    for cn, shs in LZ.items():
        for DH, sh in zip((32, 16, 8, 4, 0), shs):
            add("lz", ("dh%d" % DH if DH else "fallback") + "-sh%d-u8c%d" % (sh, cn), (sh, 30), "u8", cn, (29, 37), LANCZOS4)
        add("lz", "last4-sh%d-u8c%d" % (shs[-1] - 1, cn), (shs[-1] - 1, 30), "u8", cn, (29, 37), LANCZOS4)
    for cn in (1, 3):
        for dw in (63, 64, 65, 129):
            add("lz", "w%d-u8c%d" % (dw, cn), (23, 100), "u8", cn, (dw, 19), LANCZOS4)
    for cn in (1, 3, 4):
        for dw in ((20, 21, 22, 23) if cn != 4 else (21,)):
            add("lz", "w%d-f32c%d" % (dw, cn), (17, 30), "f32", cn, (dw, 25), LANCZOS4, data="mixed")
    for dtype, cn in (("u8", 1), ("u8", 3), ("f32", 1)):
        add("lz", "check-up-%s" % _tn(dtype, cn), (16, 16), dtype, cn, (37, 35), LANCZOS4, data="check")
        add("lz", "check-down-%s" % _tn(dtype, cn), (40, 40), dtype, cn, (27, 23), LANCZOS4, data="check")

    # ---- fx: explicit scales ----
    for it in (NEAREST, LINEAR, CUBIC):
        for dtype, cn in (("u8", 3), ("f32", 1), ("u8", 1)):
            for fx, fy in ((0.333, 0.61), (1.7, 2.3), (0.4567, 1.234)):
                add("fx", "%g,%g-%s-%s" % (fx, fy, _tn(dtype, cn), INAME[it]), (77, 100), dtype, cn, None, it, fxfy=(fx, fy))
    for dtype, cn in (("u8", 1), ("f32", 3), ("u8", 4)):
        add("fx", "half-even-%s" % _tn(dtype, cn), (62, 90), dtype, cn, None, LINEAR, fxfy=(0.5, 0.5))

    # ---- bt: batches, one per kernel family ----
    for name, src, dtype, cn, dsize, it in (
            ("nn", (50, 61), "u8", 3, (41, 30), NEAREST), ("nn-walk", (20, 37), "u8", 1, (40, 45), NEAREST),
            ("nn-f32", (50, 61), "f32", 4, (41, 30), NEAREST), ("sep-lin", (40, 300), "u8", 3, (257, 37), LINEAR),
            ("sep-cub", (40, 300), "u8", 4, (129, 37), CUBIC), ("pp-lin", (13 * 28, 63), "u8", 1, (150, 13), LINEAR),
            ("pp-cub", (13 * 9, 64), "u8", 3, (45, 13), CUBIC), ("f32-lin", (31, 29), "f32", 3, (42, 45), LINEAR),
            ("f32-cub", (31, 29), "f32", 1, (43, 45), CUBIC), ("a2-u8", (22, 82), "u8", 3, (41, 11), AREA),
            ("a2-f32", (22, 82), "f32", 1, (41, 11), AREA), ("ai", (21, 18), "f32", 3, (9, 7), AREA),
            ("ag", (77, 101), "u8", 3, (29, 31), AREA), ("am", (60, 30), "u8", 3, (70, 25), AREA),
            ("linx", (20, 30), "u8", 3, (67, 51), LINEAR_EXACT), ("nnx", (30, 45), "f32", 3, (77, 61), NEAREST_EXACT),
            ("lz-sep", (23, 100), "u8", 3, (65, 19), LANCZOS4), ("lz-f32", (17, 30), "f32", 3, (22, 25), LANCZOS4),
            ("lz-pp", (618, 30), "u8", 3, (29, 37), LANCZOS4)):
        add("bt", name, src, dtype, cn, dsize, it, frames=3)

    # ---- dg: degenerate sizes ----
    for it in (NEAREST, LINEAR, CUBIC, AREA, LANCZOS4):
        for dtype, cn in (("u8", 3), ("f32", 1)):
            t = "%s-%s" % (_tn(dtype, cn), INAME[it])
            add("dg", "s1x1-" + t, (1, 1), dtype, cn, (5, 4), it)
            add("dg", "d1x1-" + t, (20, 30), dtype, cn, (1, 1), it)
            add("dg", "row-" + t, (1, 50), dtype, cn, (30, 1), it)
            add("dg", "col-" + t, (50, 1), dtype, cn, (1, 30), it)
            add("dg", "to-row-" + t, (20, 30), dtype, cn, (41, 1), it)
            add("dg", "same-" + t, (20, 30), dtype, cn, (30, 20), it)
    for it in (NEAREST, LINEAR, CUBIC):
        add("dg", "rows65535-u8c1-%s" % INAME[it], (65535, 3), "u8", 1, (2, 65535), it)
    add("dg", "rows65535-down-u8c1-lin", (65535, 3), "u8", 1, (5, 1000), LINEAR)

    # ---- nf: extreme float data ----
    for cn in (1, 3):
        for name, src, dsize, it in (("lin-up", (20, 23), (41, 37), LINEAR), ("lin-down", (37, 41), (23, 20), LINEAR),
                                     ("cub-up", (20, 23), (41, 37), CUBIC), ("cub-int", (20, 23), (46, 40), CUBIC),
                                     ("cub-down", (37, 41), (23, 20), CUBIC), ("area-int", (21, 27), (9, 7), AREA),
                                     ("area-frac", (37, 41), (23, 20), AREA), ("area2", (22, 42), (21, 11), AREA),
                                     ("nn", (37, 41), (23, 20), NEAREST), ("lz4", (20, 23), (41, 37), LANCZOS4)):
            add("nf", "%s-f32c%d" % (name, cn), src, "f32", cn, dsize, it, data="extreme")
    return out


CASES = _cases()
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)

# Calls the library declines with NOT_IMPLEMENTED, leaving the destination alone (the reference computes them; they are not in CASES).
REFUSALS = [
    Case("rf-src-rows65536", "rf", (65536, 2), "u8", 1, (3, 100), LINEAR, None, 1, "rand"),
    Case("rf-dst-rows65536", "rf", (100, 2), "u8", 1, (3, 65536), NEAREST, None, 1, "rand"),
    Case("rf-nnx-sw32768", "rf", (2, 32768), "u8", 1, (100, 3), NEAREST_EXACT, None, 1, "rand"),
    Case("rf-nnx-sh32768", "rf", (32768, 2), "u8", 1, (3, 100), NEAREST_EXACT, None, 1, "rand"),
    Case("rf-half-odd-w", "rf", (62, 91), "u8", 1, (46, 31), LINEAR, (0.5, 0.5), 1, "rand"),
    Case("rf-half-odd-h", "rf", (61, 90), "f32", 3, (45, 30), AREA, (0.5, 0.5), 1, "rand"),
    Case("rf-fx-area", "rf", (60, 90), "u8", 3, (30, 20), AREA, (0.333, 0.333), 1, "rand"),
]


# ---- inputs -------------------------------------------------------------------------------------------------------------------
EXTREME = np.array([np.inf, -np.inf, np.nan, -0.0, 0.0, 1e-45, -1e-45, 1.17e-38, 3e38, -3e38, 1e-3, -2.5, 7.0, 255.0], np.float32)


def frames_of(case):
    """the case's source frames, a list of (h, w) or (h, w, cn) arrays"""
    rng = np.random.default_rng(int.from_bytes(hashlib.sha256(case.id.encode()).digest()[:8], "little"))
    h, w = case.src
    shape = (h, w) if case.cn == 1 else (h, w, case.cn)
    out = []
    for _ in range(case.frames):
        if case.data == "check":                               # 1-pixel checkerboard of 0 and 255: overshoots both ways
            a = (((np.arange(h)[:, None] + np.arange(w)[None, :]) & 1) * 255).astype(np.uint8)
            a = a if case.cn == 1 else np.repeat(a[:, :, None], case.cn, 2)
        elif case.data == "ties":                              # even columns v = 1 mod 4 (one v per row and channel), odd columns 0
            a = np.zeros(shape, np.uint8)
            a[:, 0::2] = (1 + 4 * rng.integers(0, 64, (h, 1) if case.cn == 1 else (h, 1, case.cn))).astype(np.uint8)
        elif case.data == "high":
            a = rng.integers(200, 256, shape, dtype=np.uint8)
        else:
            a = rng.integers(0, 256, shape, dtype=np.uint8)
        if case.dtype == "u8":
            out.append(a)
            continue
        f = (a.astype(np.float32) + np.float32(0.37)) * np.float32(0.731)
        if case.data == "mixed":                               # magnitudes 1e-6 .. 1e6 with both signs: the summation order shows
            f = f * np.float32(10.0) ** rng.integers(-6, 7, shape).astype(np.float32) * rng.choice(np.float32([-1, 1]), shape)
        elif case.data == "extreme":                           # a quarter of the elements from EXTREME, the rest ordinary
            pick = rng.random(shape) < 0.25
            f = np.where(pick, EXTREME[rng.integers(0, len(EXTREME), shape)], f).astype(np.float32)
            f[:3] = np.float32(-0.0)                           # whole rows of -0.0: the sign of zero through every tap
        out.append(f.astype(np.float32))
    return out


def run(oracle, case, img):
    """the case through an oracle.api.Oracle (port or reference)"""
    if case.fxfy is not None:
        return oracle.resize_fxfy(img, case.fxfy[0], case.fxfy[1], case.interp)
    return oracle.resize(img, case.dsize, case.interp)


def canonical(a):
    """float arrays: every NaN as 0x7FC00000 (x86 produces 0xFFC00000, CUDA 0x7FFFFFFF); other values, -0.0 included, as they are"""
    a = np.ascontiguousarray(a)
    if a.dtype != np.float32:
        return a
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000
    return b.view(np.float32)


def differs(got, want):
    """elementwise: not bit-identical after canonical()"""
    g, w = canonical(got), canonical(want)
    if g.dtype == np.float32:
        g, w = g.view(np.uint32), w.view(np.uint32)
    return g != w


def same(got, want):
    return np.asarray(got).shape == np.asarray(want).shape and not differs(got, want).any()


def digest(arrays):
    """SHA-256 over the canonical bytes of the results of a case's frames, its first 64 bits in hex"""
    h = hashlib.sha256()
    for a in arrays:
        a = canonical(a)
        h.update(("%s%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()[:16]


# ---- the dispatch restated: which kernel a case runs on ---------------------------------------------------------------------
Pred = collections.namedtuple("Pred", "kernel args DH")
RS_BUDGET, RS_ROW_BYTES, LS_BUDGET, LS_DW = 40 * 1024, 48, 44 * 1024, 64


def scales(case):
    """(inv_x, inv_y): dsize / ssize, or fx, fy when given"""
    if case.fxfy is not None:
        return case.fxfy
    return case.dsize[0] / case.src[1], case.dsize[1] / case.src[0]


def src_index(n, scale, area_mode=False):
    """the reference's source index of destinations 0 .. n-1 (resize.cpp:4097-4124): floor(float((d + 0.5) scale - 0.5)), or
    floor(d scale) in area mode"""
    d = np.arange(n, dtype=np.float64)
    if area_mode:
        return np.floor(d * scale).astype(np.int64)
    return np.floor(((d + 0.5) * scale - 0.5).astype(np.float32)).astype(np.int64)


def rs_rmax(case, cubic, area_mode, DH):
    """resize_sep.cu:rs_host_rmax: the most distinct source rows a tile of DH destination rows reads"""
    sh, dh = case.src[0], case.dsize[1]
    s = src_index(dh, 1.0 / scales(case)[1], area_mode)
    y0 = np.arange(0, dh, DH)
    first = np.clip(s[y0] - (1 if cubic else 0), 0, sh - 1)
    last = np.clip(s[np.minimum(y0 + DH, dh) - 1] + (2 if cubic else 1), 0, sh - 1)
    return max(1, int((last - first + 1).max()))


def rs_tile(case, cubic, area_mode=False):
    """launch_rs's choice: (DH, RMAX), or (None, None) when no tile fits in 40 KB"""
    E = (128 if cubic else 256) * case.cn
    for DH in (64, 48, 32, 24, 16, 8, 4):
        r = rs_rmax(case, cubic, area_mode, DH)
        if r * E * (4 if cubic else 2) + DH * RS_ROW_BYTES <= RS_BUDGET:
            return DH, r
    return None, None


def lz_tile(case):
    """launch_lanczos_sep's choice of DH, or None"""
    dh = case.dsize[1]
    s = src_index(dh, 1.0 / scales(case)[1])
    for DH in (32, 16, 8, 4):
        y0 = np.arange(0, dh, DH)
        rmax = int((s[np.minimum(y0 + DH, dh) - 1] + 4 - (s[y0] - 3) + 1).max())
        if rmax * LS_DW * case.cn * 4 <= LS_BUDGET:
            return DH
    return None


def hpass_margins(case):
    """A + NT CN + 7 - row_bytes for every destination column whose taps are interior (resize_sep.cu:rs_hpass_thread): <= 0 takes the
    word-load path"""
    sw, dw, cn = case.src[1], case.dsize[0], case.cn
    s = src_index(dw, 1.0 / scales(case)[0])
    if case.interp == CUBIC:
        return {int((x - 1) * cn + 4 * cn + 7 - sw * cn) for x in s if x >= 1 and x + 2 <= sw - 1}
    return {int(x * cn + 2 * cn + 7 - sw * cn) for x in s if 0 <= x < sw - 1}


def predict(case, path=None, src_aligned=None, dst_aligned=None):
    """the kernel resize_impl runs for the case: Pred(name, template arguments, DH of the tiled kernels) or Pred("copy" | "refused", ...).
    path: ("nn", "v1" | "walk") or ("lz", "v1") for B200CV_RESIZE_NN_PATH / B200CV_RESIZE_LANCZOS_PATH.  *_aligned: the 4-byte alignment
    of data, row step and frame step; by default that of a contiguous array"""
    sh, sw = case.src
    dw, dh = case.dsize
    u8 = case.dtype == "u8"
    pix = case.cn * (1 if u8 else 4)
    T = case.dtype
    if src_aligned is None:
        src_aligned = sw * pix % 4 == 0
    if dst_aligned is None:
        dst_aligned = dw * pix % 4 == 0
    it = case.interp
    if sh >= 65536 or dh >= 65536:
        return Pred("refused", (), None)
    if (sw, sh) == (dw, dh):
        return Pred("copy", (), None)
    inv_x, inv_y = scales(case)
    explicit = case.fxfy is not None and (inv_x != dw / sw or inv_y != dh / sh)
    if explicit and it not in (NEAREST, LINEAR, CUBIC):
        return Pred("refused", (), None)
    if it == NEAREST_EXACT:
        if sw >= 32768 or sh >= 32768:
            return Pred("refused", (), None)
        return Pred("resize_nn_exact_kernel", (pix,), None)
    if it == LINEAR_EXACT and not u8:
        it = LINEAR
    if it == NEAREST:
        env = path[1] if path and path[0] == "nn" else None
        walk = env == "walk" or (dh > sh and env != "v1")
        if walk and u8 and dst_aligned:
            return Pred("resize_nn_walk_kernel", (pix,), None)
        return Pred("resize_nn_kernel", (pix,), None)
    scale_x, scale_y = 1.0 / inv_x, 1.0 / inv_y
    isx, isy = int(round(scale_x)), int(round(scale_y))
    area_fast = abs(scale_x - isx) < 2.220446049250313e-16 and abs(scale_y - isy) < 2.220446049250313e-16
    if it in (LINEAR, AREA, LINEAR_EXACT) and area_fast and isx == 2 and isy == 2:
        if 2 * dw != sw or 2 * dh != sh:
            return Pred("refused", (), None)
        return Pred("resize_area2_u8_kernel" if u8 else "resize_area2_f32_kernel", (case.cn,), None)
    if it == LINEAR_EXACT:
        return Pred("resize_linear_exact_kernel", (case.cn,), None)
    if it == LANCZOS4:
        if u8 and not (path and path[0] == "lz" and path[1] == "v1"):
            DH = lz_tile(case)
            if DH:
                return Pred("resize_lanczos4_sep_kernel", (case.cn,), DH)
        return Pred("resize_lanczos4_kernel", (T, case.cn), None)
    area_mode = False
    if it == AREA:
        if scale_x >= 1 and scale_y >= 1:
            isx, isy = int(np.rint(scale_x)), int(np.rint(scale_y))
            integer = abs(scale_x - isx) < 2.220446049250313e-16 and abs(scale_y - isy) < 2.220446049250313e-16
            return Pred("resize_area_int_kernel" if integer else "resize_area_kernel", (T, case.cn), None)
        area_mode, it = True, LINEAR
    cubic = it == CUBIC
    if u8:
        DH, _ = rs_tile(case, cubic, area_mode)
        if DH:
            return Pred("resize_sep_u8_kernel", (case.cn, cubic), DH)
    return Pred("resize_cubic_kernel" if cubic else "resize_linear_kernel", (T, case.cn), None)


def tile_of(pred):
    """(destination columns, destination rows) one CTA / thread block of the kernel covers, for naming where a difference lies"""
    k = pred.kernel
    if k == "resize_sep_u8_kernel":
        return (128 if pred.args[1] else 256), pred.DH
    if k == "resize_lanczos4_sep_kernel":
        return LS_DW, pred.DH
    if k in ("resize_linear_kernel", "resize_cubic_kernel"):
        return 256, 8
    if k == "resize_nn_walk_kernel":
        return 512, 32
    if k in ("resize_nn_kernel", "resize_area2_u8_kernel"):
        return 512 if k == "resize_nn_kernel" else 1024, 1
    return 256, 1


def body_limit(case, pred):
    """elements of a destination row computed by the reference's vector body (the rest: its scalar tail), or None where the kernel
    does not split"""
    n = case.dsize[0] * case.cn
    if case.interp == CUBIC and case.dtype == "u8":
        return n // 8 * 8
    if case.dtype == "f32" and (case.interp == CUBIC or case.interp == LANCZOS4):
        return n // 4 * 4
    if pred.kernel == "resize_area2_f32_kernel" and case.cn == 1:
        return n // 4 * 4
    return None
