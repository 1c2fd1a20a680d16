"""The C port's cv::resize (oracle/port/port_geometry.c) against the reference over the whole table of tests/resize_cases.py, 8-bit and
float, bit for bit (NaN compared as NaN, every other value by its bits, the sign of zero included).

tests/test_gpu_resize_exact_edges.py ties the CUDA kernels to the port, and the port and the kernels were written from one reading of
resize.cpp: a formula wrong in both would pass there.  This file is where such an error shows.  With oracle/_ref built the port is
compared with the live reference; without it with the SHA-256 of the reference's answers recorded in tests/golden/resize_ref.json by
tools/make_resize_golden.py.

It also checks, on the CPU, the claims the case table is built on (which DH launch_rs and launch_lanczos_sep choose at the `sy` and `lz`
source heights, where the `sx` edge widths put the H pass's word loads), and runs the `sx` / `sy` / `am` cases through the host
emulation of resize_sep_u8_kernel at the DH predict() names, where a tile that reads more source rows than the host sized its shared
memory for (R > RMAX, which the kernel clamps silently) is an error.
"""
import json
import os

import numpy as np
import pytest

import resize_cases as rc
from oracle.api import Oracle, available

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_ref.json")


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)


@pytest.fixture(scope="module")
def live_ref():
    return Oracle("ref") if available("ref") else None


def first_difference(got, want):
    bad = np.argwhere(rc.differs(got, want))
    g, w = rc.canonical(got), rc.canonical(want)
    return "%d elements differ, first at %s: got %r want %r" % (len(bad), tuple(bad[0]), g[tuple(bad[0])], w[tuple(bad[0])])


def test_golden_covers_the_table(golden):
    assert set(golden["resize"]) == {c.id for c in rc.CASES}


@pytest.mark.parametrize("case", rc.CASES, ids=lambda c: c.id)
def test_port_vs_reference(port, live_ref, golden, case):
    frames = rc.frames_of(case)
    got = [rc.run(port, case, f) for f in frames]
    if live_ref is not None:
        for i, f in enumerate(frames):
            want = rc.run(live_ref, case, f)
            assert rc.same(got[i], want), "%s frame %d (%s): %s" % (case.id, i, rc.predict(case).kernel, first_difference(got[i], want))
    assert rc.digest(got) == golden["resize"][case.id], "%s: the port's result is not the one recorded from the reference" % case.id


@pytest.mark.parametrize("case", rc.REFUSALS, ids=lambda c: c.id)
def test_refusals_are_refusals(case):
    assert rc.predict(case).kernel == "refused"


# ---- the claims the table is built on ------------------------------------------------------------------------------------------
def test_row_block_edges():
    """each `sy` case gets the DH its id names; last4 / fallback are neighbouring source heights on either side of the per-pixel fallback"""
    for c in rc.CASES:
        if c.group != "sy":
            continue
        p = rc.predict(c)
        name = c.id.split("-")[1]
        if name.startswith("dh"):
            assert p == rc.Pred("resize_sep_u8_kernel", (c.cn, c.interp == rc.CUBIC), int(name[2:])), c.id
        elif name == "last4":
            assert p.DH == 4, c.id
            nxt = rc.BY_ID[c.id.replace("last4-sh%d" % c.src[0], "fallback-sh%d" % (c.src[0] + 1))]
            assert rc.predict(nxt).kernel == ("resize_cubic_kernel" if c.interp == rc.CUBIC else "resize_linear_kernel"), nxt.id
    for cn in (1, 3, 4):
        for it in (rc.LINEAR, rc.CUBIC):
            got = {rc.predict(c).DH for c in rc.CASES if c.group == "sy" and c.cn == cn and c.interp == it}
            assert got == {64, 48, 32, 24, 16, 8, 4, None}, (cn, it, got)


def test_lanczos_row_block_edges():
    for c in rc.CASES:
        if c.group != "lz" or c.dtype != "u8" or not c.id.split("-")[1].startswith(("dh", "fallback", "last4")):
            continue
        p, name = rc.predict(c), c.id.split("-")[1]
        if name == "fallback":
            assert p == rc.Pred("resize_lanczos4_kernel", ("u8", c.cn), None), c.id
        else:
            assert p == rc.Pred("resize_lanczos4_sep_kernel", (c.cn,), 4 if name == "last4" else int(name[2:])), c.id


def test_hpass_edge_widths():
    """`edge-on`: a column whose NW + 1 words end exactly at the row end takes the word path (margin m0, the largest <= 0 its residue
    allows); `edge-past`: the nearest column is one step (CN bytes) past it and takes the byte path"""
    n = 0
    for c in rc.CASES:
        if c.group == "sx" and c.id.startswith("sx-edge"):
            m = rc.hpass_margins(c)
            m0 = next(v for v in range(-c.cn + 1, 1) if (v - min(m)) % c.cn == 0)
            if "-on-" in c.id:
                assert m0 in m, (c.id, sorted(m)[-4:])
            else:
                assert m0 not in m and m0 + c.cn in m, (c.id, sorted(m)[-4:])
            n += 1
    assert n == 12


def test_area_threshold_cases_straddle_1e3():
    """the `ag-below` / `ag-above` factors put partial pixels of 1/1001 and 1/999 of a pixel next to whole ones: under and over the
    1e-3 below which computeResizeAreaTab drops them"""
    for sw, dw, under in ((2001, 1001, True), (1997, 999, False)):
        scale = 1.0 / (dw / sw)
        smallest = min(v for v in (np.ceil(d * scale) - d * scale for d in range(dw)) if v > 0)
        assert (smallest <= 1e-3) == under and 0.99e-3 < smallest < 1.01e-3, (sw, dw, smallest)


def test_kernels_each_case_family_reaches():
    """every kernel and instantiation the table is meant to reach is predicted for some case"""
    preds = {(p.kernel, p.args) for p in map(rc.predict, rc.CASES)}
    for T in ("u8", "f32"):
        for cn in (1, 3, 4):
            for k in ("resize_linear_kernel", "resize_cubic_kernel", "resize_area_int_kernel", "resize_area_kernel", "resize_lanczos4_kernel"):
                assert (k, (T, cn)) in preds, (k, T, cn)
    for cn in (1, 3, 4):
        for k in ("resize_area2_u8_kernel", "resize_area2_f32_kernel", "resize_linear_exact_kernel", "resize_nn_walk_kernel"):
            assert (k, (cn,)) in preds, (k, cn)
        assert ("resize_lanczos4_sep_kernel", (cn,)) in preds
        for cubic in (False, True):
            assert ("resize_sep_u8_kernel", (cn, cubic)) in preds
    for pix in (1, 3, 4, 12, 16):
        assert ("resize_nn_kernel", (pix,)) in preds and ("resize_nn_exact_kernel", (pix,)) in preds


# ---- explicit scales: the port's own entry against plain meaning ---------------------------------------------------------------
def test_port_explicit_scale_differs_from_dsize(port):
    """with cols * fx not an integer the sampling scale fx differs from dsize / ssize, and so does the answer"""
    c = rc.BY_ID["fx-0.333,0.61-u8c3-lin"]
    img = rc.frames_of(c)[0]
    assert c.dsize == (33, 47)
    assert not np.array_equal(port.resize_fxfy(img, 0.333, 0.61, rc.LINEAR), port.resize(img, c.dsize, rc.LINEAR))
    even = rc.BY_ID["fx-half-even-u8c1"]
    img = rc.frames_of(even)[0]
    assert np.array_equal(port.resize_fxfy(img, 0.5, 0.5, rc.LINEAR), port.resize(img, even.dsize, rc.AREA))
