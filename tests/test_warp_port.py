"""The C port's warpAffine / warpPerspective / remap (oracle/port/port_geometry.c, warp_impl) against the reference over the whole table
of tests/warp_cases.py, 8-bit and float, bit for bit.

tests/test_gpu_warp_exact.py ties the CUDA kernels to the port, and the port and the kernels were written from one reading of
imgwarp.cpp: a formula wrong in both (the projective block width for destinations under 16 rows, say) would pass there.  This file is
where such an error shows.  With oracle/_ref built the port is compared with the live reference; without it (a machine that has no
reference sources) with the SHA-256 of the reference's answers recorded in tests/golden/warp_ref.json by tools/make_warp_golden.py.
"""
import json
import os

import numpy as np
import pytest

import warp_cases as wc
from oracle.api import Oracle, available
from util import assert_exact

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "warp_ref.json")


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)


@pytest.fixture(scope="module")
def live_ref():
    return Oracle("ref") if available("ref") else None


def test_golden_covers_the_table(golden):
    assert set(golden["warp"]) == {c.id for c in wc.CASES}


@pytest.mark.parametrize("case", wc.CASES, ids=lambda c: c.id)
def test_port_vs_reference(port, live_ref, golden, case):
    frames = wc.frames_of(case)
    got = [wc.run(port, case, f) for f in frames]
    if live_ref is not None:
        for i, f in enumerate(frames):
            assert_exact(got[i], wc.run(live_ref, case, f), "%s frame %d, bw0 = %d" % (case.id, i, wc.block_width(case)))
    assert wc.digest(got) == golden["warp"][case.id], "%s: the port's result is not the one recorded from the reference" % case.id


def test_row0_of_h_ties_tells_block_widths_apart():
    """The claim beside warp_cases.H_TIES, recomputed in float64: in destination row 0 the rounded coordinate depends on the column
    block the reference evaluates relative to, so the cases built on H_TIES separate one block width from another and from none."""
    M = np.array(wc.H_TIES)

    def row0(bw0, nearest, dw=1100):
        x = np.arange(dw)
        xb = x // bw0 * bw0 if bw0 else x
        x1 = (x - xb).astype(np.float64)
        xb = xb.astype(np.float64)
        W = (1.0 if nearest else 32.0) / ((M[6] * xb + M[7] * 0.0 + M[8]) + M[6] * x1)
        return np.rint(((M[0] * xb + M[1] * 0.0 + M[2]) + M[0] * x1) * W), np.rint(((M[3] * xb + M[4] * 0.0 + M[5]) + M[3] * x1) * W)

    for nearest, axis in ((True, 0), (False, 1)):
        b64, absolute, b204 = row0(64, nearest)[axis], row0(0, nearest)[axis], row0(204, nearest)[axis]
        assert (b64 != absolute).sum() > 100 and (b64 != b204).sum() > 100
        assert set(np.unique(b64)) <= ({2.0, 3.0} if nearest else {80.0, 81.0})


def test_footprint_decision_flips_between_neighbouring_cases():
    """the `fp` cases straddle the 96 KB decisions instead of sitting on one side: 8UC3 passes from the 128x32 kernel to the 64x16
    one and on to the direct gather, 32FC3 from the 64x16 kernel to the direct gather"""
    def kernels(t):
        return [wc.predict(wc.BY_ID["fp-x%g-%s-lin" % (s, t)]) for s in (1.0, 2.0, 2.5, 3.0, 4.0, 5.0, 5.5, 7.0)]
    assert kernels("u8c3") == ["warp_tile4_kernel"] * 2 + ["warp_tile_kernel"] * 3 + ["warp_kernel"] * 3
    assert kernels("f32c3") == ["warp_tile_kernel"] * 2 + ["warp_kernel"] * 6


# ---- remap with fixed-point maps and no fraction map ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,cn", wc.TYPES6)
def test_port_remap_fixed_point_without_fractions(port, live_ref, golden, dtype, cn):
    """cv::remap(CV_16SC2, noArray(), INTER_NEAREST): the map is "already in the right format" (imgwarp.cpp:1166) and is used as it
    is -- the rounding table of the two-map form does not apply"""
    case = wc.remap_case(dtype, cn)
    src = wc.frames_of(case)[0]
    xy = wc.fixed_maps()
    got = []
    for border in wc.BORDERS:
        got.append(port.remap(src, xy, None, wc.NEAREST, border, wc.BV4))
        if live_ref is not None:
            assert_exact(got[-1], live_ref.remap(src, xy, None, wc.NEAREST, border, wc.BV4), "%s border %d" % (case.id, border))
    # the plain meaning, independent of both: dst(y, x) = src(map(y, x)) inside the image
    inside = (xy[..., 0] >= 0) & (xy[..., 0] < 70) & (xy[..., 1] >= 0) & (xy[..., 1] < 50)
    assert inside.mean() > 0.2
    assert np.array_equal(got[0][inside], src[xy[..., 1][inside], xy[..., 0][inside]])
    assert wc.digest(got) == golden["remap"][case.id]
