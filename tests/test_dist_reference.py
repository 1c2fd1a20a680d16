"""The plain-C restatement of cv::distanceTransform (oracle/port/port_distance.c) against the reference over the whole table of
tests/dist_cases.py, bit for bit: always against the SHA-256 of the reference's answers recorded in tests/golden/dist_ref.json by
tools/make_dist_golden.py, and against the live reference where oracle/_ref/libdistref.so is built.

tests/test_gpu_distance_transform.py holds the CUDA kernels to the restatement.  This file also checks, on the CPU, the two claims the
device's kernels rest on: the 8-bit L1 call equals the L1 3x3 chamfer with the epilogue min(t >> 16, 255), and the row pass's binary
search over z picks the parabola of the reference's linear walk, on every case of the table.
"""
import ctypes
import json
import os

import numpy as np
import pytest

import dist_cases as dc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dist_ref.json")
IMAGES = sorted({c.image: c for c in dc.CASES}.values(), key=lambda c: c.image)


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)["dist"]


@pytest.fixture(scope="module")
def port_lib(port):          # the session fixture builds oracle/_build/liboracle_port.so
    return ctypes.CDLL(dc.PORT_LIB)


def test_golden_covers_the_table(golden):
    assert set(golden) == {c.id for c in dc.CASES}


def test_table_covers_every_call(golden):
    calls = {c.call for c in dc.CASES}
    assert calls == set(dc.CALLS)
    for c in dc.CASES:
        assert (golden[c.id] == "refused") == (c.call in dc.REFUSED), c.id
        if c.call not in dc.REFUSED:
            assert golden[c.id].startswith("0:" if dc.out_is_u8(c.call) else "5:"), c.id


@pytest.mark.parametrize("case", dc.CASES, ids=lambda c: c.id)
def test_port_vs_reference(port, golden, case):
    img = dc.image_of(case)
    depth, got = dc.run("port", img, case.call)
    if dc.ref_available():
        rdepth, want = dc.run("ref", img, case.call)
        assert depth == rdepth, "%s: depth %d vs the reference's %d" % (case.id, depth, rdepth)
        if want is not None:
            bad = np.argwhere(got.view(np.uint8 if got.dtype == np.uint8 else np.int32) != want.view(np.uint8 if want.dtype == np.uint8 else np.int32))
            assert len(bad) == 0, "%s: %d elements differ, first at %s" % (case.id, len(bad), tuple(bad[0]))
    assert dc.digest(depth, got) == golden[case.id], "%s: the port's result is not the one recorded from the reference" % case.id


@pytest.mark.parametrize("case", IMAGES, ids=lambda c: c.image)
def test_l1_u8_scans_equal_the_l1_chamfer_epilogue(port_lib, case):
    """the reference's saturating 8-bit L1 scans and the L1 3x3 chamfer (weights 1, 2) with min(t >> 16, 255) agree"""
    img = np.ascontiguousarray(dc.image_of(case))
    H, W = img.shape
    scans = dc.run("port", img, "l1_u8")[1]
    chamfer = np.zeros((H, W), np.uint8)
    assert port_lib.port_dist_l1_u8_chamfer(ctypes.c_void_p(img.ctypes.data), ctypes.c_size_t(W), ctypes.c_void_p(chamfer.ctypes.data),
                                            ctypes.c_size_t(W), W, H) == 0
    bad = np.argwhere(scans != chamfer)
    assert len(bad) == 0, "%s: %d pixels differ, first at %s" % (case.image, len(bad), tuple(bad[0]))


@pytest.mark.parametrize("case", IMAGES, ids=lambda c: c.image)
def test_binary_search_picks_the_linear_walks_parabola(port_lib, case):
    """on every row, z increases strictly along the envelope's stack and the smallest k with z[k+1] >= q is the k of the reference's
    walk `while (z[k+1] < q) k++`"""
    img = np.ascontiguousarray(dc.image_of(case))
    H, W = img.shape
    fn = port_lib.port_dist_lookup_mismatches
    fn.restype = ctypes.c_long
    assert fn(ctypes.c_void_p(img.ctypes.data), ctypes.c_size_t(W), W, H) == 0, case.image
