"""The numpy restatement of cv::erode / cv::dilate / cv::morphologyEx (tests/morph_reference.py) against the reference over the whole
table of tests/morph_cases.py: always against the SHA-256 digests recorded in tests/golden/morph_ref.json by tools/make_morph_golden.py,
and against the live reference where oracle/_ref/libmorphref.so is built.  32F elements whose windows hold a NaN or a -0.0 are zeroed on
both sides (the reference's answer there depends on the column).  opencv_b200.getStructuringElement is held to the reference the same way.

tests/test_gpu_morphology.py holds the CUDA kernels to the restatement.
"""
import hashlib
import json
import os

import numpy as np
import pytest

import morph_cases as mc
import morph_reference as mr
import opencv_b200 as C

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "morph_ref.json")


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)


def test_golden_covers_the_table(golden):
    assert set(golden["morph"]) == {"%s/%s" % (c.id, n) for c in mc.CASES for n in c.calls}
    assert all(any(n in c.calls for c in mc.CASES) for n in mc.ALL_CALLS)


@pytest.mark.parametrize("case", mc.CASES, ids=lambda c: c.id)
def test_restatement_vs_reference(golden, case):
    img = mc.image_of(case)
    for name, call in case.calls.items():
        try:
            got, excl = mc.restated(img, call)
        except mr.Refused:
            got, excl = None, None
        if mc.ref_available():
            want = mc.reference(img, case.depth, call)
            assert (want is None) == (got is None), "%s/%s: refusal differs from the reference" % (case.id, name)
            if want is not None:
                bad = np.argwhere((got.view(np.uint8) != want.view(np.uint8)).reshape(got.shape + (-1,)).any(-1) & ~excl)
                assert len(bad) == 0, "%s/%s: %d elements differ, first at %s" % (case.id, name, len(bad), tuple(bad[0]))
        assert mc.digest(got, excl) == golden["morph"]["%s/%s" % (case.id, name)], "%s/%s: not the recorded answer" % (case.id, name)


@pytest.mark.parametrize("name", sorted(mc.UNDEFINED))
def test_element_without_a_non_zero_entry_is_refused(name):
    call = mc.UNDEFINED[name]
    with pytest.raises(mr.Refused):
        mc.restated(np.zeros((5, 5), np.uint8), call)


def test_excluded_windows_are_the_special_ones():
    """a NaN or -0.0 excludes exactly the outputs whose window reaches it; +-inf excludes nothing"""
    img = np.ones((9, 9), np.float32)
    img[4, 4] = np.nan
    img[0, 8] = np.inf
    ex = mr.excluded(img, "erode", 0, np.ones((3, 3), np.uint8))
    assert ex.sum() == 9 and ex[3:6, 3:6].all()


def test_structuring_elements(golden):
    for shape, w, h, anchor in mc.STRUCTURING:
        key = "%d-%dx%d-%d,%d" % (shape, w, h, anchor[0], anchor[1])
        try:
            e = C.getStructuringElement(shape, (w, h), anchor)
        except C.B200cvError:
            e = None
        if mc.ref_available():
            want = mc.ref_structuring_element(shape, w, h, anchor)
            assert (want is None) == (e is None) and (e is None or np.array_equal(e, want)), key
        assert ("refused" if e is None else hashlib.sha256(e.tobytes()).hexdigest()) == golden["structuring"][key], key


@pytest.mark.parametrize("border", [mr.BORDER_CONSTANT, mr.BORDER_REPLICATE, mr.BORDER_REFLECT, mr.BORDER_REFLECT_101])
def test_rectangles_reaching_past_twice_the_image_change_nothing(border):
    """a window that reaches more than twice the line's length past an end holds no value it would not hold at that reach: the device
    shrinks such rectangles (opencv_b200/csrc/morph.cu, vh_extent), so the answers at 40 and 100 iterations of 3x3 on 13x17 agree"""
    img = mc.image_of(mc.Case("h", "h-%d" % border, (13, 17), "16S", 2, "random", {}))
    k = np.ones((3, 3), np.uint8)
    for op in (mr.MORPH_ERODE, mr.MORPH_DILATE, mr.MORPH_TOPHAT):
        a = mr.morphology(img, "mex", op, k, (-1, -1), 2 * 17 + 6, border)
        b = mr.morphology(img, "mex", op, k, (-1, -1), 100, border)
        assert np.array_equal(a, b), (op, border)


def test_empty_elements_of_every_kind_reach_the_abi_alike():
    """morphologyEx turns every empty element (None, [], an empty array or tensor) into the 3x3 rectangle; erode / dilate keep it empty"""
    import torch
    for empty in (None, [], np.zeros((0, 3), np.uint8), torch.empty(0, dtype=torch.uint8)):
        k, kp, kw, kh, bv = C._morph_args(empty, None, True)
        assert (kw, kh) == (3, 3) and k.all()
        k, kp, kw, kh, bv = C._morph_args(empty, None, False)
        assert (k, kp, kw, kh) == (None, None, 0, 0)
