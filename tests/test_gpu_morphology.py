"""GPU: cv::erode / cv::dilate / cv::morphologyEx (opencv_b200/csrc/morph.cu) bit for bit against the numpy restatement
(tests/morph_reference.py, which tests/test_morph_reference.py holds to the reference's recorded answers) over the whole table of
tests/morph_cases.py, 32F compared as int32 bits outside the windows that hold a NaN or a -0.0.  Then the device's own refusals, batches
whose frames differ, views at odd byte offsets with guard bytes, the launch count, the host path and the C++ GpuMat mirror.
Each table test uploads one image and checks every call the table makes on it."""
import os
import subprocess

import numpy as np
import pytest

import morph_cases as mc
import morph_reference as mr
import opencv_b200 as C
import opencv_b200.hal  # noqa: F401  (C.hal)
from util import cpu, gpu

pytestmark = [pytest.mark.gpu]


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a


def assert_bits(got, want, excl, what):
    assert got.shape == want.shape and got.dtype == want.dtype, "%s: %s %s vs %s %s" % (what, got.shape, got.dtype, want.shape, want.dtype)
    bad = np.argwhere((bits(got) != bits(want)) & ~excl)
    assert len(bad) == 0, "%s: %d/%d elements differ, first at %s (got %r want %r)" % (
        what, len(bad), got.size, tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])


def call_device(src, call, dst=None):
    k = mc.element(call.elem)
    if call.entry == mc.X:
        return C.morphologyEx(src, call.op, k, dst=dst, anchor=call.anchor, iterations=call.it, borderType=call.border, borderValue=call.bv)
    f = C.erode if call.entry == mc.E else C.dilate
    return f(src, k, dst=dst, anchor=call.anchor, iterations=call.it, borderType=call.border, borderValue=call.bv)


@pytest.mark.parametrize("case", mc.CASES, ids=lambda c: c.id)
def test_case(cvb, case):
    """every call the table makes on one image: the restatement's answer, or an argument error with dst untouched"""
    img = mc.image_of(case)
    src = gpu(img)
    for name, call in case.calls.items():
        try:
            want, excl = mc.restated(img, call)
        except mr.Refused:
            dst = gpu(np.full(img.shape, 7, img.dtype))
            with pytest.raises(C.B200cvError) as e:
                call_device(src, call, dst)
            assert not isinstance(e.value, C.NotImplementedOnDevice), name
            assert (cpu(dst) == 7).all(), "%s/%s: dst written" % (case.id, name)
            continue
        assert_bits(cpu(call_device(src, call)), want, excl, "%s/%s" % (case.id, name))


def test_device_refusals_leave_dst_untouched(cvb):
    """HITMISS, 64F, WRAP and a 64x64 ellipse are not implemented; an element with no non-zero entry, a dst of another type or size,
    and overlapping src / dst are argument errors"""
    import torch
    img = gpu(np.arange(30 * 40, dtype=np.uint8).reshape(30, 40))
    k3 = np.ones((3, 3), np.uint8)

    def dst7(shape=(30, 40), dtype=torch.uint8):
        return torch.full(shape, 7, dtype=dtype, device="cuda")

    ni = [lambda d: C.morphologyEx(img, C.MORPH_HITMISS, k3, dst=d),
          lambda d: C.erode(img.double(), k3, dst=d),
          lambda d: C.dilate(img, k3, dst=d, borderType=C.BORDER_WRAP),
          lambda d: C.erode(img, C.getStructuringElement(C.MORPH_ELLIPSE, (64, 64)), dst=d),
          lambda d: C.dilate(img, C.getStructuringElement(C.MORPH_CROSS, (5, 70)), dst=d)]
    for i, f in enumerate(ni):
        d = dst7(dtype=torch.float64 if i == 1 else torch.uint8)
        with pytest.raises(C.NotImplementedOnDevice):
            f(d)
        assert (cpu(d) == 7).all(), i
    bad = [(img, dst7(), lambda s, d: C.erode(s, np.zeros((3, 3), np.uint8), dst=d)),
           (img, dst7(), lambda s, d: C.morphologyEx(s, C.MORPH_OPEN, np.zeros((1, 4), np.uint8), dst=d, iterations=3)),
           (img, dst7(dtype=torch.int16), lambda s, d: C.erode(s, k3, dst=d)),
           (img, dst7((30, 41)), lambda s, d: C.dilate(s, k3, dst=d)),
           (img, dst7(), lambda s, d: C.morphologyEx(s, 9, k3, dst=d))]
    for i, (s, d, f) in enumerate(bad):
        with pytest.raises(C.B200cvError) as e:
            f(s, d)
        assert not isinstance(e.value, C.NotImplementedOnDevice), i
        assert (cpu(d) == 7).all(), i
    buf = gpu(np.arange(31 * 40, dtype=np.uint8).reshape(31, 40))
    before = cpu(buf)
    for s, d in ((buf[:30], buf[1:]), (buf[:30], buf[:30])):
        with pytest.raises(C.B200cvError):
            C.erode(s, k3, dst=d)
        assert (cpu(buf) == before).all()


def test_zero_element_copies_with_no_iterations(cvb):
    img = mc.image_of(mc.BY_ID["37x45-8U-c1-random"])
    got = cpu(C.erode(gpu(img), np.zeros((3, 3), np.uint8), iterations=0))
    assert (got == img).all()


BATCH_CALLS = ["e3", "e5ell101", "e33x5", "black3x3it", "close3x2", "rect_it10", "open_rand_it2", "d1x100", "vh_top41_bv", "vh_open33"]


@pytest.mark.parametrize("depth", list(mc.DTYPES))
def test_batch_of_different_frames(cvb, depth):
    """four frames of different content with 3 spare rows after each in both buffers: each frame its own answer, spare rows kept"""
    H, W, cn = 23, 50, 2
    frames = [mc.image_of(mc.Case("b", "b-%s-%d" % (depth, i), (H, W), depth, cn, "random", {})) for i in range(4)]
    dt = frames[0].dtype
    sbig = np.zeros((4, H + 3, W, cn), dt)
    sbig[:, :H] = np.stack(frames)
    src = gpu(sbig)[:, :H]
    for name in BATCH_CALLS:
        call = mc.ALL_CALLS[name]
        dbig = gpu(np.full((4, H + 3, W, cn), 5, dt))
        call_device(src, call, dbig[:, :H])
        out = cpu(dbig)
        for i, img in enumerate(frames):
            want, excl = mc.restated(img, call)
            assert_bits(out[i, :H], want, excl, "%s %s frame %d" % (depth, name, i))
        assert (out[:, H:] == 5).all(), "spare rows between frames were written"


@pytest.mark.parametrize("depth,cn", [("8U", 1), ("8U", 3), ("16U", 1), ("16S", 2), ("32F", 1), ("32F", 4)])
def test_views_with_guard_bytes(cvb, depth, cn):
    """source and destination as windows into larger buffers, 3 and 5 elements into padded rows (an odd byte offset for 8-bit); every
    element around the destination window keeps its value"""
    H, W = 19, 41
    img = mc.image_of(mc.Case("v", "v-%s-%d" % (depth, cn), (H, W), depth, cn, "random", {}))
    dt = img.dtype
    sbig = np.zeros((H + 2, W + 9, cn), dt)
    sbig[1:1 + H, 3:3 + W] = img.reshape(H, W, cn)
    src = gpu(sbig)[1:1 + H, 3:3 + W]
    for name in ("e3", "d15", "e33x5", "top7", "grad3", "ell31", "d33"):
        call = mc.ALL_CALLS[name]
        dbig = gpu(np.full((H + 2, W + 7, cn), 9, dt))
        call_device(src if cn > 1 else src[:, :, 0], call, dbig[1:1 + H, 5:5 + W] if cn > 1 else dbig[1:1 + H, 5:5 + W, 0])
        out = cpu(dbig)
        want, excl = mc.restated(img, call)
        expect = np.full(out.shape, 9, dt)
        expect[1:1 + H, 5:5 + W] = want.reshape(H, W, cn)
        ex = np.zeros(out.shape, bool)
        ex[1:1 + H, 5:5 + W] = excl.reshape(H, W, cn)
        assert_bits(out, expect, ex, "%s %s window and surroundings" % (depth, name))


def test_launch_count_does_not_depend_on_content_or_batch(cvb):
    """one launch per pass of the fused kernel, two per van Herk pass; compound ops add their second chain, never a subtraction launch"""
    import torch
    expect = {"e3": 1, "d33": 2, "e101x1": 2, "open5ell": 2, "grad3": 2, "black3x3it": 2, "close3x2": 4, "top_rect_it3": 2,
              "cross_it3": 3, "it0": 1, "rect_it10": 1, "empty_d3": 1, "vh_open33": 4, "vh_top41": 4, "vh_grad_it20": 4}
    for name, n in expect.items():
        for frames in (1, 3):
            for fill in ("random", "blobs"):
                img = mc.image_of(mc.Case("n", "n-%s" % fill, (40, 70), "8U", 1, fill, {}))
                src = gpu(np.stack([img] * frames)[..., None]) if frames > 1 else gpu(img)
                torch.cuda.synchronize()
                n0 = C.launch_count()
                call_device(src, mc.ALL_CALLS[name])
                assert C.launch_count() - n0 == n, (name, frames, fill)


@pytest.mark.parametrize("border", [mc.C0, mc.REP, mc.REF, mc.R101])
def test_huge_iterations_reach_only_what_the_image_holds(cvb, border):
    """3x3 with 2^29 - 1 iterations grows to a 2^30 + 1 rectangle: it runs (the van Herk walk is bounded by the image, not by the
    element) and equals the answer at 100 iterations, which already reaches past every border (tests/test_morph_reference.py checks
    that the answer no longer changes there)"""
    img = mc.image_of(mc.Case("h", "h-%d" % border, (13, 17), "16S", 2, "random", {}))
    k = np.ones((3, 3), np.uint8)
    for op in (C.MORPH_ERODE, C.MORPH_DILATE, C.MORPH_TOPHAT):
        want = mr.morphology(img, "mex", op, k, (-1, -1), 100, border)
        for it in (100, (1 << 29) - 1):
            got = cpu(C.morphologyEx(gpu(img), op, k, iterations=it, borderType=border))
            assert_bits(got, want, np.zeros(want.shape, bool), "op %d, %d iterations, border %d" % (op, it, border))


def test_empty_elements_of_every_kind(cvb):
    """None, [], an empty array and an empty tensor are all the empty element: morphologyEx's 3x3 rectangle, erode's (1+2it)^2"""
    import torch
    img = mc.image_of(mc.BY_ID["29x70-8U-c1-random"])
    for empty in (None, [], np.zeros((0, 0), np.uint8), torch.empty(0, dtype=torch.uint8)):
        for op in (C.MORPH_ERODE, C.MORPH_DILATE, C.MORPH_GRADIENT):
            want = mr.morphology(img, "mex", op, None, (-1, -1), 2)
            got = cpu(C.morphologyEx(gpu(img), op, empty, iterations=2))
            assert_bits(got, want, np.zeros(want.shape, bool), "morphologyEx op %d, %r" % (op, type(empty)))
            assert_bits(C.hal.morphologyEx(img, op, empty, iterations=2), want, np.zeros(want.shape, bool), "hal op %d" % op)
        want = mr.morphology(img, "erode", 0, None, (-1, -1), 2)
        assert_bits(cpu(C.erode(gpu(img), empty, iterations=2)), want, np.zeros(want.shape, bool), "erode %r" % type(empty))


@pytest.mark.parametrize("name", ["e3", "top7", "open_rand_it2", "d33", "bv_d", "empty_mex_e2"])
def test_host_path(cvb, name):
    """opencv_b200.hal on numpy arrays (b200cv_host_morphology), one frame and a batch of two"""
    call = mc.ALL_CALLS[name]
    case = mc.BY_ID["29x70-16S-c3-random"]
    img = mc.image_of(case)
    want, excl = mc.restated(img, call)
    k = mc.element(call.elem)
    if call.entry == mc.X:
        run = lambda s: C.hal.morphologyEx(s, call.op, k, anchor=call.anchor, iterations=call.it, borderType=call.border, borderValue=call.bv)
    else:
        f = C.hal.erode if call.entry == mc.E else C.hal.dilate
        run = lambda s: f(s, k, anchor=call.anchor, iterations=call.it, borderType=call.border, borderValue=call.bv)
    assert_bits(run(img), want, excl, name + " (host)")
    other = (img[::-1] // 2).copy()
    got = run(np.stack([img, other]))
    assert_bits(got[0], want, excl, name + " (host batch, frame 0)")
    w1, e1 = mc.restated(other, call)
    assert_bits(got[1], w1, e1, name + " (host batch, frame 1)")


def test_cpp_gpumat_morphology(cvb, tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_morph_host")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "cpp", "test_morph_host.cpp"),
                        "-L" + os.path.join(root, "opencv_b200", "lib"), "-lb200cv", "-Wl,-rpath," + os.path.join(root, "opencv_b200", "lib")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
