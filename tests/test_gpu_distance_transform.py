"""GPU: cv::distanceTransform (opencv_b200/csrc/distance.cu) bit for bit against the plain-C restatement (oracle/port/port_distance.c,
which tests/test_dist_reference.py holds to the reference's recorded answers) over the whole table of tests/dist_cases.py, floats compared
as int32 bits; then batches whose frames differ, padded views with guard bytes, the in-place 8-bit call, the refusals, the launch count,
the host path and the C++ GpuMat mirror."""
import os
import subprocess

import numpy as np
import pytest

import dist_cases as dc
import opencv_b200 as C
from util import cpu, gpu

pytestmark = [pytest.mark.gpu]


def bits(a):
    a = np.ascontiguousarray(a)
    return a if a.dtype == np.uint8 else a.view(np.int32)


def assert_bits(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, "%s: %s %s vs %s %s" % (what, got.shape, got.dtype, want.shape, want.dtype)
    bad = np.argwhere(bits(got) != bits(want))
    assert len(bad) == 0, "%s: %d/%d elements differ, first at %s (got %r want %r)" % (
        what, len(bad), got.size, tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])


def ported(img, call):
    depth, out = dc.run("port", img, call)
    assert depth >= 0
    return out


def _by_image(refused):
    groups = {}
    for c in dc.CASES:
        if (c.call in dc.REFUSED) == refused:
            groups.setdefault(c.image, []).append(c)
    return list(groups.values())


@pytest.mark.parametrize("cases", _by_image(False), ids=lambda cs: cs[0].image)
def test_case(cvb, port, cases):
    """every call the table makes on one image (one source upload, each result checked against the port)"""
    img = dc.image_of(cases[0])
    src = gpu(img)
    for case in cases:
        dt, mask, dst_type = dc.CALLS[case.call]
        got = cpu(cvb.distanceTransform(src, dt, mask, dstType=dst_type))
        assert_bits(got, ported(img, case.call), case.id)


@pytest.mark.parametrize("cases", _by_image(True), ids=lambda cs: cs[0].image)
def test_refused_case(cvb, port, cases):
    """the reference asserts on these arguments: an argument error, and the destination keeps its bytes"""
    img = dc.image_of(cases[0])
    src = gpu(img)
    for case in cases:
        dt, mask, dst_type = dc.CALLS[case.call]
        dst = gpu(np.full(img.shape, 7, np.uint8 if dc.out_is_u8(case.call) else np.float32))
        with pytest.raises(C.B200cvError) as e:
            cvb.distanceTransform(src, dt, mask, dst=dst, dstType=dst_type)
        assert not isinstance(e.value, C.NotImplementedOnDevice), case.id
        assert (cpu(dst) == 7).all(), case.id


@pytest.mark.parametrize("call", list(dc.MODES))
def test_batch_of_different_frames(cvb, port, call):
    """four frames of different content (no zero, sparse, edges, ties) with 3 spare rows after each in both buffers"""
    H, W = 45, 70
    fills = ("none", "sparse", "edges", "ties")
    frames = [dc.image_of(dc.Case("b", "b-%d-%s" % (i, f), (H, W), f, call)) for i, f in enumerate(fills)]
    u8 = dc.out_is_u8(call)
    sbig = np.full((4, H + 3, W, 1), 9, np.uint8)
    sbig[:, :H, :, 0] = np.stack(frames)
    dbig = gpu(np.full((4, H + 3, W, 1), 0x77 if u8 else 0.5, np.uint8 if u8 else np.float32))
    dt, mask, dst_type = dc.CALLS[call]
    cvb.distanceTransform(gpu(sbig)[:, :H], dt, mask, dst=dbig[:, :H], dstType=dst_type)
    out = cpu(dbig)
    for i, img in enumerate(frames):
        assert_bits(out[i, :H, :, 0], ported(img, call), "%s frame %d (%s)" % (call, i, fills[i]))
    assert (out[:, H:] == (0x77 if u8 else 0.5)).all(), "spare rows between frames were written"


@pytest.mark.parametrize("call", list(dc.MODES))
@pytest.mark.parametrize("shape", [(13, 11), (33, 65), (5, 4097)])
def test_views_with_guard_bytes(cvb, port, call, shape):
    """source and destination as windows into larger buffers with padded rows, the source 3 bytes and an 8-bit destination 5 bytes into
    their rows (a float destination 5 elements in); everything around the destination window must come back unchanged"""
    H, W = shape
    img = dc.image_of(dc.Case("v", "v-%dx%d" % shape, shape, "sparse", call))
    want = ported(img, call)
    u8 = dc.out_is_u8(call)
    sbig = np.full((H + 2, W + 9), 0, np.uint8)
    sbig[1:1 + H, 3:3 + W] = img
    src = gpu(sbig)[1:1 + H, 3:3 + W]
    if u8:
        dbig = gpu(np.full((H + 2, W + 7), 0xA5, np.uint8))
        dst = dbig[1:1 + H, 5:5 + W]
        cvb.distanceTransform(src, *dc.CALLS[call][:2], dst=dst, dstType=C.CV_8U)
        out = cpu(dbig)
        expect = np.full(out.shape, 0xA5, np.uint8)
        expect[1:1 + H, 5:5 + W] = want
    else:
        import torch
        plane = torch.full((H + 2, W + 7), -1.5, dtype=torch.float32, device="cuda")
        dst = plane[1:1 + H, 5:5 + W]
        cvb.distanceTransform(src, *dc.CALLS[call][:2], dst=dst, dstType=C.CV_32F)
        out = cpu(plane)
        expect = np.full(out.shape, -1.5, np.float32)
        expect[1:1 + H, 5:5 + W] = want
    assert_bits(out, expect, "%s %dx%d window and surroundings" % (call, H, W))


@pytest.mark.parametrize("mask", [0, 3, 5, 7])
def test_l1_u8_in_place(cvb, port, mask):
    """the 8-bit L1 call with dst = src (the reference allows it), whatever the mask"""
    img = dc.image_of(dc.BY_ID["64x96-edges-l1_u8"])
    t = gpu(img)
    out = cvb.distanceTransform(t, C.DIST_L1, mask, dst=t, dstType=C.CV_8U)
    assert out.data_ptr() == t.data_ptr()
    assert_bits(cpu(t), ported(img, "l1_u8"), "in place, mask %d" % mask)


def test_python_output_types(cvb):
    img = gpu(dc.image_of(dc.BY_ID["13x11-sparse-c3"]))
    assert cvb.distanceTransform(img, C.DIST_L1, 3, dstType=C.CV_8U).dtype == __import__("torch").uint8
    for dt in (C.DIST_L2, C.DIST_C):
        assert cvb.distanceTransform(img, dt, 3, dstType=C.CV_8U).dtype == __import__("torch").float32   # the reference gives 32F


def test_argument_errors_leave_dst_untouched(cvb):
    """src not 8UC1, a destination of the wrong type or size, and an 8UC1 destination with a type other than L1"""
    import torch
    img = gpu(dc.image_of(dc.BY_ID["13x11-sparse-c3"]))
    calls = [(img.to(torch.float32), torch.full((13, 11), 7.0, device="cuda"), C.DIST_L2, 3),
             (img, torch.full((13, 11), 7, dtype=torch.int16, device="cuda"), C.DIST_L2, 3),
             (img, torch.full((13, 12), 7.0, device="cuda"), C.DIST_L2, 0),
             (img, torch.full((13, 11), 7, dtype=torch.uint8, device="cuda"), C.DIST_C, 3),
             (img, torch.full((13, 11), 7, dtype=torch.uint8, device="cuda"), C.DIST_L2, 0)]
    for src, dst, dt, mask in calls:
        with pytest.raises(C.B200cvError) as e:
            cvb.distanceTransform(src, dt, mask, dst=dst)
        assert not isinstance(e.value, C.NotImplementedOnDevice)
        assert (cpu(dst) == 7).all(), (dt, mask, dst.dtype, tuple(dst.shape))


def test_launch_count_does_not_depend_on_content(cvb):
    import torch
    expect = {"c3": 1, "l1_3": 1, "l2_3": 1, "l2_5": 1, "precise": 2, "l1_u8": 1}
    for call, n in expect.items():
        for fill in ("none", "zero", "sparse", "edges"):
            for shape in ((40, 50), (3, 20000)):
                img = gpu(dc.image_of(dc.Case("n", "n-%s" % fill, shape, fill, call)))
                dt, mask, dst_type = dc.CALLS[call]
                torch.cuda.synchronize()
                n0 = cvb.launch_count()
                cvb.distanceTransform(img, dt, mask, dstType=dst_type)
                assert cvb.launch_count() - n0 == n, (call, fill, shape)


@pytest.mark.parametrize("case_id", ["64x96-ties-precise", "64x96-edges-l2_5", "120x257-lines-l1_u8", "31x17-ties-user_0", "7x9-none-c5",
                                     "2x19371-sparse-precise"])
def test_host_path(cvb, port, case_id):
    """opencv_b200.hal.distanceTransform on numpy arrays (b200cv_host_distance_transform), and a host batch of two frames"""
    case = dc.BY_ID[case_id]
    img = dc.image_of(case)
    dt, mask, dst_type = dc.CALLS[case.call]
    want = ported(img, case.call)
    assert_bits(cvb.distanceTransform(img, dt, mask, dstType=dst_type), want, case_id + " (host)")
    batch = np.empty((2,) + img.shape + (1,), np.uint8)
    batch[0, :, :, 0], batch[1, :, :, 0] = img, 255 - img
    got = C.hal.distanceTransform(batch, dt, mask, dstType=dst_type)
    assert_bits(got[0, :, :, 0], want, case_id + " (host batch, frame 0)")
    assert_bits(got[1, :, :, 0], ported(255 - img, case.call), case_id + " (host batch, frame 1)")


def test_host_l1_u8_in_place(cvb, port):
    img = dc.image_of(dc.BY_ID["64x96-sparse-l1_u8"])
    buf = img.copy()
    out = C.hal.distanceTransform(buf, C.DIST_L1, 3, dst=buf, dstType=C.CV_8U)
    assert out is buf
    assert_bits(buf, ported(img, "l1_u8"), "host, in place")


def test_cpp_gpumat_distance_transform(cvb, tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_dist_host")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "cpp", "test_dist_host.cpp"),
                        "-L" + os.path.join(root, "opencv_b200", "lib"), "-lb200cv", "-Wl,-rpath," + os.path.join(root, "opencv_b200", "lib")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
