"""GPU: cv::Laplacian (opencv_b200/csrc/laplacian.cu) bit for bit against the plain-C restatement (port_laplacian in
oracle/port/port_laplacian.c, which tests/test_laplacian_reference.py holds to the reference's recorded answers) over the whole table of
tests/laplacian_cases.py, floats compared as int32 bits with any NaN equal to any NaN; then padded views with guard bytes, batches
with spare rows, the launch count, the refusals, the host path, the C++ GpuMat mirror and a HAL-built reference."""
import os
import subprocess

import numpy as np
import pytest

import laplacian_cases as lc
import opencv_b200 as C
from util import cpu, gpu

pytestmark = [pytest.mark.gpu]


def assert_same(got, want, what):
    got = np.asarray(got)
    assert got.shape == want.shape and got.dtype == want.dtype, "%s: %s %s vs %s %s" % (what, got.shape, got.dtype, want.shape, want.dtype)
    if not lc.same_bits(got, want):
        gn, wn = np.isnan(got.astype(np.float32)), np.isnan(want.astype(np.float32))
        g = got.view(np.int32) if got.dtype == np.float32 else got
        w = want.view(np.int32) if want.dtype == np.float32 else want
        bad = np.argwhere((g != w) & ~(gn & wn))
        raise AssertionError("%s: %d/%d elements differ, first at %s (got %r want %r)" % (
            what, len(bad), got.size, tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])]))


def ported(port, img, ddepth, ksize, scale, delta, border):
    out = lc.run("port", img, ddepth, ksize, scale, delta, border)
    assert out is not None
    return out


def _by_image():
    groups = {}
    for c in lc.CASES:
        if c.ddepth >= 0:
            groups.setdefault(c.image.id, []).append(c)
    return list(groups.values())


@pytest.mark.parametrize("cases", _by_image(), ids=lambda cs: cs[0].image.id)
def test_case(cvb, port, cases):
    """every call the table makes on one image (one source upload, each result checked against the port)"""
    img = lc.image_of(cases[0].image)
    src = gpu(img)
    reach = None
    if img.dtype == np.float32:
        # ksize 1 / 3 run the filter2D dispatch, which multiplies the 3x3 kernel's zero taps too: a non-finite pixel makes the outputs
        # around it NaN, where the reference skips those taps.  Those outputs (every 3x3 window holding one) are left out here.
        bad = ~np.isfinite(img.reshape(img.shape[0], img.shape[1], -1)).all(axis=2)
        pad = np.pad(bad, 1, mode="edge")
        reach = np.zeros_like(bad)
        for dy in (0, 1, 2):
            for dx in (0, 1, 2):
                reach |= pad[dy:dy + bad.shape[0], dx:dx + bad.shape[1]]
    for c in cases:
        got = cpu(cvb.Laplacian(src, c.ddepth, c.ksize, c.scale, c.delta, c.border))
        want = ported(port, img, c.ddepth, c.ksize, c.scale, c.delta, c.border)
        if reach is not None and c.ksize <= 3 and reach.any():
            got, want = got.copy(), want.copy()
            got[reach] = 0
            want[reach] = 0
        assert_same(got, want, c.id)


def test_refused_ksize_leaves_dst_untouched(cvb):
    """even, zero, negative and 33 apertures: an argument error (the reference asserts), and dst keeps its bytes"""
    src = gpu(np.arange(7 * 9, dtype=np.uint8).reshape(7, 9))
    for k in lc.BAD_KSIZES:
        dst = gpu(np.full((7, 9), 7, np.int16))
        with pytest.raises(C.B200cvError) as e:
            cvb.Laplacian(src, lc.CV_16S, k, dst=dst)
        assert not isinstance(e.value, C.NotImplementedOnDevice), k
        assert (cpu(dst) == 7).all(), k


def test_unsupported_calls_leave_dst_untouched(cvb):
    """BORDER_WRAP, a 16U source, a 64F destination, 16S -> 16S and src == dst: refused, dst unchanged"""
    import torch
    u8 = gpu(np.arange(11 * 13, dtype=np.uint8).reshape(11, 13))
    for k in (1, 3, 5, 7):
        dst = gpu(np.full((11, 13), 7, np.int16))
        with pytest.raises(C.NotImplementedOnDevice):
            cvb.Laplacian(u8, lc.CV_16S, k, borderType=3, dst=dst)
        assert (cpu(dst) == 7).all(), ("wrap", k)
        dst = torch.full((11, 13), 7, dtype=torch.float32, device="cuda")
        with pytest.raises(C.NotImplementedOnDevice):
            cvb.Laplacian(u8.to(torch.int32).to(torch.uint16), lc.CV_32F, k, dst=dst)
        assert (cpu(dst) == 7).all(), ("16U", k)
        dst = torch.full((11, 13), 7, dtype=torch.float64, device="cuda")
        with pytest.raises(C.NotImplementedOnDevice):
            cvb.Laplacian(u8, 6, k, dst=dst)
        assert (cpu(dst) == 7).all(), ("64F", k)
        s16 = u8.to(torch.int16)
        dst = torch.full((11, 13), 7, dtype=torch.int16, device="cuda")
        with pytest.raises(C.NotImplementedOnDevice):
            cvb.Laplacian(s16, -1, k, dst=dst)
        assert (cpu(dst) == 7).all(), ("16S", k)
        f = u8.to(torch.float32)
        with pytest.raises(C.B200cvError, match="in-place"):
            cvb.Laplacian(f, -1, k, dst=f)


@pytest.mark.parametrize("ksize", [1, 5, 7, 31])
@pytest.mark.parametrize("pair", lc.PAIRS, ids=lambda p: "%d-%d" % p)
def test_views_with_guard_bytes(cvb, port, ksize, pair):
    """source and destination as windows into larger buffers with padded rows, 3 and 5 elements into their rows (odd byte offsets for
    8-bit data); everything around the destination window must come back unchanged"""
    import torch
    sd, dd = pair
    H, W, cn = 37, 45, 3
    img = lc.image_of(lc.Image("view-%d" % sd, (H, W), cn, sd, "random"))
    want = ported(port, img, dd, ksize, 0.5, 0.5, 1)
    sbig = np.zeros((H + 2, W + 9, cn), lc.NP[sd])
    sbig[1:1 + H, 3:3 + W] = img
    src = gpu(sbig)[1:1 + H, 3:3 + W]
    guard = {lc.CV_8U: 0xA5, lc.CV_16S: -1234, lc.CV_32F: -1.5}[dd]
    dbig = gpu(np.full((H + 2, W + 7, cn), guard, lc.NP[dd]))
    dst = dbig[1:1 + H, 5:5 + W]
    cvb.Laplacian(src, dd, ksize, 0.5, 0.5, 1, dst=dst)
    torch.cuda.synchronize()
    out = cpu(dbig)
    expect = np.full(out.shape, guard, lc.NP[dd])
    expect[1:1 + H, 5:5 + W] = want
    assert_same(out, expect, "k=%d %d->%d window and surroundings" % (ksize, sd, dd))


@pytest.mark.parametrize("ksize", [3, 5, 9])
@pytest.mark.parametrize("pair", [(lc.CV_8U, lc.CV_16S), (lc.CV_32F, lc.CV_32F)], ids=["8u-16s", "32f-32f"])
def test_batch_with_spare_rows(cvb, port, ksize, pair):
    """four frames of different content with 3 spare rows after each in both buffers: each frame is its own image, and one launch
    serves the batch from ksize 5 on"""
    import torch
    sd, dd = pair
    H, W = 41, 67
    frames = [lc.image_of(lc.Image("batch-%d-%d" % (sd, i), (H, W), 1, sd, f)) for i, f in enumerate(("random", "impulse", "checker", "const"))]
    sbig = np.zeros((4, H + 3, W, 1), lc.NP[sd])
    sbig[:, :H, :, 0] = np.stack(frames)
    dbig = gpu(np.full((4, H + 3, W, 1), 77, lc.NP[dd]))
    torch.cuda.synchronize()
    n0 = cvb.launch_count()
    cvb.Laplacian(gpu(sbig)[:, :H], dd, ksize, 1.0, 0.0, 4, dst=dbig[:, :H])
    if ksize >= 5:
        assert cvb.launch_count() - n0 == 1
    out = cpu(dbig)
    for i, img in enumerate(frames):
        assert_same(out[i, :H, :, 0], ported(port, img, dd, ksize, 1.0, 0.0, 4), "k=%d frame %d" % (ksize, i))
    assert (out[:, H:] == 77).all(), "spare rows between frames were written"


def test_one_launch_per_call_from_ksize_5(cvb):
    import torch
    for sd, dd in lc.PAIRS:
        for cn in (1, 4):
            img = gpu(lc.image_of(lc.Image("n-%d-%d" % (sd, cn), (64, 300), cn, sd, "random")))
            for k in (5, 7, 15, 31):
                torch.cuda.synchronize()
                n0 = cvb.launch_count()
                cvb.Laplacian(img, dd, k, 2.0, 1.0)
                assert cvb.launch_count() - n0 == 1, (sd, dd, cn, k)


@pytest.mark.parametrize("ksize", [1, 3, 5, 9])
def test_host_path(cvb, port, ksize):
    """opencv_b200.hal.Laplacian on numpy arrays (b200cv_host_laplacian), one image and a host batch of two frames"""
    img = lc.image_of(lc.Image("host", (53, 61), 2, lc.CV_8U, "random"))
    want = ported(port, img, lc.CV_16S, ksize, 1.0, 0.0, 4)
    assert_same(cvb.Laplacian(img, lc.CV_16S, ksize), want, "host k=%d" % ksize)
    batch = np.stack([img, 255 - img])
    got = C.hal.Laplacian(batch, lc.CV_16S, ksize)
    assert_same(got[0], want, "host batch frame 0, k=%d" % ksize)
    assert_same(got[1], ported(port, 255 - img, lc.CV_16S, ksize, 1.0, 0.0, 4), "host batch frame 1, k=%d" % ksize)


def test_cpp_gpumat_laplacian(cvb, tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_laplacian_host")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "cpp", "test_laplacian_host.cpp"),
                        "-L" + os.path.join(root, "opencv_b200", "lib"), "-lb200cv", "-Wl,-rpath," + os.path.join(root, "opencv_b200", "lib")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


def test_hal_built_reference_sends_ksize_3_here(cvb):
    """the reference built with hal/b200cv_hal_replacement.hpp: cv::Laplacian ksize 3 goes through filter2D's HAL hook, reaches the
    device and returns the stock reference's bytes"""
    if not (lc.ref_available("ref") and lc.ref_available("ref_hal")):
        pytest.skip("liblapref.so / liblapref_hal.so not built (tools/build_laplacian_ref.py with the HAL-built reference)")
    for sd, dd in lc.PAIRS:
        img = lc.image_of(lc.Image("hal-%d" % sd, (240, 320), 1, sd, "random"))
        n0 = cvb.launch_count()
        out = lc.run("ref_hal", img, dd, 3, 0.5, 2.0, 4)
        assert out is not None
        assert cvb.launch_count() > n0, "cv::Laplacian ksize 3 did not reach the device (%d -> %d)" % (sd, dd)
        assert_same(out, lc.run("ref", img, dd, 3, 0.5, 2.0, 4), "cv::Laplacian ksize 3 via the HAL, %d -> %d" % (sd, dd))
