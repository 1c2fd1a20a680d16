"""GPU: the tensor-core filter2D kernels' tile schedule against the direct-sum kernels.

8-bit filter2D from 130 taps on runs filter2d_tc.cu: 16-column tiles for kernels at most 17 taps wide, 32-column tiles above, 128-row
tiles that the CTA's two consumer warpgroups take in turns.  Float filter2D from 14 kernel rows on runs filter2d_tc_f32.cu: 256-row
strips shared by both warpgroups, the second one a few kernel rows behind.  The shapes below give tile counts that are odd, below and
above the SM count (so CTAs have one, two or several tiles, and some warpgroups none), heights that are not multiples of the tile
height, widths that are not multiples of the tile width, one frame and several, and destinations whose rows are not 16-byte aligned.
Bars: 1 LSB for 8-bit destinations (exact integer sums; only .5 ties may round differently), the direct sum's own accuracy elsewhere.
These compare two device paths; tests/test_gpu_filter2d_tc_exact.py holds the tensor-core kernels to an exact restatement of their
arithmetic (tests/f2d_reference.py), bit for bit for 8-bit sources.
"""
import numpy as np
import pytest
import torch

from util import assert_close, cpu, gpu

pytestmark = pytest.mark.gpu

# (frames, rows, cols): 7 tiles on one frame; ragged multi-frame; several tiles per CTA for either tile width
SHAPES = [(1, 100, 107), (3, 301, 263), (2, 1000, 900)]


def _kernel(rng, kh, kw):
    ker = rng.random((kh, kw)).astype(np.float32) - 0.25
    return ker / (np.abs(ker).sum() * 0.5)


def _run(cvb, monkeypatch, img, ddepth, ker, anchor, delta, border, direct, dst=None):
    if direct:
        monkeypatch.setenv("B200CV_FILTER2D_PATH", "direct")
    try:
        n0 = cvb.launch_count()
        out = cvb.filter2D(img, ddepth, ker, anchor=anchor, delta=delta, borderType=border, dst=dst)
        torch.cuda.synchronize()
        return cpu(out), cvb.launch_count() - n0
    finally:
        if direct:
            monkeypatch.delenv("B200CV_FILTER2D_PATH")


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("kw", [17, 19])            # both sides of the 16 / 32-column switch
@pytest.mark.parametrize("ddepth", [-1, 3, 5])      # 8U, 16S, 32F
def test_filter2d_u8_tc_schedule(cvb, rng, monkeypatch, shape, kw, ddepth):
    n, h, w = shape
    img = gpu(rng.integers(0, 256, (n, h, w, 1), dtype=np.uint8))
    ker = _kernel(rng, 13, kw) * (64 if ddepth == 3 else 1)
    anchor, delta = (kw // 3, 4), 1.5
    for border in (0, 4):
        got, l_tc = _run(cvb, monkeypatch, img, ddepth, ker, anchor, delta, border, False)
        want, l_direct = _run(cvb, monkeypatch, img, ddepth, ker, anchor, delta, border, True)
        assert l_tc != l_direct, "the tensor-core path did not run"
        what = "filter2D u8 tc vs direct %s kw=%d dd=%d b=%d" % (shape, kw, ddepth, border)
        if ddepth == 5:
            assert_close(got, want, atol=2e-3, rtol=1e-5, what=what)
        else:
            assert_close(got, want, atol=1, what=what)
        if ddepth == -1:    # 16S: 64x larger sums, where the direct float sum's own rounding flips more results by 1
            assert (got != want).mean() < 1e-3, what + ": more than .5 ties differ"


@pytest.mark.parametrize("ddepth", [-1, 3, 5])
def test_filter2d_u8_tc_unaligned_dst(cvb, rng, monkeypatch, ddepth):
    """destination rows that are not 16-byte aligned (a column window of a wider buffer) take element stores"""
    n, h, w = 2, 301, 263
    img = gpu(rng.integers(0, 256, (n, h, w, 1), dtype=np.uint8))
    ker = _kernel(rng, 13, 15) * (64 if ddepth == 3 else 1)
    dt = {-1: torch.uint8, 3: torch.int16, 5: torch.float32}[ddepth]
    base = torch.zeros((n, h, w + 5, 1), dtype=dt, device="cuda")
    got, _ = _run(cvb, monkeypatch, img, ddepth, ker, (-1, -1), 0.0, 4, False, dst=base[:, :, 1:w + 1])
    want, _ = _run(cvb, monkeypatch, img, ddepth, ker, (-1, -1), 0.0, 4, True)
    assert_close(got, want, atol=2e-3 if ddepth == 5 else 1, rtol=1e-5 if ddepth == 5 else 0, what="filter2D u8 tc unaligned dst dd=%d" % ddepth)
    rest = cpu(base)
    assert not rest[:, :, 0].any() and not rest[:, :, w + 1:].any(), "stores outside the destination window"


@pytest.mark.parametrize("shape", SHAPES + [(3, 1000, 900)])
@pytest.mark.parametrize("khw", [(15, 15), (21, 21), (31, 31), (14, 11)])
def test_filter2d_f32_tc_schedule(cvb, rng, monkeypatch, shape, khw):
    n, h, w = shape
    kh, kw = khw
    img = gpu(((rng.random((n, h, w, 1)) - 0.3) * 300).astype(np.float32))
    ker = _kernel(rng, kh, kw)
    for border in (0, 4):
        got, l_tc = _run(cvb, monkeypatch, img, -1, ker, (-1, -1), 0.25, border, False)
        want, l_direct = _run(cvb, monkeypatch, img, -1, ker, (-1, -1), 0.25, border, True)
        assert l_tc != l_direct, "the tensor-core path did not run"
        scale = float(np.abs(want).max())
        what = "filter2D f32 tc vs direct %s %dx%d b=%d" % (shape, kh, kw, border)
        assert_close(got, want, atol=1e-4 * scale, what=what)
        assert float(np.abs(got - want).mean()) <= 1e-5 * scale, what + ": mean error"


def test_filter2d_f32_tc_unaligned_dst(cvb, rng, monkeypatch):
    n, h, w = 2, 301, 263
    img = gpu(((rng.random((n, h, w, 1)) - 0.3) * 300).astype(np.float32))
    ker = _kernel(rng, 21, 21)
    base = torch.zeros((n, h, w + 5, 1), dtype=torch.float32, device="cuda")
    got, _ = _run(cvb, monkeypatch, img, -1, ker, (-1, -1), 0.0, 4, False, dst=base[:, :, 1:w + 1])
    want, _ = _run(cvb, monkeypatch, img, -1, ker, (-1, -1), 0.0, 4, True)
    assert_close(got, want, atol=1e-4 * float(np.abs(want).max()), what="filter2D f32 tc unaligned dst")
    rest = cpu(base)
    assert not rest[:, :, 0].any() and not rest[:, :, w + 1:].any(), "stores outside the destination window"


@pytest.mark.parametrize("kh", [1, 2, 5])
def test_filter2d_tc_few_kernel_rows(cvb, rng, monkeypatch, kh):
    """fewer kernel rows than the float kernel's warpgroup lag, and 8-bit tiles with almost no MMAs: the tensor-core paths forced on
    below their usual switch points"""
    monkeypatch.setenv("B200CV_FILTER2D_TC_MIN_TAPS", "1")
    n, h, w = 2, 1000, 900
    imf = gpu(((rng.random((n, h, w, 1)) - 0.3) * 300).astype(np.float32))
    ker = _kernel(rng, kh, 7)
    got, l_tc = _run(cvb, monkeypatch, imf, -1, ker, (-1, -1), 0.0, 4, False)
    want, l_direct = _run(cvb, monkeypatch, imf, -1, ker, (-1, -1), 0.0, 4, True)
    assert l_tc != l_direct, "the tensor-core path did not run"
    assert_close(got, want, atol=1e-4 * float(np.abs(want).max()), what="filter2D f32 tc %dx7" % kh)
    imu = gpu(rng.integers(0, 256, (n, h, w, 1), dtype=np.uint8))
    for kw in (17, 19):
        ker = _kernel(rng, kh, kw)
        got, l_tc = _run(cvb, monkeypatch, imu, -1, ker, (-1, -1), 0.0, 4, False)
        want, l_direct = _run(cvb, monkeypatch, imu, -1, ker, (-1, -1), 0.0, 4, True)
        assert l_tc != l_direct, "the tensor-core path did not run"
        assert_close(got, want, atol=1, what="filter2D u8 tc %dx%d" % (kh, kw))
