"""GPU parity: cv::integral, 8UC1 -> 32S sum (+ 64F sum of squares): BIT-EXACT (integers; the doubles hold integers below 2^53).

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("size", [(1, 1), (5, 7), (17, 15), (33, 65), (240, 321), (1080, 1920), (2160, 3840)])
def test_integral(cvb, oracle, rng, size):
    img = rng.integers(0, 256, size, dtype=np.uint8)
    ws, wq = oracle.integral(img, True)
    gs, gq = cvb.integral(gpu(img), with_sqsum=True)
    assert_exact(cpu(gs), ws, "integral sum %s" % (size,))
    assert_exact(cpu(gq), wq, "integral sqsum %s" % (size,))
    assert_exact(cpu(cvb.integral(gpu(img))), ws, "integral sum only %s" % (size,))


def test_integral_batch_host_and_hal(cvb, oracle, rng):
    batch = rng.integers(0, 256, (6, 480, 640, 1), dtype=np.uint8)
    out = cpu(cvb.integral(gpu(batch)))
    assert out.shape == (6, 481, 641, 1)
    for f in (0, 5):
        assert_exact(out[f, :, :, 0], oracle.integral(batch[f, :, :, 0]), "integral batch frame %d" % f)
    from opencv_b200 import hal
    img = batch[2, :, :, 0].copy()
    hs, hq = hal.integral(img, True)
    ws, wq = oracle.integral(img, True)
    assert_exact(hs, ws, "host integral sum"); assert_exact(hq, wq, "host integral sqsum")
    from oracle.api import Oracle, available
    if available("ref_hal") and Oracle("ref_hal").has("integral"):
        n0 = cvb.launch_count()
        rs, rq = Oracle("ref_hal").integral(img, True)
        assert_exact(rs, ws, "cv::integral via HAL"); assert_exact(rq, wq, "cv::integral sqsum via HAL")
        assert cvb.launch_count() > n0, "cv::integral did not reach the B200 HAL"
    # size-independent property: any box sum from four corners of the integral equals the direct sum
    s = ws.astype(np.int64)
    assert s[300, 400] - s[100, 400] - s[300, 200] + s[100, 200] == int(img[100:300, 200:400].sum(dtype=np.int64))


def test_integral_first_version_still_agrees(cvb, oracle, rng, monkeypatch):
    """B200CV_INTEGRAL_PATH=v1: the six map-only kernels (the ones the host emulation runs) against the warp-scan kernels and the oracle"""
    img = rng.integers(0, 256, (3, 333, 517, 1), dtype=np.uint8)
    s2, q2 = cvb.integral(gpu(img), with_sqsum=True)
    monkeypatch.setenv("B200CV_INTEGRAL_PATH", "v1")
    s1, q1 = cvb.integral(gpu(img), with_sqsum=True)
    monkeypatch.delenv("B200CV_INTEGRAL_PATH")
    assert_exact(cpu(s2), cpu(s1), "integral sum: scan kernels vs map-only kernels")
    assert_exact(cpu(q2), cpu(q1), "integral sqsum: scan kernels vs map-only kernels")
    assert_exact(cpu(s2)[1, :, :, 0], oracle.integral(img[1, :, :, 0]), "integral sum vs oracle")
