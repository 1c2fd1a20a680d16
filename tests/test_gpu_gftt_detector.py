"""GPU: cv::GFTTDetector, the Feature2D wrapper over goodFeaturesToTrack (features2d/src/gftt.cpp:131-148).  It only composes calls that
tests/test_gpu_features.py verifies (cvtColor + goodFeaturesToTrack).

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_close, gpu

pytestmark = [pytest.mark.gpu]


def test_host_sobel_scharr_wrappers(cvb, oracle, rng):
    """opencv_b200.hal.Sobel / Scharr: numpy wrappers over b200cv_host_sobel (the call the HAL hook already makes)"""
    from opencv_b200 import hal
    from util import assert_exact
    batch = rng.integers(0, 256, (4, 240, 320, 1), dtype=np.uint8)
    sc = hal.Scharr(batch, 3, 1, 0)
    assert_exact(sc[3, :, :, 0], oracle.Sobel(batch[3, :, :, 0], 3, 1, 0, -1), "host Scharr")
    so = hal.Sobel(batch[0, :, :, 0].copy(), 5, 0, 1, 3, scale=0.5)
    want = oracle.Sobel(batch[0, :, :, 0], 5, 0, 1, 3, scale=0.5)
    assert np.abs(so - want).max() <= 1e-4


def test_gftt_detector(cvb, oracle, rng):
    small = rng.random((32, 42)).astype(np.float32)
    gray = (np.kron(small, np.ones((8, 8), np.float32)) * 255).astype(np.uint8)[:240, :320]
    det = C.GFTTDetector.create(200, 0.01, 5, 3, 3, True, 0.04)
    kp = det.detect(gpu(gray))
    want, wq = oracle.goodFeaturesToTrack(gray, 200, 0.01, 5, 3, 3, True, 0.04)
    assert kp.shape == (len(want), 4)
    assert np.array_equal(kp[:, :2], want) and (kp[:, 2] == 3).all()
    assert_close(kp[:, 3], wq, atol=5e-7 * float(np.abs(wq).max()), what="keypoint responses")
    bgr = np.stack([gray, gray, gray], axis=-1)
    kp3 = det.detect(gpu(bgr))                      # BGR2GRAY of an r = g = b image is the image itself
    assert np.array_equal(kp3[:, :2], kp[:, :2])
    det.setMaxFeatures(10)
    assert len(det.detect(gpu(gray))) == 10 and det.getMaxFeatures() == 10
