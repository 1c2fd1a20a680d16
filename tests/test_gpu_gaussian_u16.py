"""GPU parity: cv::GaussianBlur on CV_16U images (16.16 fixed point): BIT-EXACT.

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("shape", [(37, 53), (64, 96, 3), (20, 31, 4), (1, 40), (33, 1), (480, 640)])
def test_gaussian_u16(cvb, oracle, rng, shape):
    img = rng.integers(0, 65536, shape, dtype=np.uint16)
    ext = np.where(rng.random(shape) < 0.5, 0, 65535).astype(np.uint16)
    for im in (img, ext):
        for k, s in [(3, 0), (5, 0), (7, 1.5), (9, 0), (15, 3.0), (0, 1.2), (31, 0), (5, 0.3)]:
            for border in (4, 1, 0, 2, 3):
                got = cpu(cvb.GaussianBlur(gpu(im), (k, k), s, s, border))
                assert_exact(got, oracle.GaussianBlur(im, (k, k), s, s, border), "GaussianBlur u16 %s k=%d s=%g border=%d" % (shape, k, s, border))


def test_gaussian_u16_4k_batch(cvb, ref, rng):
    batch = rng.integers(0, 65536, (4, 2160, 3840, 1), dtype=np.uint16)
    out = cpu(cvb.GaussianBlur(gpu(batch), (5, 5), 0))
    assert_exact(out[3, :, :, 0], ref.GaussianBlur(batch[3, :, :, 0], (5, 5), 0, 0, 4), "GaussianBlur u16 4K frame 3")


def test_gaussian_u16_first_version_still_agrees(cvb, oracle, rng, monkeypatch):
    """B200CV_GAUSS_U16_PATH=v1: the direct kw x kh window kernel (the one the host emulation runs) against the separable tiled kernel"""
    img = rng.integers(0, 65536, (2, 131, 157, 3), dtype=np.uint16)
    for k, s, border in ((5, 0, 4), (9, 2.0, 2), (31, 0, 3)):
        v2 = cpu(cvb.GaussianBlur(gpu(img), (k, k), s, s, border))
        monkeypatch.setenv("B200CV_GAUSS_U16_PATH", "v1")
        v1 = cpu(cvb.GaussianBlur(gpu(img), (k, k), s, s, border))
        monkeypatch.delenv("B200CV_GAUSS_U16_PATH")
        assert_exact(v2, v1, "GaussianBlur u16 separable vs direct k=%d border=%d" % (k, border))
