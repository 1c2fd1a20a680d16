"""GPU parity: cv::resize INTER_AREA in its true area mode (both factors >= 1), integer and fractional factors, 8-bit and float: BIT-EXACT.

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]

CASES = [((120, 180), (40, 60)), ((120, 180), (30, 90)), ((121, 183), (40, 61)), ((100, 150), (37, 41)), ((480, 640), (300, 400)),
         ((97, 131), (96, 130)), ((64, 64), (16, 16)), ((90, 120), (30, 24)), ((50, 70), (49, 23)), ((33, 47), (1, 1)), ((300, 400), (7, 399))]


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("ssize,dsize", CASES)
def test_area_resize(cvb, oracle, rng, ssize, dsize, cn):
    (sh, sw), (dh, dw) = ssize, dsize
    shape = (sh, sw) if cn == 1 else (sh, sw, cn)
    for img in (rng.integers(0, 256, shape, dtype=np.uint8), (rng.random(shape, dtype=np.float32) * 255).astype(np.float32)):
        got = cpu(cvb.resize(gpu(img), (dw, dh), interpolation=C.INTER_AREA))
        assert_exact(got, oracle.resize(img, (dw, dh), 3), "INTER_AREA %s %s -> %s cn=%d" % (img.dtype, ssize, dsize, cn))


def test_area_resize_8k_batch(cvb, ref, rng):
    """bench.py workload c3 geometry with INTER_AREA: 4 frames 7680x4320 8UC3 -> 5120x2880 (factor 1.5) and -> 2560x1440 (factor 3) in one launch each"""
    base = rng.integers(0, 256, (4320, 7680, 3), dtype=np.uint8)
    batch = np.stack([np.roll(base, 11 * i, axis=1) for i in range(2)])
    for dsize in ((5120, 2880), (2560, 1440)):
        out = cpu(cvb.resize(gpu(batch), dsize, interpolation=C.INTER_AREA))
        assert_exact(out[1], ref.resize(batch[1], dsize, 3), "INTER_AREA 8K -> %s" % (dsize,))


@pytest.mark.parametrize("ssize,dsize", [((40, 60), (120, 180)), ((40, 60), (97, 131)), ((100, 150), (237, 341)), ((97, 131), (98, 132)), ((64, 64), (160, 32)),
                                         ((64, 64), (32, 160)), ((1, 47), (5, 90)), ((50, 1), (75, 23)), ((3, 5), (30, 50)), ((120, 160), (121, 100))])
def test_area_resize_with_an_enlarging_axis(cvb, oracle, rng, ssize, dsize):
    """INTER_AREA with a factor < 1 on either axis = the bilinear kernel with area-mode weights on both axes (resize.cpp:4104-4109, :4158-4163)"""
    (sh, sw), (dh, dw) = ssize, dsize
    for cn in (1, 3, 4):
        shape = (sh, sw) if cn == 1 else (sh, sw, cn)
        for img in (rng.integers(0, 256, shape, dtype=np.uint8), (rng.random(shape, dtype=np.float32) * 255).astype(np.float32)):
            got = cpu(cvb.resize(gpu(img), (dw, dh), interpolation=C.INTER_AREA))
            assert_exact(got, oracle.resize(img, (dw, dh), 3), "INTER_AREA %s %s -> %s cn=%d" % (img.dtype, ssize, dsize, cn))
