"""GPU parity: cv::resize INTER_LINEAR_EXACT (8-bit, 8.8 fixed point) and INTER_NEAREST_EXACT (16.16 pixel-centre coordinates): BIT-EXACT.

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]

CASES = [((120, 180), (40, 60)), ((120, 180), (60, 90)), ((121, 183), (40, 61)), ((100, 150), (237, 341)), ((480, 640), (300, 400)),
         ((97, 131), (96, 130)), ((64, 64), (160, 160)), ((1, 47), (5, 90)), ((50, 1), (49, 23)), ((33, 47), (1, 1)), ((300, 400), (7, 399)),
         ((2, 2), (9, 9)), ((3, 5), (30, 50))]


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("ssize,dsize", CASES)
def test_exact_resizers(cvb, oracle, rng, ssize, dsize, cn):
    (sh, sw), (dh, dw) = ssize, dsize
    shape = (sh, sw) if cn == 1 else (sh, sw, cn)
    for img in (rng.integers(0, 256, shape, dtype=np.uint8), (rng.random(shape, dtype=np.float32) * 255).astype(np.float32)):
        for interp in (C.INTER_LINEAR_EXACT, C.INTER_NEAREST_EXACT):
            got = cpu(cvb.resize(gpu(img), (dw, dh), interpolation=interp))
            assert_exact(got, oracle.resize(img, (dw, dh), interp), "interp %d %s %s -> %s cn=%d" % (interp, img.dtype, ssize, dsize, cn))


def test_reference_goldens(cvb):
    """Resize_Bitexact.Nearest8U (test_resize_bitexact.cpp:190-241) and the Imgproc_resize_area rounding regressions (test_imgwarp.cpp:1285-1317)"""
    from test_oracle import resize_golden_cases
    for src, dsize, interp, want, tol in resize_golden_cases():
        got = cpu(cvb.resize(gpu(src), dsize, interpolation=interp))
        assert np.abs(got.astype(int) - want.astype(int)).max() <= tol, "interp %d %s -> %s" % (interp, src.shape, dsize)


def test_exact_resizers_8k(cvb, ref, rng):
    """bench.py workload c3 geometry: 7680x4320 8UC3 -> 5120x2880 and 3840x2160 (LINEAR_EXACT 2 x 2 = the area fast path)"""
    img = rng.integers(0, 256, (4320, 7680, 3), dtype=np.uint8)
    for dsize in ((5120, 2880), (3840, 2160)):
        for interp in (C.INTER_LINEAR_EXACT, C.INTER_NEAREST_EXACT):
            assert_exact(cpu(cvb.resize(gpu(img), dsize, interpolation=interp)), ref.resize(img, dsize, interp), "8K -> %s interp %d" % (dsize, interp))
