"""GPU parity: cv::cvtColor BGR / RGB <-> Lab (sRGB and linear) and <-> CIE XYZ, 8-bit: BIT-EXACT on the whole 2^24 colour cube.

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]
CODES = [C.COLOR_BGR2XYZ, C.COLOR_RGB2XYZ, C.COLOR_XYZ2BGR, C.COLOR_XYZ2RGB, C.COLOR_BGR2Lab, C.COLOR_RGB2Lab, C.COLOR_LBGR2Lab, C.COLOR_LRGB2Lab, C.COLOR_Lab2BGR, C.COLOR_Lab2RGB, C.COLOR_Lab2LBGR, C.COLOR_Lab2LRGB]


@pytest.mark.parametrize("code", CODES)
def test_lab_whole_colour_cube(cvb, oracle, code):
    v = np.arange(1 << 24, dtype=np.uint32)
    cube = np.stack([v & 255, (v >> 8) & 255, (v >> 16) & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)
    assert_exact(cpu(cvb.cvtColor(gpu(cube), code)), oracle.cvtColorLab(cube, code), "Lab code %d on 2^24 colours" % code)


def test_lab_channels_batches_and_hal(cvb, oracle, rng):
    bgra = rng.integers(0, 256, (240, 322, 4), dtype=np.uint8)
    assert_exact(cpu(cvb.cvtColor(gpu(bgra), C.COLOR_BGR2Lab)), oracle.cvtColorLab(np.ascontiguousarray(bgra[:, :, :3]), C.COLOR_BGR2Lab), "BGRA -> Lab")
    lab = rng.integers(0, 256, (3, 240, 322, 3), dtype=np.uint8)
    out = cpu(cvb.cvtColor(gpu(lab), C.COLOR_Lab2BGR, 4))
    assert out.shape == (3, 240, 322, 4) and (out[..., 3] == 255).all()
    assert_exact(out[2, :, :, :3], oracle.cvtColorLab(lab[2], C.COLOR_Lab2BGR), "Lab -> BGRA batch frame 2")
    from oracle.api import Oracle, available
    if available("ref_hal") and available("ref"):
        rh, ref = Oracle("ref_hal"), Oracle("ref")
        img = np.ascontiguousarray(bgra[:, :, :3])
        n0 = cvb.launch_count()
        for code in (C.COLOR_BGR2Lab, C.COLOR_LRGB2Lab, C.COLOR_Lab2RGB):
            assert_exact(rh.cvtColor(img, code, 3), ref.cvtColor(img, code, 3), "cv::cvtColor Lab code %d via HAL" % code)
        assert cvb.launch_count() - n0 >= 3, "cv::cvtColor(Lab) did not reach the B200 HAL"
