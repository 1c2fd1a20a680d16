"""GPU parity: cvtColor through the device C ABI.  Everything integer is BIT-EXACT, and so is HSV->BGR because the
kernel reproduces the reference's AVX2 vector-body / scalar-tail split.  Known-answer hashes are the reference's own
(modules/imgproc/test/test_color.cpp:2847-2855) on its RNG(0) 263x255 input, committed as tests/golden/cvtcolor_kat_input.npy."""
import os
import zlib

import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu, rand_u8

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")

KAT = {C.COLOR_RGB2GRAY: 0x416bd44a, C.COLOR_BGR2GRAY: 0x3008c6b8, C.COLOR_BGR2YUV: 0xc2cbcfda, C.COLOR_RGB2YUV: 0x4e98e757,
       C.COLOR_YUV2BGR: 0xb2c62a3f, C.COLOR_YUV2RGB: 0x6d242a3f}


@pytest.mark.parametrize("code", sorted(KAT))
def test_known_answer_hashes(cvb, code):
    img = np.load(os.path.join(GOLD, "cvtcolor_kat_input.npy"))
    out = cpu(cvb.cvtColor(gpu(img), code))
    assert zlib.adler32(np.ascontiguousarray(out).tobytes()) == KAT[code]


CODES3 = [(C.COLOR_BGR2GRAY, 1), (C.COLOR_RGB2GRAY, 1), (C.COLOR_BGR2YUV, 3), (C.COLOR_RGB2YUV, 3), (C.COLOR_BGR2YCrCb, 3),
          (C.COLOR_RGB2YCrCb, 3), (C.COLOR_BGR2HSV, 3), (C.COLOR_RGB2HSV, 3), (C.COLOR_BGR2HSV_FULL, 3), (C.COLOR_RGB2HSV_FULL, 3),
          (C.COLOR_BGR2RGB, 3), (C.COLOR_BGR2BGRA, 4), (C.COLOR_BGR2RGBA, 4),
          (C.COLOR_YUV2BGR, 3), (C.COLOR_YUV2RGB, 3), (C.COLOR_YCrCb2BGR, 3), (C.COLOR_YCrCb2RGB, 3),
          (C.COLOR_HSV2BGR, 3), (C.COLOR_HSV2RGB, 3), (C.COLOR_HSV2BGR_FULL, 3), (C.COLOR_HSV2RGB_FULL, 3),
          (C.COLOR_YUV2BGR, 4), (C.COLOR_HSV2BGR, 4), (C.COLOR_YCrCb2RGB, 4)]


@pytest.mark.parametrize("shape", [(255, 263), (64, 1024), (37, 31), (1, 1), (480, 640)])
@pytest.mark.parametrize("code,dcn", CODES3)
def test_cvt_3ch(cvb, oracle, rng, shape, code, dcn):
    img = rand_u8(rng, shape[0], shape[1], 3)
    got = cpu(cvb.cvtColor(gpu(img), code, dcn))
    assert_exact(got, oracle.cvtColor(img, code, dcn), "cvtColor code=%d dcn=%d %s" % (code, dcn, shape))


@pytest.mark.parametrize("code,dcn", [(C.COLOR_BGRA2GRAY, 1), (C.COLOR_RGBA2GRAY, 1), (C.COLOR_BGRA2BGR, 3), (C.COLOR_RGBA2BGR, 3),
                                      (C.COLOR_BGRA2RGBA, 4), (C.COLOR_BGR2YUV, 3), (C.COLOR_RGB2HSV, 3)])
def test_cvt_4ch(cvb, oracle, rng, code, dcn):
    img = rand_u8(rng, 255, 263, 4)
    assert_exact(cpu(cvb.cvtColor(gpu(img), code, dcn)), oracle.cvtColor(img, code, dcn), "cvtColor 4ch code=%d" % code)


def test_gray2bgr_and_batch(cvb, oracle, rng):
    g = rand_u8(rng, 255, 263)
    assert_exact(cpu(cvb.cvtColor(gpu(g), C.COLOR_GRAY2BGR)), oracle.cvtColor(g, C.COLOR_GRAY2BGR, 3), "GRAY2BGR")
    assert_exact(cpu(cvb.cvtColor(gpu(g), C.COLOR_GRAY2BGRA)), oracle.cvtColor(g, C.COLOR_GRAY2BGRA, 4), "GRAY2BGRA")
    batch = np.stack([rand_u8(rng, 96, 160, 3) for _ in range(4)])
    out = cpu(cvb.cvtColor(gpu(batch), C.COLOR_BGR2HSV))
    for i in range(4):
        assert_exact(out[i], oracle.cvtColor(batch[i], C.COLOR_BGR2HSV, 3), "batch %d" % i)


def test_unaligned_rows(cvb, oracle, rng):
    """a ROI whose rows are not 16-byte aligned takes the byte path of the same kernel"""
    import torch
    big = rand_u8(rng, 100, 301, 3)
    t = gpu(big)
    roi_t = t[3:90, 5:266]          # strides stay those of the parent: a cv::Mat ROI
    roi = big[3:90, 5:266]
    out = torch.empty((87, 261, 3), dtype=torch.uint8, device="cuda")
    cvb.cvtColor(roi_t, C.COLOR_BGR2YUV, dst=out)
    assert_exact(cpu(out), oracle.cvtColor(np.ascontiguousarray(roi), C.COLOR_BGR2YUV, 3), "ROI")


@pytest.mark.parametrize("code,dcn", [(C.COLOR_BGR2GRAY, 1), (C.COLOR_BGR2YUV, 3), (C.COLOR_BGR2HSV, 3), (C.COLOR_YUV2BGR, 3), (C.COLOR_HSV2BGR, 3)])
def test_cvt_8k(cvb, ref, rng, code, dcn):
    """bench.py workload c3 (cvtColor leg) at full 7680x4320 size against the real reference"""
    img = rand_u8(rng, 4320, 7680, 3)
    assert_exact(cpu(cvb.cvtColor(gpu(img), code, dcn)), ref.cvtColor(img, code, dcn), "8K code=%d" % code)
