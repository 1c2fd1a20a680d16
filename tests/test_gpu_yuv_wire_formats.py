"""GPU parity: cvtColor for the subsampled-YUV wire formats (NV12 / NV21 / YV12 / IYUV / UYVY / YUY2 / YVYU -> BGR family, Y extraction,
BGR family -> I420 / YV12) through the device C ABI, the host API and the HAL seam.  All integer: BIT-EXACT, checked against the reference's
own known-answer hashes (modules/imgproc/test/test_color.cpp:2857-2900; inputs = its RNG(0) stream, tests/golden/) and the oracle.

A failure here fails the suite."""
import os
import zlib

import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]
GOLD = os.path.join(os.path.dirname(__file__), "golden")

# modules/imgproc/test/test_color.cpp:2857-2900
KAT_YUV = {90: 0x46a1bb76, 91: 0x3843bb76, 92: 0xf3fdf2ea, 93: 0x6e84f2ea, 94: 0xb6a16bd3, 95: 0xa8436bd3, 96: 0x1c7fa347, 97: 0x96f7a347,
           98: 0xc5da1651, 99: 0x12161651, 100: 0xb4e62ea5, 101: 0xfa632ea5, 102: 0x0db4c69f, 103: 0x59e1c69f, 104: 0xfe09def3, 105: 0x4395def3,
           106: 0xf672b440,
           107: 0x69bea2c1, 108: 0xdc51a2c1, 111: 0x851eab45, 112: 0xf7b1ab45, 115: 0x607e8889, 116: 0xfb148889, 117: 0x239b13d4, 118: 0x402b13d4,
           119: 0xf6af910d, 120: 0x9154910d, 121: 0x14481c58, 122: 0x30d81c58, 123: 0x228e669c, 124: 0x125c62fd,
           127: 0x44bb076a, 128: 0xf908ff52, 129: 0x44bb076a, 130: 0xf908ff52, 131: 0x1b0d076a, 132: 0xda8aff52, 133: 0x1b0d076a, 134: 0xda8aff52}
CODES_420 = list(range(90, 107))
CODES_422 = [107, 108, 111, 112, 115, 116, 117, 118, 119, 120, 121, 122, 123, 124]
CODES_TO_420 = list(range(127, 135))
CODES_TO_422 = list(range(143, 155))


def kat_input(code):
    name = "cvtcolor_kat_yuv420_input.npy" if code <= 106 else "cvtcolor_kat_yuv422_input.npy" if code <= 124 else "cvtcolor_kat_bgr_262x254_input.npy"
    return np.load(os.path.join(GOLD, name))


@pytest.mark.parametrize("code", sorted(KAT_YUV))
def test_known_answer_hashes(cvb, code):
    out = cpu(cvb.cvtColor(gpu(kat_input(code)), code))
    assert zlib.adler32(np.ascontiguousarray(out).tobytes()) == KAT_YUV[code]


@pytest.mark.parametrize("size", [(4, 6), (18, 34), (36, 66), (250, 322), (480, 640), (1080, 1920)])     # (h, w); h % 4 == 2 included
def test_yuv_vs_oracle(cvb, oracle, rng, size):
    h, w = size
    yuv = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    for code in CODES_420:
        assert_exact(cpu(cvb.cvtColor(gpu(yuv), code)), oracle.cvtColorYUV(yuv, code), "4:2:0 code %d %dx%d" % (code, w, h))
    y2 = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
    for code in CODES_422:
        assert_exact(cpu(cvb.cvtColor(gpu(y2), code)), oracle.cvtColorYUV(y2, code), "4:2:2 code %d %dx%d" % (code, w, h))
    for code in CODES_TO_420:
        img = rng.integers(0, 256, (h, w, 4 if (code - 127) & 2 else 3), dtype=np.uint8)
        assert_exact(cpu(cvb.cvtColor(gpu(img), code)), oracle.cvtColorYUV(img, code), "to 4:2:0 code %d %dx%d" % (code, w, h))
    for code in CODES_TO_422:
        for scn in (3, 4):
            img = rng.integers(0, 256, (h, w, scn), dtype=np.uint8)
            assert_exact(cpu(cvb.cvtColor(gpu(img), code)), oracle.cvtColorYUV(img, code), "to 4:2:2 code %d scn %d %dx%d" % (code, scn, w, h))


def test_yuv_padded_rows_and_batches(cvb, oracle, rng):
    """row pitches that defeat the 8-/16-byte paths (odd offsets into a wider buffer) and a batch of frames in one launch"""
    import torch
    h, w = 64, 106
    wide = rng.integers(0, 256, (h * 3 // 2, w + 7), dtype=np.uint8)
    src = gpu(wide)[:, 3:3 + w]                                   # pitch w + 7, base address off by 3
    want_src = np.ascontiguousarray(wide[:, 3:3 + w])
    for code in (C.COLOR_YUV2BGR_NV12, C.COLOR_YUV2RGBA_NV21, C.COLOR_YUV2BGR_I420, C.COLOR_YUV2RGB_YV12, C.COLOR_YUV2GRAY_420):
        assert_exact(cpu(cvb.cvtColor(src, code)), oracle.cvtColorYUV(want_src, code), "unaligned 4:2:0 code %d" % code)
    batch = rng.integers(0, 256, (5, 1080 * 3 // 2, 1920, 1), dtype=np.uint8)
    out = cpu(cvb.cvtColor(gpu(batch), C.COLOR_YUV2BGR_NV12))
    assert out.shape == (5, 1080, 1920, 3)
    for f in (0, 4):
        assert_exact(out[f], oracle.cvtColorYUV(batch[f, :, :, 0], C.COLOR_YUV2BGR_NV12), "NV12 batch frame %d" % f)
    bgr = rng.integers(0, 256, (3, 240, 322, 3), dtype=np.uint8)
    out = cpu(cvb.cvtColor(gpu(bgr), C.COLOR_BGR2YUV_I420))
    assert out.shape == (3, 360, 322, 1)
    assert_exact(out[2, :, :, 0], oracle.cvtColorYUV(bgr[2], C.COLOR_BGR2YUV_I420), "I420 batch frame 2")
    assert torch.cuda.is_available()


def test_two_plane(cvb, oracle, rng):
    """cv::cvtColorTwoPlane: luma and interleaved chroma in buffers of their own (own pitches), single frames and a batch"""
    for (h, w) in [(18, 34), (250, 322), (1080, 1920)]:
        y = rng.integers(0, 256, (h, w), dtype=np.uint8)
        wide = rng.integers(0, 256, (h // 2, w // 2 + 3, 2), dtype=np.uint8)
        uv = gpu(wide)[:, 1:1 + w // 2]
        for code in range(90, 98):
            got = cpu(cvb.cvtColorTwoPlane(gpu(y), uv, code))
            assert_exact(got, oracle.cvtColorTwoPlane(y, np.ascontiguousarray(wide[:, 1:1 + w // 2]), code), "two-plane code %d %dx%d" % (code, w, h))
    yb = rng.integers(0, 256, (3, 240, 320, 1), dtype=np.uint8); uvb = rng.integers(0, 256, (3, 120, 160, 2), dtype=np.uint8)
    out = cpu(cvb.cvtColorTwoPlane(gpu(yb), gpu(uvb), C.COLOR_YUV2BGR_NV12))
    assert_exact(out[2], oracle.cvtColorTwoPlane(yb[2, :, :, 0], uvb[2], C.COLOR_YUV2BGR_NV12), "two-plane batch frame 2")


def test_yuv_round_trip_4k(cvb, rng):
    """size-independent property at full size: BGR -> I420 -> BGR stays within the quantisation of the 4:2:0 format on a smooth image,
    and NV12 -> GRAY returns the luma plane untouched"""
    yy, xx = np.mgrid[0:2160, 0:3840]
    img = np.stack([(xx / 16) % 256, (yy / 9) % 256, ((xx + yy) / 24) % 256], axis=-1).astype(np.uint8)
    i420 = cvb.cvtColor(gpu(img), C.COLOR_BGR2YUV_I420)
    back = cpu(cvb.cvtColor(i420, C.COLOR_YUV2BGR_I420)).astype(np.int32)
    assert np.percentile(np.abs(back - img.astype(np.int32)), 99) <= 6
    nv = rng.integers(0, 256, (3240, 3840), dtype=np.uint8)
    assert_exact(cpu(cvb.cvtColor(gpu(nv), C.COLOR_YUV2GRAY_NV12)), nv[:2160], "GRAY_420")


def test_yuv_host_and_hal_paths(cvb, oracle, rng):
    """host buffers through b200cv_host_cvt_color, and plain cv::cvtColor of an OpenCV built with the B200 HAL (hal_ni_cvtTwoPlaneYUVtoBGR,
    cvtThreePlaneYUVtoBGR, cvtBGRtoThreePlaneYUV, cvtOnePlaneYUVtoBGR)"""
    from opencv_b200 import hal
    nv = rng.integers(0, 256, (720, 640), dtype=np.uint8)
    assert_exact(hal.cvtColor(nv, C.COLOR_YUV2BGR_NV12), oracle.cvtColorYUV(nv, C.COLOR_YUV2BGR_NV12), "host NV12")
    from oracle.api import Oracle, available
    if not available("ref_hal") or not available("ref"):
        return
    rh, ref = Oracle("ref_hal"), Oracle("ref")
    if not rh.has("cvt_color_yuv"):
        return
    y2 = rng.integers(0, 256, (480, 640, 2), dtype=np.uint8)
    bgr = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
    n0 = cvb.launch_count()
    for src, code in ((nv, 91), (nv, 96), (nv, 99), (nv, 104), (y2, 108), (y2, 117), (y2, 120), (bgr, 128), (bgr, 131), (bgr, 144), (bgr, 147), (bgr, 150)):
        assert_exact(rh.cvtColorYUV(src, code), ref.cvtColorYUV(src, code), "cv::cvtColor code %d via HAL" % code)
    assert cvb.launch_count() - n0 >= 12, "cv::cvtColor(YUV wire formats) did not reach the B200 HAL"
