"""GPU parity: cv::cvtColor for the Bayer mosaics (BG / GB / RG / GR -> BGR, BGRA; bilinear and edge-aware), 8- and 16-bit: BIT-EXACT.

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("size", [(3, 3), (4, 5), (17, 33), (64, 96), (241, 323), (1080, 1920)])
def test_bayer_demosaic(cvb, oracle, rng, size):
    img = rng.integers(0, 256, size, dtype=np.uint8)
    for code in (C.COLOR_BayerBG2BGR, C.COLOR_BayerGB2BGR, C.COLOR_BayerRG2BGR, C.COLOR_BayerGR2BGR,
                 C.COLOR_BayerBG2BGRA, C.COLOR_BayerGB2BGRA, C.COLOR_BayerRG2BGRA, C.COLOR_BayerGR2BGRA):
        assert_exact(cpu(cvb.cvtColor(gpu(img), code)), oracle.cvtColorYUV(img, code), "Bayer code %d %s" % (code, size))


def test_bayer_demosaic_4k_batch(cvb, ref, rng):
    batch = rng.integers(0, 256, (4, 2160, 3840, 1), dtype=np.uint8)
    out = cpu(cvb.cvtColor(gpu(batch), C.COLOR_BayerRG2BGR))
    assert out.shape == (4, 2160, 3840, 3)
    assert_exact(out[3], ref.cvtColorYUV(batch[3, :, :, 0], C.COLOR_BayerRG2BGR), "Bayer 4K batch frame 3")


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
@pytest.mark.parametrize("size", [(3, 3), (4, 5), (17, 33), (64, 96), (241, 323), (1080, 1920)])
def test_bayer_edge_aware_and_16bit(cvb, ref, rng, size, dtype):
    """COLOR_Bayer*2BGR_EA (green at red / blue sites follows the weaker gradient) for both depths; 16-bit mosaics also through the bilinear codes"""
    img = rng.integers(0, 256 if dtype == np.uint8 else 65536, size).astype(dtype)
    codes = [(C.COLOR_BayerBG2BGR_EA, 3), (C.COLOR_BayerGB2BGR_EA, 3), (C.COLOR_BayerRG2BGR_EA, 3), (C.COLOR_BayerGR2BGR_EA, 3)]
    if dtype == np.uint16:
        codes += [(C.COLOR_BayerBG2BGR, 3), (C.COLOR_BayerGB2BGR, 3), (C.COLOR_BayerRG2BGR, 3), (C.COLOR_BayerGR2BGR, 3), (C.COLOR_BayerBG2BGRA, 4), (C.COLOR_BayerGR2BGRA, 4)]
    for code, dcn in codes:
        got = cpu(cvb.cvtColor(gpu(img), code, dcn))
        assert got.dtype == dtype
        assert_exact(got, ref.cvtColor(img, code, dcn), "Bayer %s code %d %s" % (np.dtype(dtype).name, code, size))
