"""GPU parity: cv::resize INTER_LANCZOS4, 8-bit and float: BIT-EXACT (weights built on the host with the reference's expressions and libm).

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]

CASES = [((40, 60), (120, 180)), ((40, 60), (97, 131)), ((100, 150), (237, 341)), ((97, 131), (98, 132)), ((64, 64), (160, 32)), ((120, 180), (40, 61)),
         ((1, 47), (5, 90)), ((50, 1), (75, 23)), ((3, 5), (30, 50)), ((120, 160), (121, 100)), ((240, 320), (150, 201)), ((480, 640), (300, 402))]


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("ssize,dsize", CASES)
def test_lanczos4_resize(cvb, oracle, rng, ssize, dsize, cn):
    (sh, sw), (dh, dw) = ssize, dsize
    shape = (sh, sw) if cn == 1 else (sh, sw, cn)
    for img in (rng.integers(0, 256, shape, dtype=np.uint8), (rng.random(shape, dtype=np.float32) * 255).astype(np.float32)):
        got = cpu(cvb.resize(gpu(img), (dw, dh), interpolation=C.INTER_LANCZOS4))
        assert_exact(got, oracle.resize(img, (dw, dh), 4), "LANCZOS4 %s %s -> %s cn=%d" % (img.dtype, ssize, dsize, cn))


def test_lanczos4_resize_8k_batch(cvb, ref, rng):
    base = rng.integers(0, 256, (4320, 7680, 3), dtype=np.uint8)
    batch = np.stack([base, np.roll(base, 5, axis=0)])
    out = cpu(cvb.resize(gpu(batch), (5120, 2880), interpolation=C.INTER_LANCZOS4))
    assert_exact(out[1], ref.resize(batch[1], (5120, 2880), 4), "LANCZOS4 8K -> 5K")


@pytest.mark.parametrize("cn", [1, 3, 4])
def test_lanczos4_first_version_equals_tiled_kernel(cvb, rng, monkeypatch, cn):
    """B200CV_RESIZE_LANCZOS_PATH=v1 (one thread per element, 64 gathers) == the tiled separable kernel; includes a strong decimation
    whose tiles do not fit shared memory and stay on the first version either way"""
    shape = (211, 333) if cn == 1 else (211, 333, cn)
    img = gpu(rng.integers(0, 256, shape, dtype=np.uint8))
    for dsz in ((500, 317), (96, 100), (666, 422), (33, 7)):
        monkeypatch.delenv("B200CV_RESIZE_LANCZOS_PATH", raising=False)
        got = cpu(cvb.resize(img, dsz, interpolation=C.INTER_LANCZOS4))
        monkeypatch.setenv("B200CV_RESIZE_LANCZOS_PATH", "v1")
        assert_exact(cpu(cvb.resize(img, dsz, interpolation=C.INTER_LANCZOS4)), got, "LANCZOS4 v1 vs tiled %s cn=%d" % (dsz, cn))
