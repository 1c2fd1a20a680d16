"""GPU: the multi-GPU batch driver (include/b200cv_batch.h, opencv_b200.batch.BatchDriver) -- sharded host batches must give exactly what the
single-device host API gives frame by frame (the kernels are the same; only sharding, staging and the template broadcast are new).
The multi-device cases run when the box shows more than one GPU (gpurun --gpus N); on one GPU the same code runs with one worker."""
import ctypes

import numpy as np
import pytest

import opencv_b200 as C
from opencv_b200 import hal
from opencv_b200.batch import BatchDriver
from util import assert_exact, cpu, gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["one", "all"])
def driver(request, cvb):
    n = C.lib().b200cv_device_count()
    if request.param == "all" and n < 2:
        pytest.skip("one GPU visible: the multi-device driver needs two or more")
    d = BatchDriver([0] if request.param == "one" else None)
    yield d
    d.close()


def test_driver_topology(driver):
    n = driver.n_devices
    assert driver.devices == list(range(n))
    assert driver.uses_nccl == (n > 1)
    blocks = [driver.shard(11, i) for i in range(n)]
    assert blocks[0][0] == 0 and blocks[-1][1] == 11 and all(blocks[i][1] == blocks[i + 1][0] for i in range(n - 1))


def test_sharded_ops_equal_single_device(driver, rng):
    n = 11
    src = driver.pinned_frames((n, 270, 480, 3), np.uint8)
    src[...] = rng.integers(0, 256, src.shape, dtype=np.uint8)
    assert_exact(driver.GaussianBlur(src, (5, 5), 0), hal.GaussianBlur(src, (5, 5), 0), "batch GaussianBlur")
    assert sum(driver.last_counts()) == n
    assert_exact(driver.cvtColor(src, C.COLOR_BGR2GRAY), hal.cvtColor(src, C.COLOR_BGR2GRAY), "batch cvtColor")
    assert_exact(driver.resize(src, (333, 199), interpolation=C.INTER_LINEAR), hal.resize(src, (333, 199), interpolation=C.INTER_LINEAR), "batch resize")
    M = np.array([[0.9, 0.1, 5], [-0.1, 0.9, 7]])
    assert_exact(driver.warpAffine(src, M, (480, 270), flags=C.INTER_CUBIC), hal.warpAffine(src, M, (480, 270), flags=C.INTER_CUBIC), "batch warpAffine")
    ker = rng.random((7, 7)).astype(np.float32)
    assert_exact(driver.filter2D(src, -1, ker / ker.sum()), hal.filter2D(src, -1, ker / ker.sum()), "batch filter2D")
    gray = np.ascontiguousarray(src[..., :1])
    assert_exact(driver.cornerHarris(gray, 2, 3, 0.04), hal.cornerHarris(gray, 2, 3, 0.04), "batch cornerHarris")
    t = np.ascontiguousarray(gray[3, 40:72, 100:148, 0])
    # the template reaches devices 1.. through ncclBroadcast
    assert_exact(driver.matchTemplate(gray, t, C.TM_CCORR_NORMED), hal.matchTemplate(gray, t, C.TM_CCORR_NORMED), "batch matchTemplate")
    fewer = src[:1]        # fewer frames than devices: the extra workers idle
    assert_exact(driver.GaussianBlur(fewer, (3, 3), 0), hal.GaussianBlur(fewer, (3, 3), 0), "batch of one frame")


def test_sift_harris_waves(driver, rng):
    """C5 pipeline: waves of pyramids + Harris; the responses equal cornerHarris, the pyramids seen by the consumer equal b200cv_sift_pyramid"""
    n, H, W = 7, 120, 160
    src = driver.pinned_frames((n, H, W, 1), np.uint8)
    base = np.kron(rng.random((H // 8 + 1, W // 8 + 1)), np.ones((8, 8)))[:H, :W]
    for f in range(n):
        src[f, :, :, 0] = (np.roll(base, (3 * f, 5 * f), (0, 1)) * 255).astype(np.uint8)
    har = driver.pinned_frames((n, H, W, 1), np.float32)
    L = C.lib()
    seen = {}

    def consumer(dev_index, f0, nf, g, gstride, d, dstride, h, hstep, hfstep):
        for k in range(nf):
            out = np.empty(256, np.float32)      # head of every frame's Gaussian pyramid
            assert L.b200cv_download(ctypes.c_void_p(g + 4 * gstride * k), ctypes.c_size_t(1024), out.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(1024),
                                     ctypes.c_size_t(1024), ctypes.c_size_t(1), None) == 0
            assert L.b200cv_stream_synchronize(None) == 0
            seen[f0 + k] = out
        return 0

    driver.sift_harris(src, har, wave=2, consumer=consumer)
    assert sorted(seen) == list(range(n))
    assert_exact(har, hal.cornerHarris(src, 2, 3, 0.04), "wave Harris responses")
    G, D, dims = C.sift_pyramid(gpu(src), 3, 1.6, True)
    Gc = cpu(G)
    for f in range(n):
        assert_exact(seen[f], Gc[f].reshape(-1)[:256], "pyramid head of frame %d" % f)
    # responses may stay on the device
    driver.sift_harris(src, None, wave=3)
    assert sum(driver.last_counts()) == n
