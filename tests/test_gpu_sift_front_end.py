"""GPU: the SIFT front end after the pyramid -- scale-space extrema, refinement, orientation, descriptors -- against the
reference's own cv::SIFT::detectAndCompute (enable_precise_upscale = true, the first octave b200cv_sift_pyramid builds).

Parity is by tolerance: the reference's SIFT objects are FMA-contracted AVX2 / AVX-512 builds with OpenCV's approximate exp / atan2, and the small
octaves of the GPU pyramid differ from the reference's by <= 1e-4 (tests/test_gpu_features.py).  Bars: keypoint count within 2 %, >= 97 % of the
reference's keypoints matched to 1e-2 px / 0.1 deg, and for matched keypoints >= 99 % of the descriptor entries within +-1 (stored bytes).
The port (oracle/port) is pinned to the reference at 99 % / 1e-3 px on the reference's own pyramids (tests/test_oracle.py), and the kernels run on
the host equal the port exactly (tests/test_kernel_emulation.py).

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import gpu

pytestmark = [pytest.mark.gpu]


def structured(rng, h, w):
    small = rng.random((h // 8 + 2, w // 8 + 2)).astype(np.float32)
    img = np.kron(small, np.ones((8, 8), np.float32))[:h, :w] + 0.15 * rng.random((h, w)).astype(np.float32)
    img = (img - img.min()) / (img.max() - img.min())
    return (img * 255).astype(np.uint8)


def match(a, b, tol_xy, tol_angle):
    """index pairs (i, j) of a one-to-one greedy match of keypoint arrays (n,5) on x, y, size, angle"""
    used = np.zeros(len(b), bool)
    order = np.argsort(b[:, 0], kind="stable")
    bx = b[order, 0]
    pairs = []
    for i, k in enumerate(a):
        lo, hi = np.searchsorted(bx, k[0] - tol_xy), np.searchsorted(bx, k[0] + tol_xy)
        for j in order[lo:hi]:
            da = abs(b[j, 3] - k[3])
            if not used[j] and abs(b[j, 1] - k[1]) <= tol_xy and abs(b[j, 2] - k[2]) <= tol_xy and min(da, 360 - da) <= tol_angle:
                used[j] = True
                pairs.append((i, j))
                break
    return pairs


def test_sift_default_first_octave(cvb, ref, rng):
    """enable_precise_upscale = false (SIFT::create's default): the first octave comes from cv::resize LINEAR"""
    from oracle.api import unpack_pyramid
    from util import assert_close, cpu
    img = structured(rng, 240, 320)
    wg, wd = ref.sift_pyramid(img, 3, 1.6, 2)
    G, D, dims = cvb.sift_pyramid(gpu(img), 3, 1.6, 2)
    gg, gd = unpack_pyramid(cpu(G)[0], cpu(D)[0], dims.reshape(-1), len(dims), 3)
    for o in range(len(wg)):
        assert_close(gg[o][5], wg[o][5], atol=1e-4, what="default first octave: gauss o=%d" % o)
    kr, octr, dr = ref.sift_detect_and_compute(img, precise_upscale=False)
    kg, octg, dg = cvb.sift_detectAndCompute(gpu(img), enable_precise_upscale=False)
    assert abs(len(kg) - len(kr)) <= max(5, len(kr) // 50) and len(match(kr, kg, 1e-2, 0.1)) >= 0.97 * len(kr)


@pytest.mark.parametrize("size", [(240, 320), (480, 640), (1080, 1920)])
def test_sift_detect_and_compute(cvb, ref, rng, size):
    img = structured(rng, *size)
    kr, octr, dr = ref.sift_detect_and_compute(img)
    kg, octg, dg = cvb.sift_detectAndCompute(gpu(img))
    assert abs(len(kg) - len(kr)) <= max(5, len(kr) // 50), "keypoint count %d vs %d" % (len(kg), len(kr))
    pairs = match(kr, kg, 1e-2, 0.1)
    assert len(pairs) >= 0.97 * len(kr), "%d of %d reference keypoints matched" % (len(pairs), len(kr))
    i, j = np.array(pairs).T
    assert (octr[i] == octg[j]).mean() >= 0.99
    diff = np.abs(dr[i] - dg[j])
    assert (diff <= 1).mean() >= 0.99, "descriptor entries within +-1: %.4f" % (diff <= 1).mean()
    # the keypoints come out in the reference's order (KeyPoint12_LessThan): sorted by x
    assert np.all(np.diff(kg[:, 0]) >= 0)
    # nfeatures = retainBest: the strongest responses (ties included), the reference's selection
    k500, _, d500 = cvb.sift_detectAndCompute(gpu(img), nfeatures=500)
    r500, _, _ = ref.sift_detect_and_compute(img, nfeatures=500)
    assert abs(len(k500) - len(r500)) <= 10 and len(match(r500, k500, 1e-2, 0.1)) >= 0.95 * len(r500)
    assert d500.shape == (len(k500), 128)
    # mask = runByPixelsMask on the rounded positions, before the descriptors; a batch is a list of per-frame results
    mask = np.zeros(img.shape, np.uint8); mask[size[0] // 4: size[0] // 2, size[1] // 4: 3 * size[1] // 4] = 255
    km, _, dm = cvb.sift_detectAndCompute(gpu(img), mask=mask)
    keep = mask[(kg[:, 1] + 0.5).astype(np.int32), (kg[:, 0] + 0.5).astype(np.int32)] != 0
    assert np.array_equal(km, kg[keep]) and np.array_equal(dm, dg[keep])
    if size[0] <= 480:
        res = cvb.sift_detectAndCompute(gpu(np.stack([img, img[::-1].copy()])[..., None]))
        assert len(res) == 2 and np.array_equal(res[0][0], kg) and np.array_equal(res[0][2], dg)


def test_sift_detect_4k(cvb, ref, rng):
    """bench.py workload c5 frame size: detectAndCompute on one 3840x2160 8UC1 frame against cv::SIFT (sift.dispatch.cpp:176-310, 405-472)"""
    img = structured(rng, 2160, 3840)
    kr, octr, dr = ref.sift_detect_and_compute(img)
    kg, octg, dg = cvb.sift_detectAndCompute(gpu(img))
    assert abs(len(kg) - len(kr)) <= max(5, len(kr) // 50), "keypoint count %d vs %d" % (len(kg), len(kr))
    pairs = match(kr, kg, 1e-2, 0.1)
    assert len(pairs) >= 0.97 * len(kr), "%d of %d reference keypoints matched" % (len(pairs), len(kr))
    i, j = np.array(pairs).T
    assert (octr[i] == octg[j]).mean() >= 0.99
    diff = np.abs(dr[i] - dg[j])
    assert (diff <= 1).mean() >= 0.99, "descriptor entries within +-1: %.4f" % (diff <= 1).mean()
    assert np.all(np.diff(kg[:, 0]) >= 0)
