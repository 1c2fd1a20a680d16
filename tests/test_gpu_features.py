"""GPU parity: matchTemplate, cornerHarris / cornerMinEigenVal, goodFeaturesToTrack, SIFT pyramid vs the CPU oracle.

Bars
  matchTemplate ......... relative 1e-3 of the result range (the reference's own bar, test_templmatch.cpp:333; its numerator is a
                          float DFT, ours is the exact integer sum for 8-bit images)
  cornerHarris/MinEig ... |d| <= 2e-6 * max|ref| + tiny  (reference test: relative 2e-6, test_goodfeaturetotrack.cpp:439-513;
                          operations are the same fp32 ones, only FMA chaining inside the 3-tap Sobel rows differs)
  goodFeaturesToTrack ... identical corner list (order included) whenever the response maps agree on the ranking; compared as
                          exact coordinates on inputs with well separated responses
  SIFT pyramid .......... per level |d| <= 1e-3 absolute on a 0..255 scale (a chain of up to 5 f32 blurs per octave and 10 octaves;
                          NOTE the reference has no test that pins these pyramids -- the oracle is the reference's own code
                          (oracle/_ref) or the same composition of public calls in the port)
"""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_close, assert_exact, cpu, gpu, rand_u8

pytestmark = pytest.mark.gpu


def smooth_img(rng, h, w):
    """band-limited random image: corners / templates with structure instead of white noise"""
    small = rng.random((h // 8 + 2, w // 8 + 2)).astype(np.float32)
    img = np.kron(small, np.ones((8, 8), np.float32))[:h, :w]
    img = img + 0.15 * rng.random((h, w)).astype(np.float32)
    img = (img - img.min()) / (img.max() - img.min())
    return (img * 255).astype(np.uint8)


@pytest.mark.parametrize("method", [C.TM_SQDIFF, C.TM_SQDIFF_NORMED, C.TM_CCORR, C.TM_CCORR_NORMED, C.TM_CCOEFF, C.TM_CCOEFF_NORMED])
@pytest.mark.parametrize("isz,tsz", [((128, 160), (17, 23)), ((200, 320), (64, 64)), ((131, 97), (1, 1)), ((90, 90), (30, 7))])
def test_match_template_u8(cvb, oracle, rng, method, isz, tsz):
    img = rand_u8(rng, *isz)
    templ = img[5:5 + tsz[0], 9:9 + tsz[1]].copy() if tsz[0] > 1 else rand_u8(rng, *tsz)
    want = oracle.matchTemplate(img, templ, method)
    got = cpu(cvb.matchTemplate(gpu(img), gpu(templ), method))
    scale = max(1.0, float(np.abs(want).max()))
    assert_close(got, want, atol=1e-3 * scale, what="matchTemplate u8 method=%d %s %s" % (method, isz, tsz))


@pytest.mark.parametrize("tsz", [(64, 64), (7, 13), (1, 3), (33, 2), (19, 130), (20, 32), (5, 16), (9, 128)])
def test_match_template_fused_window_sums(cvb, rng, monkeypatch, tsz):
    """8-bit images: the fused window-sum + normalisation kernel (exact u32 sums, one pass) against the first version (f64 planes of
    sliding sums): the same exact integers enter the same f64 formula, so the results must be IDENTICAL -- all six methods, ragged sizes,
    templates narrower than a word, a batch, an unaligned sub-view (which must take the planes path and agree too)."""
    import torch
    img = rng.integers(0, 256, (3, 211, 333, 1), dtype=np.uint8)
    templ = np.ascontiguousarray(img[1, 40:40 + tsz[0], 50:50 + tsz[1], 0])
    for method in range(6):
        got = cpu(cvb.matchTemplate(gpu(img), gpu(templ), method))
        monkeypatch.setenv("B200CV_MATCHTEMPLATE_NORM", "planes")
        want = cpu(cvb.matchTemplate(gpu(img), gpu(templ), method))
        monkeypatch.delenv("B200CV_MATCHTEMPLATE_NORM")
        assert_exact(got, want, "matchTemplate fused vs planes method=%d templ=%s" % (method, tsz))
    view = gpu(img)[:, 3:, 1:, :]               # base not 4-byte aligned: planes path
    sub = np.ascontiguousarray(img[:, 3:, 1:, :])
    if tsz[0] <= sub.shape[1] and tsz[1] <= sub.shape[2]:
        assert_exact(cpu(cvb.matchTemplate(view, gpu(templ), C.TM_CCOEFF_NORMED)), cpu(cvb.matchTemplate(gpu(sub), gpu(templ), C.TM_CCOEFF_NORMED)), "matchTemplate unaligned view")


@pytest.mark.parametrize("method", [C.TM_SQDIFF_NORMED, C.TM_CCORR, C.TM_CCORR_NORMED, C.TM_CCOEFF_NORMED])
def test_match_template_f32(cvb, oracle, rng, method):
    img = rand_u8(rng, 128, 160).astype(np.float32)
    templ = img[20:20 + 19, 30:30 + 33].copy()
    want = oracle.matchTemplate(img, templ, method)
    got = cpu(cvb.matchTemplate(gpu(img), gpu(templ), method))
    assert_close(got, want, atol=1e-3 * max(1.0, float(np.abs(want).max())), what="matchTemplate f32 method=%d" % method)


def test_match_template_4k(cvb, ref, rng):
    """bench.py workload c4: TM_CCORR_NORMED, 3840x2160 8UC1 frame vs a 64x64 crop at (1000,700)"""
    img = rand_u8(rng, 2160, 3840)
    templ = img[700:764, 1000:1064].copy()
    want = ref.matchTemplate(img, templ, C.TM_CCORR_NORMED)
    got = cpu(cvb.matchTemplate(gpu(img), gpu(templ), C.TM_CCORR_NORMED))
    assert_close(got, want, atol=1e-3, what="C4 matchTemplate")
    assert np.unravel_index(got.argmax(), got.shape) == (700, 1000)


@pytest.mark.parametrize("bs,ks", [(2, 3), (3, 3), (5, 5), (3, 7), (2, 1), (7, 3)])
@pytest.mark.parametrize("border", [C.BORDER_REFLECT_101, C.BORDER_REPLICATE, C.BORDER_CONSTANT, C.BORDER_REFLECT])
def test_corner_harris(cvb, oracle, rng, bs, ks, border):
    for img in (smooth_img(rng, 97, 131), smooth_img(rng, 64, 200).astype(np.float32) / 255.0):
        want = oracle.cornerHarris(img, bs, ks, 0.04, border)
        got = cpu(cvb.cornerHarris(gpu(img), bs, ks, 0.04, border))
        assert_close(got, want, atol=5e-7 * float(np.abs(want).max()) + 1e-12, what="cornerHarris %s bs=%d ks=%d border=%d" % (img.dtype, bs, ks, border))
        want = oracle.cornerMinEigenVal(img, bs, ks, border)
        got = cpu(cvb.cornerMinEigenVal(gpu(img), bs, ks, border))
        assert_close(got, want, atol=5e-7 * float(np.abs(want).max()) + 1e-12, what="cornerMinEigenVal %s bs=%d ks=%d" % (img.dtype, bs, ks))


def test_corner_harris_4k(cvb, ref, rng):
    """bench.py workload c4: cornerHarris(blockSize=2, ksize=3, k=0.04) on 3840x2160 8UC1"""
    img = smooth_img(rng, 2160, 3840)
    want = ref.cornerHarris(img, 2, 3, 0.04)
    got = cpu(cvb.cornerHarris(gpu(img), 2, 3, 0.04))
    assert_close(got, want, atol=5e-7 * float(np.abs(want).max()), what="C4 cornerHarris")


@pytest.mark.parametrize("harris", [True, False])
@pytest.mark.parametrize("mind", [0, 1, 5, 10.5])
def test_good_features(cvb, oracle, rng, harris, mind):
    img = smooth_img(rng, 240, 320)
    want, wq = oracle.goodFeaturesToTrack(img, 200, 0.01, mind, 3, 3, harris, 0.04)
    got, gq = cvb.goodFeaturesToTrack(gpu(img), 200, 0.01, mind, 3, 3, harris, 0.04, with_quality=True)
    assert len(got) == len(want), "corner count %d vs %d" % (len(got), len(want))
    # same set; same order wherever neighbouring responses are separated by more than the fp32 noise of the response map
    assert_close(gq, wq, atol=5e-7 * float(np.abs(wq).max()), what="corner qualities")
    same = np.all(got == want, axis=1)
    if not same.all():
        gs = set(map(tuple, got.tolist())); ws = set(map(tuple, want.tolist()))
        assert len(gs ^ ws) <= max(2, len(want) // 50), "corner sets differ: %s" % sorted(gs ^ ws)[:10]


def test_good_features_4k(cvb, ref, rng):
    """bench.py workload c4: goodFeaturesToTrack(1000, 0.01, 10, blockSize 3, gradientSize 3, Harris k=0.04) on 4K"""
    img = smooth_img(rng, 2160, 3840)
    want, wq = ref.goodFeaturesToTrack(img, 1000, 0.01, 10, 3, 3, True, 0.04)
    got, gq = cvb.goodFeaturesToTrack(gpu(img), 1000, 0.01, 10, 3, 3, True, 0.04, with_quality=True)
    assert len(got) == len(want) == 1000
    gs = set(map(tuple, got.tolist())); ws = set(map(tuple, want.tolist()))
    assert len(gs ^ ws) <= 20, "corner sets differ in %d entries" % len(gs ^ ws)


@pytest.mark.parametrize("max_corners,mind", [(1000, 10), (300, 0), (6000, 60), (50000, 3)])
def test_good_features_preselection_equals_full_sort(cvb, rng, monkeypatch, max_corners, mind):
    """the top-K preselection (histogram of the response code, compaction, sort of the prefix) gives the corner list of the full sort:
    the walk ending inside the prefix (1000/10, 300/0), the prefix running out -> redone with every candidate (6000/60), more corners
    asked for than the prefix holds (50000/3)"""
    img = rng.integers(0, 256, (2160, 3840), dtype=np.uint8)              # noise: ~10^6 local maxima above the quality level
    d = gpu(img)
    got, gq = cvb.goodFeaturesToTrack(d, max_corners, 0.01, mind, 3, 3, True, 0.04, with_quality=True)
    monkeypatch.setenv("B200CV_GFTT_PRESELECT", "0")
    want, wq = cvb.goodFeaturesToTrack(d, max_corners, 0.01, mind, 3, 3, True, 0.04, with_quality=True)
    assert len(got) == len(want) and len(got) > 0
    assert np.array_equal(got, want) and np.array_equal(gq, wq)


@pytest.mark.parametrize("shape,upscale", [((135, 240), True), ((100, 75), True), ((96, 128), False)])
def test_sift_pyramid(cvb, oracle, rng, shape, upscale):
    from oracle.api import unpack_pyramid
    img = smooth_img(rng, *shape)
    wg, wd = oracle.sift_pyramid(img, 3, 1.6, upscale)
    G, D, dims = cvb.sift_pyramid(gpu(img), 3, 1.6, upscale)
    no = len(dims)
    assert no == len(wg)
    gg, gd = unpack_pyramid(cpu(G)[0], cpu(D)[0], dims.reshape(-1), no, 3)
    exact = True     # octaves are bit-exact as long as no level so far had remainder columns (width % 8) in the reference's SIMD loops
    for o in range(no):
        exact = exact and wg[o][0].shape[1] % 8 == 0
        for i in range(6):
            if exact:
                assert_exact(gg[o][i], wg[o][i], "gauss o=%d i=%d" % (o, i))
            else:
                assert_close(gg[o][i], wg[o][i], atol=1e-4, what="gauss o=%d i=%d" % (o, i))
        for i in range(5):
            if exact:
                assert_exact(gd[o][i], wd[o][i], "dog o=%d i=%d" % (o, i))
            else:
                assert_close(gd[o][i], wd[o][i], atol=1e-4, what="dog o=%d i=%d" % (o, i))
            # the fused DoG must be exactly the f32 difference of the two stored Gaussian levels
            assert_exact(gd[o][i], gg[o][i + 1] - gg[o][i], "dog == G[i+1]-G[i] o=%d i=%d" % (o, i))


def test_sift_pyramid_batch_1080p(cvb, ref, rng):
    base = smooth_img(rng, 540, 960)
    batch = np.stack([np.roll(base, (17 * i, 31 * i), axis=(0, 1)) for i in range(3)])[..., None]
    G, D, dims = cvb.sift_pyramid(gpu(batch), 3, 1.6, True)
    from oracle.api import unpack_pyramid
    for f in (0, 2):
        wg, wd = ref.sift_pyramid(batch[f, :, :, 0], 3, 1.6, True)
        gg, gd = unpack_pyramid(cpu(G)[f], cpu(D)[f], dims.reshape(-1), len(dims), 3)
        exact = True
        for o in range(len(dims)):
            exact = exact and wg[o][0].shape[1] % 8 == 0
            if exact:      # 1920, 960, 480, 240, 120 wide: the whole level equals the reference bit for bit
                assert_exact(gg[o][5], wg[o][5], "frame %d gauss o=%d" % (f, o))
                assert_exact(gd[o][4], wd[o][4], "frame %d dog o=%d" % (f, o))
            else:
                assert_close(gg[o][5], wg[o][5], atol=1e-4, what="frame %d gauss o=%d" % (f, o))
                assert_close(gd[o][4], wd[o][4], atol=1e-4, what="frame %d dog o=%d" % (f, o))


def test_sift_pyramid_4k(cvb, ref, rng):
    """bench.py workload c5 frame size: the whole Gaussian + DoG pyramid of one 3840x2160 8UC1 frame against the reference's
    buildGaussianPyramid / buildDoGPyramid (sift.dispatch.cpp:176-310).  7680 ... 120 wide octaves (W % 8 == 0): bit for bit, all levels."""
    from oracle.api import unpack_pyramid
    img = smooth_img(rng, 2160, 3840)
    wg, wd = ref.sift_pyramid(img, 3, 1.6, True)
    G, D, dims = cvb.sift_pyramid(gpu(img), 3, 1.6, True)
    gg, gd = unpack_pyramid(cpu(G)[0], cpu(D)[0], dims.reshape(-1), len(dims), 3)
    assert len(dims) == len(wg)
    exact = True
    for o in range(len(dims)):
        exact = exact and wg[o][0].shape[1] % 8 == 0
        for i in range(6):
            if exact:
                assert_exact(gg[o][i], wg[o][i], "4K gauss o=%d i=%d" % (o, i))
            else:
                assert_close(gg[o][i], wg[o][i], atol=1e-4, what="4K gauss o=%d i=%d" % (o, i))
        for i in range(5):
            if exact:
                assert_exact(gd[o][i], wd[o][i], "4K dog o=%d i=%d" % (o, i))
            else:
                assert_close(gd[o][i], wd[o][i], atol=1e-4, what="4K dog o=%d i=%d" % (o, i))


@pytest.mark.parametrize("shape", [(135, 241), (64, 96), (211, 77), (540, 960)])
@pytest.mark.parametrize("switch", ["B200CV_SIFT_UPSCALE_WARP", "B200CV_SIFT_NO_SMALL_OCTAVES"])
def test_sift_fused_stages_equal_the_composition(cvb, rng, monkeypatch, shape, switch):
    """Two fused stages of the pyramid against the reference's own composition of calls (sift.dispatch.cpp:196-202, 224-310), which stays
    reachable through a switch: (1) createInitialImage's precise 2x upscale as one u8 -> f32 + upsample kernel vs the general warpAffine kernel;
    (2) the small octaves (levels that fit shared memory) as ONE launch vs resize(NEAREST) + GaussianBlur per level.  Every level of both
    pyramids must be identical -- odd widths / heights, a batch, with and without the doubled base."""
    img = rng.integers(0, 256, (2,) + shape + (1,), dtype=np.uint8)
    for upscale in (True, False):
        G, D, dims = cvb.sift_pyramid(gpu(img), 3, 1.6, upscale)
        monkeypatch.setenv(switch, "1")
        G2, D2, dims2 = cvb.sift_pyramid(gpu(img), 3, 1.6, upscale)
        monkeypatch.delenv(switch)
        assert np.array_equal(dims, dims2)
        _, ge, de, _ = C.sift_pyramid_layout(shape[1], shape[0], 3, upscale)        # the frame stride is rounded up: compare the pyramids, not the padding
        assert_exact(cpu(G)[:, :ge], cpu(G2)[:, :ge], "Gaussian pyramid with and without %s (upscale=%s)" % (switch, upscale))
        assert_exact(cpu(D)[:, :de], cpu(D2)[:, :de], "DoG pyramid with and without %s (upscale=%s)" % (switch, upscale))


@pytest.mark.parametrize("bs", [2, 3])
@pytest.mark.parametrize("shape", [(2, 333, 517), (1, 200, 1031), (3, 131, 290)])
def test_corner_response_fast_kernel_equals_tile_kernel(cvb, rng, monkeypatch, bs, shape):
    """cornerHarris / cornerMinEigenVal with the 3-tap Sobel and a 2 x 2 or 3 x 3 block: interior tiles run on the register-marching kernel,
    the border ring on the tile kernel (harris.cu).  Same operations in the same order: the two must agree bit for bit (8-bit and float
    sources, a batch, sizes that leave partial tiles), and the composite must equal the all-tile result."""
    for dt in (np.uint8, np.float32):
        img = smooth_img(rng, shape[1], shape[2] * shape[0]).reshape(shape[1], shape[0], shape[2]).transpose(1, 0, 2).copy()[..., None]
        img = img if dt == np.uint8 else img.astype(np.float32) / 255.0
        for fn, args in ((cvb.cornerHarris, (bs, 3, 0.04)), (cvb.cornerMinEigenVal, (bs, 3))):
            got = cpu(fn(gpu(img), *args))
            monkeypatch.setenv("B200CV_HARRIS_PATH", "tile")
            want = cpu(fn(gpu(img), *args))
            monkeypatch.delenv("B200CV_HARRIS_PATH")
            assert_exact(got, want, "%s bs=%d %s %s: fast + border tiles vs tile kernel" % (fn.__name__, bs, np.dtype(dt).name, shape))
