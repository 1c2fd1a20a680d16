"""GPU parity: resize / warpAffine / warpPerspective through the device C ABI vs the CPU oracle.

Bars (the reference's own strict test allows |d| <= 1 for LINEAR/CUBIC, test_imgwarp_strict.cpp:231-243):
  resize NEAREST, LINEAR u8, AREA 2x2 u8, CUBIC u8 ......... BIT-EXACT (the SSE vector-body / scalar-tail split of the
                                                             reference's u8 CUBIC column pass is reproduced)
  warp* u8 (NEAREST/LINEAR/CUBIC) .......................... BIT-EXACT (fixed-point coordinates + 2^15 tap tables)
  f32 (resize and warps, every interpolation and border) ... BIT-EXACT: same float operations in the same order

Resize and the warps here run at a few everyday geometries and at 8K.  tests/test_gpu_warp_exact.py takes each of the four warp
kernels to its tile, column-block, footprint and alignment edges (table: tests/warp_cases.py; the port it compares with is held to the
reference over the same table by tests/test_warp_port.py); tests/test_gpu_resize_exact_edges.py does the same for every resize kernel
(table: tests/resize_cases.py; port against reference: tests/test_resize_port.py).
"""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_close, assert_exact, cpu, gpu, rand_u8

pytestmark = pytest.mark.gpu

SIZES = [((97, 131), (61, 77)), ((64, 48), (128, 96)), ((120, 160), (60, 80)), ((33, 300), (100, 41)), ((50, 50), (75, 33)), ((7, 9), (31, 45))]


@pytest.mark.parametrize("ssz,dsz", SIZES)
@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
def test_resize_u8(cvb, oracle, rng, ssz, dsz, cn, interp):
    img = rand_u8(rng, ssz[0], ssz[1], cn)
    want = oracle.resize(img, (dsz[1], dsz[0]), interp)
    got = cpu(cvb.resize(gpu(img), (dsz[1], dsz[0]), interpolation=interp))
    assert_exact(got, want, "resize u8 %s->%s cn=%d interp=%d" % (ssz, dsz, cn, interp))


@pytest.mark.parametrize("ssz,dsz", SIZES)
@pytest.mark.parametrize("cn", [1, 3])
@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
def test_resize_f32(cvb, oracle, rng, ssz, dsz, cn, interp):
    img = rand_u8(rng, ssz[0], ssz[1], cn).astype(np.float32)
    want = oracle.resize(img, (dsz[1], dsz[0]), interp)
    got = cpu(cvb.resize(gpu(img), (dsz[1], dsz[0]), interpolation=interp))
    assert_exact(got, want, "resize f32 %s->%s cn=%d interp=%d" % (ssz, dsz, cn, interp))      # same float operations in the same order
    frac = (rand_u8(rng, ssz[0], ssz[1], cn).astype(np.float32) + 0.37) * 0.731                # non-integer data: rounding shows
    assert_exact(cpu(cvb.resize(gpu(frac), (dsz[1], dsz[0]), interpolation=interp)), oracle.resize(frac, (dsz[1], dsz[0]), interp),
                 "resize f32 (fractional data) %s->%s cn=%d interp=%d" % (ssz, dsz, cn, interp))




@pytest.mark.parametrize("fx,fy", [(0.333, 0.333), (1.7, 0.61), (0.25, 0.5), (2.0, 3.0), (0.4567, 1.234)])
def test_resize_by_factor(cvb, ref, rng, fx, fy):
    """cv::resize(src, dst, Size(), fx, fy): the destination is round(cols*fx) x round(rows*fy) but the sampling scale stays fx, fy -- so
    whenever cols*fx is not an integer the coordinates differ from the dsize form (W=100, fx=0.333: 1/0.333 = 3.003 vs 100/33 = 3.0303).
    Device ABI (torch), host ABI (numpy) and the HAL entry, against the reference called the same way: BIT-EXACT."""
    from opencv_b200 import hal
    for shape, dt in (((100, 131, 3), np.uint8), ((77, 100), np.uint8), ((60, 90), np.float32)):
        img = (rng.random(shape) * 255).astype(dt)
        for interp in (C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC):
            want = ref.resize_fxfy(img, fx, fy, interp)
            assert_exact(cpu(cvb.resize(gpu(img), None, fx, fy, interp)), want, "resize fx=%g fy=%g interp=%d %s (device ABI)" % (fx, fy, interp, dt.__name__))
            assert_exact(hal.resize(img, None, fx, fy, interp), want, "resize fx=%g fy=%g interp=%d %s (host ABI)" % (fx, fy, interp, dt.__name__))


@pytest.mark.parametrize("interp", [C.INTER_LINEAR, C.INTER_AREA])
def test_resize_half_area(cvb, oracle, rng, interp):
    for cn in (1, 3, 4):
        img = rand_u8(rng, 122, 250, cn)
        assert_exact(cpu(cvb.resize(gpu(img), (125, 61), interpolation=interp)), oracle.resize(img, (125, 61), interp), "half u8 cn=%d" % cn)
        f = img.astype(np.float32)
        assert_exact(cpu(cvb.resize(gpu(f), (125, 61), interpolation=interp)), oracle.resize(f, (125, 61), interp), "half f32 cn=%d" % cn)


@pytest.mark.parametrize("dsize,interp", [((3840, 2160), C.INTER_NEAREST), ((3840, 2160), C.INTER_LINEAR), ((5120, 2880), C.INTER_LINEAR),
                                          ((5120, 2880), C.INTER_CUBIC), ((5120, 2880), C.INTER_NEAREST)])
def test_resize_8k(cvb, ref, rng, dsize, interp):
    """bench.py workload c3 (resize leg): 7680x4320 8UC3 source"""
    img = rand_u8(rng, 4320, 7680, 3)
    assert_exact(cpu(cvb.resize(gpu(img), dsize, interpolation=interp)), ref.resize(img, dsize, interp), "8K -> %s interp %d" % (dsize, interp))


def test_resize_4k_to_8k(cvb, ref, rng):
    img = rand_u8(rng, 2160, 3840, 3)
    for interp in (C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC):
        assert_exact(cpu(cvb.resize(gpu(img), (7680, 4320), interpolation=interp)), ref.resize(img, (7680, 4320), interp), "4K->8K interp %d" % interp)


@pytest.mark.parametrize("cn", [1, 3, 4])
def test_resize_nearest_first_version(cvb, rng, monkeypatch, cn):
    """the per-pixel NEAREST kernel (B200CV_RESIZE_NN_PATH=v1; the default when shrinking, for float and for unaligned images) == the walking kernel"""
    img = gpu(rand_u8(rng, 211, 333, cn))
    for dsz in ((500, 317), (96, 100), (666, 422)):
        monkeypatch.setenv("B200CV_RESIZE_NN_PATH", "walk")
        got = cpu(cvb.resize(img, dsz, interpolation=C.INTER_NEAREST))
        monkeypatch.setenv("B200CV_RESIZE_NN_PATH", "v1")
        assert_exact(cpu(cvb.resize(img, dsz, interpolation=C.INTER_NEAREST)), got, "NEAREST v1 vs walking kernel %s cn=%d" % (dsz, cn))


def _rot(oracle, w, h, ang=7.0, sc=0.9):
    return oracle.getRotationMatrix2D((w / 2.0, h / 2.0), ang, sc) if oracle.has("get_rotation_matrix2d") else \
        np.array([[sc * np.cos(np.deg2rad(ang)), sc * np.sin(np.deg2rad(ang)), 3.0], [-sc * np.sin(np.deg2rad(ang)), sc * np.cos(np.deg2rad(ang)), 5.0]])


H0 = np.array([[0.95, 0.02, 5.0], [-0.015, 0.97, 3.0], [1e-5, 2e-5, 1.0]])


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
@pytest.mark.parametrize("border", [C.BORDER_CONSTANT, C.BORDER_REPLICATE, C.BORDER_REFLECT, C.BORDER_REFLECT_101, C.BORDER_WRAP])
def test_warp_affine_u8(cvb, oracle, rng, cn, interp, border):
    img = rand_u8(rng, 131, 157, cn)
    M = _rot(oracle, 157, 131)
    for flags in (interp, interp | C.WARP_INVERSE_MAP):
        want = oracle.warpAffine(img, M, (170, 140), flags, border, (10, 20, 30, 40))
        got = cpu(cvb.warpAffine(gpu(img), M, (170, 140), flags, border, (10, 20, 30, 40)))
        assert_exact(got, want, "warpAffine u8 cn=%d flags=%d border=%d" % (cn, flags, border))


@pytest.mark.parametrize("cn", [1, 3])
@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
@pytest.mark.parametrize("border", [C.BORDER_CONSTANT, C.BORDER_REPLICATE, C.BORDER_REFLECT_101])
def test_warp_perspective_u8(cvb, oracle, rng, cn, interp, border):
    img = rand_u8(rng, 131, 157, cn)
    for flags in (interp, interp | C.WARP_INVERSE_MAP):
        want = oracle.warpPerspective(img, H0, (170, 140), flags, border, (10, 20, 30, 40))
        got = cpu(cvb.warpPerspective(gpu(img), H0, (170, 140), flags, border, (10, 20, 30, 40)))
        assert_exact(got, want, "warpPerspective u8 cn=%d flags=%d border=%d" % (cn, flags, border))


@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
@pytest.mark.parametrize("border", [C.BORDER_CONSTANT, C.BORDER_REPLICATE, C.BORDER_REFLECT])
def test_warp_f32(cvb, oracle, rng, interp, border):
    img = (rand_u8(rng, 131, 157, 1).astype(np.float32) + 0.37) * 0.731
    M = _rot(oracle, 157, 131)
    # float sums in the reference's order (remapBilinear / remapBicubic incl. its two cubic formulas): bit-exact
    assert_exact(cpu(cvb.warpAffine(gpu(img), M, (170, 140), interp, border, 7.5)), oracle.warpAffine(img, M, (170, 140), interp, border, 7.5),
                 "warpAffine f32 interp=%d border=%d" % (interp, border))
    assert_exact(cpu(cvb.warpPerspective(gpu(img), H0, (170, 140), interp, border, 7.5)), oracle.warpPerspective(img, H0, (170, 140), interp, border, 7.5),
                 "warpPerspective f32 interp=%d border=%d" % (interp, border))


@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
@pytest.mark.parametrize("cn", [1, 3])
def test_warp_border_transparent(cvb, ref, rng, interp, cn):
    """BORDER_TRANSPARENT (imgwarp.cpp:373,408 / :788-815 / :925,965-968): destination pixels whose source lies outside keep their previous content;
    a bilinear point inside the image that lacks some of its four neighbours is blended from the ones that exist, re-normalised; a bicubic point
    with its centre inside takes its missing taps by REFLECT_101.  Bit for bit against the reference, 8-bit and float, affine / projective / remap."""
    for dt in (np.uint8, np.float32):
        img = rand_u8(rng, 131, 157, cn)
        img = img if dt == np.uint8 else (img.astype(np.float32) + 0.37) * 0.731
        back = rand_u8(rng, 140, 170, cn)
        back = back if dt == np.uint8 else back.astype(np.float32) * 0.5
        M = _rot(ref, 157, 131)
        want = ref.warpAffine(img, M, (170, 140), interp, C.BORDER_TRANSPARENT, 0, dst=back)
        got = cpu(cvb.warpAffine(gpu(img), M, (170, 140), interp, C.BORDER_TRANSPARENT, 0, dst=gpu(back.copy())))
        assert_exact(got, want, "warpAffine TRANSPARENT %s cn=%d interp=%d" % (np.dtype(dt).name, cn, interp))
        assert (want == back).mean() > 0.02 and (want != back).mean() > 0.3       # both kinds of pixels exist
        want = ref.warpPerspective(img, H0, (170, 140), interp, C.BORDER_TRANSPARENT, 0, dst=back)
        got = cpu(cvb.warpPerspective(gpu(img), H0, (170, 140), interp, C.BORDER_TRANSPARENT, 0, dst=gpu(back.copy())))
        assert_exact(got, want, "warpPerspective TRANSPARENT %s cn=%d interp=%d" % (np.dtype(dt).name, cn, interp))
        yy, xx = np.mgrid[0:140, 0:170].astype(np.float32)
        mx = (xx * 1.05 - 9.3 + 0.02 * yy).astype(np.float32); my = (yy * 0.97 - 4.6 + 0.03 * xx).astype(np.float32)
        want = ref.remap(img, mx, my, interp, C.BORDER_TRANSPARENT, 0, dst=back)
        got = cpu(cvb.remap(gpu(img), gpu(mx), gpu(my), interp, C.BORDER_TRANSPARENT, 0, dst=gpu(back.copy())))
        assert_exact(got, want, "remap TRANSPARENT %s cn=%d interp=%d" % (np.dtype(dt).name, cn, interp))


@pytest.mark.parametrize("cn", [1, 3])
@pytest.mark.parametrize("border", [C.BORDER_CONSTANT, C.BORDER_REPLICATE, C.BORDER_REFLECT_101, C.BORDER_TRANSPARENT])
def test_warp_lanczos4(cvb, ref, rng, cn, border):
    """INTER_LANCZOS4 in warpAffine / warpPerspective / remap (remapLanczos4, imgwarp.cpp:1012-1113; tables initInterTab2D :213-287 with
    interpolateLanczos4 :162-188): 8 x 8 taps, 8-bit fixed point (bit for bit) and float (the reference's summation order; the table's sin / cos
    come from the host's libm on both sides)"""
    for dt in (np.uint8, np.float32):
        img = rand_u8(rng, 131, 157, cn)
        img = img if dt == np.uint8 else (img.astype(np.float32) + 0.37) * 0.731
        back = rand_u8(rng, 140, 170, cn).astype(dt)
        M = _rot(ref, 157, 131)
        kw = dict(dst=back) if border == C.BORDER_TRANSPARENT else {}
        gk = (lambda: dict(dst=gpu(back.copy()))) if border == C.BORDER_TRANSPARENT else (lambda: {})
        want = ref.warpAffine(img, M, (170, 140), C.INTER_LANCZOS4, border, (10, 20, 30, 40), **kw)
        got = cpu(cvb.warpAffine(gpu(img), M, (170, 140), C.INTER_LANCZOS4, border, (10, 20, 30, 40), **gk()))
        assert_exact(got, want, "warpAffine LANCZOS4 %s cn=%d border=%d" % (np.dtype(dt).name, cn, border))
        want = ref.warpPerspective(img, H0, (170, 140), C.INTER_LANCZOS4 | C.WARP_INVERSE_MAP, border, 7, **kw)
        got = cpu(cvb.warpPerspective(gpu(img), H0, (170, 140), C.INTER_LANCZOS4 | C.WARP_INVERSE_MAP, border, 7, **gk()))
        assert_exact(got, want, "warpPerspective LANCZOS4 %s cn=%d border=%d" % (np.dtype(dt).name, cn, border))
        yy, xx = np.mgrid[0:140, 0:170].astype(np.float32)
        mx = (xx * 1.05 - 9.3 + 0.02 * yy).astype(np.float32); my = (yy * 0.97 - 4.6 + 0.03 * xx).astype(np.float32)
        want = ref.remap(img, mx, my, C.INTER_LANCZOS4, border, 5, **kw)
        got = cpu(cvb.remap(gpu(img), gpu(mx), gpu(my), C.INTER_LANCZOS4, border, 5, **gk()))
        assert_exact(got, want, "remap LANCZOS4 %s cn=%d border=%d" % (np.dtype(dt).name, cn, border))


def test_sift_upsample_warp(cvb, oracle, rng):
    """the 2x upsample SIFT uses: warpAffine(INTER_LINEAR | WARP_INVERSE_MAP, BORDER_REFLECT) on f32 (sift.dispatch.cpp:196-202)"""
    img = rand_u8(rng, 67, 91, 1).astype(np.float32)
    M = np.array([[0.5, 0, 0], [0, 0.5, 0]])
    want = oracle.warpAffine(img, M, (182, 134), C.INTER_LINEAR | C.WARP_INVERSE_MAP, C.BORDER_REFLECT)
    got = cpu(cvb.warpAffine(gpu(img), M, (182, 134), C.INTER_LINEAR | C.WARP_INVERSE_MAP, C.BORDER_REFLECT))
    assert_exact(got, want, "sift upsample")


@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
def test_warp_8k(cvb, ref, rng, interp):
    """bench.py workload c3 (warp leg): 7680x4320 8UC3, rotation 7 deg x0.9 about the centre; projective H"""
    img = rand_u8(rng, 4320, 7680, 3)
    M = ref.getRotationMatrix2D((3840, 2160), 7.0, 0.9)
    for border in (C.BORDER_CONSTANT, C.BORDER_REPLICATE):
        assert_exact(cpu(cvb.warpAffine(gpu(img), M, (7680, 4320), interp, border)), ref.warpAffine(img, M, (7680, 4320), interp, border), "8K affine %d %d" % (interp, border))
    H = np.array([[0.95, 0.02, 50], [-0.015, 0.97, 30], [1e-6, 2e-6, 1]])
    assert_exact(cpu(cvb.warpPerspective(gpu(img), H, (7680, 4320), interp, C.BORDER_CONSTANT)), ref.warpPerspective(img, H, (7680, 4320), interp, C.BORDER_CONSTANT),
                 "8K perspective %d" % interp)


@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
def test_warp_tile_and_direct_paths(cvb, oracle, rng, interp, monkeypatch):
    """The tiled kernel stages each 64x16 tile's source footprint in shared memory; maps whose footprint does not fit (strong
    minification, a horizon inside the image) use the direct gather, per launch or per tile/pixel.  Both must equal the CPU."""
    img = rand_u8(rng, 331, 517, 3)
    f32 = rand_u8(rng, 207, 333).astype(np.float32)
    maps = [
        np.array([[0.8, 0.6, -40.0], [-0.6, 0.8, 120.0]]),        # 37 degree rotation
        np.array([[6.5, 0.3, -100.0], [0.2, 7.0, -50.0]]),        # 7x minification: footprint too large -> direct kernel
        np.array([[-1.0, 0.0, 500.0], [0.0, -1.0, 300.0]]),       # 180 degree flip: decreasing coordinates
    ]
    for M in maps:
        for border in (C.BORDER_CONSTANT, C.BORDER_REFLECT_101):
            flags = interp | C.WARP_INVERSE_MAP
            assert_exact(cpu(cvb.warpAffine(gpu(img), M, (401, 283), flags, border, (9, 8, 7, 6))), oracle.warpAffine(img, M, (401, 283), flags, border, (9, 8, 7, 6)),
                         "warpAffine tile path %s" % M[0])
            assert_close(cpu(cvb.warpAffine(gpu(f32), M, (401, 283), flags, border, 3.0)), oracle.warpAffine(f32, M, (401, 283), flags, border, 3.0),
                         atol=2e-4, what="warpAffine f32 tile path")
    Hs = [np.array([[0.9, 0.1, 5.0], [-0.08, 1.1, 3.0], [4e-4, 3e-4, 1.0]]),
          np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, -8e-3, 1.0]])]       # W crosses zero inside the destination
    for Hm in Hs:
        got = cpu(cvb.warpPerspective(gpu(img), Hm, (401, 283), interp | C.WARP_INVERSE_MAP, C.BORDER_REPLICATE))
        assert_exact(got, oracle.warpPerspective(img, Hm, (401, 283), interp | C.WARP_INVERSE_MAP, C.BORDER_REPLICATE), "warpPerspective tile path")
        monkeypatch.setenv("B200CV_WARP_PATH", "direct")
        assert_exact(got, cpu(cvb.warpPerspective(gpu(img), Hm, (401, 283), interp | C.WARP_INVERSE_MAP, C.BORDER_REPLICATE)), "tile vs direct")
        monkeypatch.delenv("B200CV_WARP_PATH")


def _test_maps(rng, h, w, sw, sh, kind):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    if kind == 0:       # barrel-like distortion reaching outside the source
        cx, cy = w / 2, h / 2
        r2 = ((xx - cx) ** 2 + (yy - cy) ** 2) / (cx * cx)
        mx = (cx + (xx - cx) * (1 + 0.35 * r2)) * sw / w; my = (cy + (yy - cy) * (1 + 0.35 * r2)) * sh / h
    elif kind == 1:     # random scatter
        mx = rng.random((h, w)) * (sw + 40) - 20; my = rng.random((h, w)) * (sh + 40) - 20
    else:               # ties, NaN, values outside short / int
        mx = xx * 1.3 - 7.25; my = yy * 0.7 + 3.5
        mx[0, 0] = np.nan; mx[0, 1] = 1e20; my[0, 2] = -1e20; mx[1, 0] = 40000.4; my[1, 1] = -40000.6; mx[2, :5] = [0.5, 1.5, 2.5, -0.5, -1.5]
    return mx.astype(np.float32), my.astype(np.float32)


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("interp", [C.INTER_NEAREST, C.INTER_LINEAR, C.INTER_CUBIC])
def test_remap(cvb, oracle, rng, cn, interp):
    """cv::remap: float x/y planes, packed CV_32FC2 maps and the fixed-point pair of cv::convertMaps; u8 and f32; every border;
    NaN / out-of-range map values follow x86 cvRound (0x80000000).  Bit-exact."""
    for dt in (np.uint8, np.float32):
        src = (rng.random((97, 131, cn) if cn > 1 else (97, 131)) * 255).astype(dt)
        for kind in (0, 1, 2):
            mx, my = _test_maps(rng, 80, 111, 131, 97, kind)
            for border in (C.BORDER_CONSTANT, C.BORDER_REPLICATE, C.BORDER_REFLECT, C.BORDER_REFLECT_101, C.BORDER_WRAP):
                want = oracle.remap(src, mx, my, interp, border, (9, 8, 7, 6))
                assert_exact(cpu(cvb.remap(gpu(src), gpu(mx), gpu(my), interp, border, (9, 8, 7, 6))), want, "remap planar %s cn=%d kind=%d b=%d" % (dt.__name__, cn, kind, border))
            m12 = np.stack([mx, my], -1)
            assert_exact(cpu(cvb.remap(gpu(src), gpu(m12), None, interp, C.BORDER_REFLECT_101)), oracle.remap(src, m12, None, interp, C.BORDER_REFLECT_101), "remap packed")
            if kind < 2 and oracle.has("convert_maps"):
                oracle.remap(src, mx, my, C.INTER_LINEAR, C.BORDER_REPLICATE)      # the reference fills NNDeltaTab_i with its bilinear table
                xy, fr = oracle.convertMaps(mx, my)
                got = cpu(cvb.remap(gpu(src), gpu(xy), gpu(fr.view(np.int16)), interp, C.BORDER_REPLICATE))
                assert_exact(got, oracle.remap(src, xy, fr, interp, C.BORDER_REPLICATE), "remap fixed-point maps")
    # a batch shares one set of maps
    batch = rng.integers(0, 256, (3, 60, 90, cn), dtype=np.uint8)
    mx, my = _test_maps(rng, 70, 50, 90, 60, 0)
    got = cpu(cvb.remap(gpu(batch), gpu(mx), gpu(my), interp, C.BORDER_REPLICATE))
    for i in range(3):
        assert_exact(got[i] if cn > 1 else got[i, :, :, 0], oracle.remap(batch[i] if cn > 1 else batch[i, :, :, 0], mx, my, interp, C.BORDER_REPLICATE), "remap batch frame %d" % i)


@pytest.mark.parametrize("shape", [(97, 131), (64, 80), (5, 7), (2, 2), (1, 9), (33, 1), (40, 51, 3), (20, 22, 4), (270, 481, 3)])
def test_pyramids(cvb, oracle, rng, shape):
    """cv::pyrDown / cv::pyrUp.  8-bit: bit-exact, every border mode the reference accepts.  Float: bit-exact for pyrUp; for
    pyrDown the reference's first / last columns and vector remainders use its scalar operation order (1 ulp): exact inside, 1e-4 there."""
    for dt in (np.uint8, np.float32):
        src = (rng.random(shape) * 255).astype(dt)
        for b in (C.BORDER_REPLICATE, C.BORDER_REFLECT, C.BORDER_REFLECT_101, C.BORDER_WRAP):
            got = cpu(cvb.pyrDown(gpu(src), borderType=b)); want = oracle.pyrDown(src, b)
            if dt is np.uint8:
                assert_exact(got, want, "pyrDown u8 %s b=%d" % (shape, b))
            else:
                assert_close(got, want, atol=1e-4, rtol=1e-6, what="pyrDown f32 %s b=%d" % (shape, b))
                if want.shape[1] > 12:
                    assert_exact(got[:, 1:want.shape[1] - 8], want[:, 1:want.shape[1] - 8], "pyrDown f32 interior %s b=%d" % (shape, b))
        assert_exact(cpu(cvb.pyrUp(gpu(src))), oracle.pyrUp(src), "pyrUp %s %s" % (dt.__name__, shape))
    batch = rng.integers(0, 256, (3,) + shape + ((1,) if len(shape) == 2 else ()), dtype=np.uint8)
    got = cpu(cvb.pyrDown(gpu(batch)))
    for i in range(3):
        a = batch[i, :, :, 0] if len(shape) == 2 else batch[i]
        assert_exact(got[i, :, :, 0] if len(shape) == 2 else got[i], oracle.pyrDown(a), "pyrDown batch")
