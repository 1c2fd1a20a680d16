"""GPU parity: GaussianBlur / sepFilter2D / filter2D / Sobel through the device C ABI vs the CPU oracle.

Tolerances
  u8 GaussianBlur, u8 sepFilter2D (8-bit-exact symmetric taps), u8->s16 integer kernels: BIT-EXACT
  f32 GaussianBlur / sepFilter2D, and 8-bit sepFilter2D through float: BIT-EXACT wherever the reference runs a full SIMD vector
    (same operation order: centre-out small rows, mirrored-pair columns, FMA); the last W*cn mod 8 (float source) / mod 32 (8-bit
    source) elements of each row are the reference's scalar remainder loops: |d| <= 1e-4 + 1e-5 |ref| there (the reference's own
    bar for the whole image: test_filter.cpp:826-830 uses 1e-5 relative).  These bars describe the reference's scalar tails, not
    the kernels: tests/test_gpu_sep_float_exact.py holds every float separable kernel to the C port bit for bit over the whole
    destination (remainder columns, anchors, walked chunks, 8-bit rounding, non-finite pixels)
  filter2D u8: BIT-EXACT below 130 taps (the CPU's direct float sum, reproduced in operation order); <= 1 LSB from 130 taps on, where
    the CPU uses a DFT (its own test allows 2, test_filter.cpp:420-425) and the GPU an exact fixed-point tensor-core correlation.
    Against the reference these bars stay; tests/test_gpu_filter2d_tc_exact.py holds both tensor-core kernels (8-bit: bit for bit;
    float: bit for bit on exactly representable data, a derived per-element bar otherwise) to their own arithmetic, restated in
    tests/f2d_reference.py
"""
import numpy as np
import pytest

from util import assert_close, assert_exact, assert_exact_body, cpu, gpu, rand_u8

pytestmark = pytest.mark.gpu

BORDERS = [0, 1, 2, 3, 4]


@pytest.mark.parametrize("shape", [(97, 131, 1), (61, 77, 3), (33, 300, 1), (270, 520, 1), (5, 7, 1), (64, 64, 4)])
@pytest.mark.parametrize("ks", [(3, 0), (5, 0), (7, 0), (9, 0), (5, 1.1), (11, 2.0), (15, 0), (21, 3.3), (31, 5.0), (0, 1.3)])
def test_gaussian_u8_bitexact(cvb, oracle, rng, shape, ks):
    h, w, cn = shape
    img = rand_u8(rng, h, w, cn)
    k, s = ks
    for b in BORDERS:
        want = oracle.GaussianBlur(img, (k, k), s, s, b)
        got = cpu(cvb.GaussianBlur(gpu(img), (k, k), s, s, b))
        assert_exact(got, want, "GaussianBlur u8 %s k=%d s=%g border=%d" % (shape, k, s, b))


@pytest.mark.parametrize("shape", [(70, 400, 3), (131, 1072, 3), (33, 112, 4), (90, 516, 4)])
@pytest.mark.parametrize("ks", [(3, 0), (5, 0), (7, 1.4), (13, 0), (21, 3.3), (31, 5.0)])
def test_gaussian_u8_multichannel_tma_path(cvb, oracle, rng, shape, ks):
    """8UC3 / 8UC4 rows whose pitch is a multiple of 16 bytes run the IDP kernel on byte elements (taps CN elements apart); several
    tiles per row, every border mode, plus the 8.8 fixed-point sepFilter2D mode.  Bit-exact."""
    h, w, cn = shape
    img = rand_u8(rng, h, w, cn)
    k, s = ks
    for b in BORDERS:
        if b == 3:
            continue                              # BORDER_WRAP stays on the generic kernel
        assert_exact(cpu(cvb.GaussianBlur(gpu(img), (k, k), s, s, b)), oracle.GaussianBlur(img, (k, k), s, s, b),
                     "GaussianBlur u8 %s k=%d s=%g border=%d" % (shape, k, s, b))
    tri = (1 + k // 2 - np.abs(np.arange(k) - k // 2)).astype(np.float32); tri /= tri.sum()
    if np.all(tri * 256 == np.rint(tri * 256)):
        assert_exact(cpu(cvb.sepFilter2D(gpu(img), -1, tri, tri)), oracle.sepFilter2D(img, -1, tri, tri), "sepFilter2D fixed mode %s k=%d" % (shape, k))


def test_gaussian_u8_rect_kernel_and_batch(cvb, oracle, rng):
    imgs = np.stack([rand_u8(rng, 120, 333) for _ in range(3)])[..., None]
    got = cpu(cvb.GaussianBlur(gpu(imgs), (7, 3), 1.2, 0.7, 4))
    for i in range(3):
        want = oracle.GaussianBlur(imgs[i, :, :, 0], (7, 3), 1.2, 0.7, 4)
        assert_exact(got[i, :, :, 0], want, "batch frame %d" % i)


def test_gaussian_u8_1080p_c3(cvb, ref, rng):
    """bench.py workload c1: GaussianBlur 5x5 on one 1920x1080 CV_8UC3 frame"""
    img = rand_u8(rng, 1080, 1920, 3)
    assert_exact(cpu(cvb.GaussianBlur(gpu(img), (5, 5), 0)), ref.GaussianBlur(img, (5, 5), 0), "C1")


@pytest.mark.parametrize("k", [3, 5, 7, 9, 11, 13, 15, 21, 31])
def test_gaussian_u8_4k(cvb, ref, rng, k):
    """bench.py workload c2 (u8 leg) at full size against the real reference"""
    img = rand_u8(rng, 2160, 3840)
    assert_exact(cpu(cvb.GaussianBlur(gpu(img), (k, k), 0)), ref.GaussianBlur(img, (k, k), 0), "4K u8 k=%d" % k)


@pytest.mark.parametrize("shape", [(97, 131, 1), (61, 77, 3), (270, 520, 1)])
@pytest.mark.parametrize("ks", [(3, 0), (5, 0), (7, 1.5), (11, 2.0), (13, 0), (17, 2.5), (27, 3.09), (31, 5.0), (0, 1.6)])
def test_gaussian_f32(cvb, oracle, rng, shape, ks):
    h, w, cn = shape
    img = rand_u8(rng, h, w, cn).astype(np.float32)
    k, s = ks
    for b in (0, 1, 2, 4):
        want = oracle.GaussianBlur(img, (k, k), s, s, b)
        got = cpu(cvb.GaussianBlur(gpu(img), (k, k), s, s, b))
        assert_exact_body(got, want, 8, atol=1e-4, rtol=1e-5, what="GaussianBlur f32 %s k=%d border=%d" % (shape, k, b))


@pytest.mark.parametrize("k", [3, 9, 31])
def test_gaussian_f32_4k(cvb, ref, rng, k):
    img = rand_u8(rng, 2160, 3840).astype(np.float32)
    assert_exact(cpu(cvb.GaussianBlur(gpu(img), (k, k), 0)), ref.GaussianBlur(img, (k, k), 0), "4K f32 k=%d" % k)      # 3840 % 8 == 0: no remainder columns
    assert_exact(cpu(cvb.GaussianBlur(gpu(img), (k, k), 0.3 * k + 0.45)), ref.GaussianBlur(img, (k, k), 0.3 * k + 0.45), "4K f32 k=%d sigma" % k)


def test_sepfilter_variants(cvb, oracle, rng):
    img1 = rand_u8(rng, 97, 131); img3 = rand_u8(rng, 61, 77, 3); f1 = img1.astype(np.float32)
    kx = rng.random(5).astype(np.float32); ky = rng.random(7).astype(np.float32)
    CV_8U, CV_16S, CV_32F = 0, 3, 5
    assert_exact_body(cpu(cvb.sepFilter2D(gpu(f1), -1, kx, ky)), oracle.sepFilter2D(f1, -1, kx, ky), 8, atol=2e-3, rtol=1e-5, what="sep f32 (no symmetry)")
    # u8 -> u8 through float (taps that are not 8-bit exact): same operation order as the reference, bit-exact
    a = cpu(cvb.sepFilter2D(gpu(img1), -1, kx / kx.sum(), ky / ky.sum())); b = oracle.sepFilter2D(img1, -1, kx / kx.sum(), ky / ky.sum())
    assert_exact_body(a, b, 32, atol=1, what="sep u8 float path (no symmetry)")
    g7 = np.exp(-0.5 * ((np.arange(7) - 3) / 1.37) ** 2).astype(np.float32); g7 /= g7.sum()
    d5 = np.array([-0.11, -0.37, 0, 0.37, 0.11], np.float32)
    for img in (img1, img3):
        assert_exact_body(cpu(cvb.sepFilter2D(gpu(img), -1, g7, g7)), oracle.sepFilter2D(img, -1, g7, g7), 32, atol=1, what="sep u8 float path (symmetric)")
        assert_exact_body(cpu(cvb.sepFilter2D(gpu(img), -1, g7, d5, delta=128)), oracle.sepFilter2D(img, -1, g7, d5, delta=128), 32, atol=1,
                          what="sep u8 float path (antisymmetric columns)")
        f = img.astype(np.float32)
        assert_exact_body(cpu(cvb.sepFilter2D(gpu(f), -1, d5, g7, delta=0.25)), oracle.sepFilter2D(f, -1, d5, g7, delta=0.25), 8, atol=1e-3, rtol=1e-5,
                          what="sep f32 antisymmetric small rows")
        assert_exact_body(cpu(cvb.sepFilter2D(gpu(f), -1, g7, d5)), oracle.sepFilter2D(f, -1, g7, d5), 8, atol=1e-3, rtol=1e-5, what="sep f32 antisymmetric columns")
    # u8 -> u8 bit-exact mode (symmetric, 8-bit exact) incl. delta and the half-even/half-up split of the reference
    for img in (img1, img3):
        for delta in (0, 3, -2.5):
            a = cpu(cvb.sepFilter2D(gpu(img), -1, [.25, .5, .25], [.125, .75, .125], delta=delta))
            b = oracle.sepFilter2D(img, -1, [.25, .5, .25], [.125, .75, .125], delta=delta)
            assert_exact(a, b, "sep u8 bit-exact mode delta=%g %s" % (delta, img.shape))
    assert_exact_body(cpu(cvb.sepFilter2D(gpu(img1), CV_32F, kx, ky, delta=1.5, borderType=1)),
                      oracle.sepFilter2D(img1, CV_32F, kx, ky, delta=1.5, borderType=1), 32, atol=2e-3, rtol=1e-5, what="sep u8->f32")
    assert_exact_body(cpu(cvb.sepFilter2D(gpu(img1), CV_32F, g7, g7, delta=1.5)), oracle.sepFilter2D(img1, CV_32F, g7, g7, delta=1.5), 32, atol=2e-3, rtol=1e-5,
                      what="sep u8->f32 symmetric")
    # anchors / even sizes go to the generic kernel
    kx4 = rng.random(4).astype(np.float32)
    assert_close(cpu(cvb.sepFilter2D(gpu(f1), -1, kx4, ky, anchor=(1, 5))), oracle.sepFilter2D(f1, -1, kx4, ky, anchor=(1, 5)),
                 atol=2e-3, rtol=1e-5, what="sep anchor")


@pytest.mark.parametrize("k", [3, 5, 9, 15, 31])
def test_sepfilter_u8_fixed_fast_path(cvb, oracle, rng, k):
    """8-bit sepFilter2D with smooth symmetric taps = the reference's 8.8 fixed-point mode (filter.dispatch.cpp:1087-1110); on rows
    that TMA can address it runs on the IDP4A/IDP2A kernel.  The width is not a multiple of 16, so both rounding regimes of the
    reference (vector body half-to-even, scalar tail half-up) are inside the image.  Bit-exact."""
    import torch
    H, W = 203, 344 + 7
    buf = torch.from_numpy(rng.integers(0, 256, (H, 352), dtype=np.uint8)).cuda()
    view = buf[:, :W]                                     # row stride 352: 16-byte aligned rows, ragged width
    img = view.cpu().numpy().copy()
    g = np.exp(-0.5 * ((np.arange(k) - k // 2) / (0.3 * ((k - 1) * 0.5 - 1) + 0.8)) ** 2); g = np.rint(g / g.sum() * 256)
    g[k // 2] += 256 - g.sum(); g = (g / 256).astype(np.float32)          # exact 8-bit taps summing to 1: the reference's bit-exact mode
    tri = (1 + k // 2 - np.abs(np.arange(k) - k // 2)).astype(np.float32); tri /= tri.sum()
    for b in (0, 1, 2, 4):
        assert_exact(cpu(cvb.sepFilter2D(view, -1, g, tri, borderType=b)), oracle.sepFilter2D(img, -1, g, tri, borderType=b), "sep u8 fixed k=%d b=%d" % (k, b))
    # taps that are NOT 8-bit exact: the reference computes in float; TMA float kernel, bit-exact outside the remainder columns
    gs = np.exp(-0.5 * ((np.arange(k) - k // 2) / (0.3 * ((k - 1) * 0.5 - 1) + 0.87)) ** 2).astype(np.float32); gs /= gs.sum()
    for b in (0, 1, 4):
        assert_exact_body(cpu(cvb.sepFilter2D(view, -1, gs, gs, borderType=b)), oracle.sepFilter2D(img, -1, gs, gs, borderType=b), 32, atol=1,
                          what="sep u8 float path, TMA kernel k=%d b=%d" % (k, b))
    # ties are rare on random data: a constant-row image whose exact value is x.5 in every pixel exercises both regimes
    tie = np.zeros((64, 352), np.uint8); tie[:, :] = (np.arange(352) % 2 * 1 + 2)[None, :]
    tbuf = torch.from_numpy(tie).cuda()[:, :W]
    timg = tbuf.cpu().numpy().copy()
    half = np.array([.25, .5, .25], np.float32)
    assert_exact(cpu(cvb.sepFilter2D(tbuf, -1, half, half)), oracle.sepFilter2D(timg, -1, half, half), "sep u8 fixed ties")


@pytest.mark.parametrize("ksize", [1, 3, 5, 7])
def test_sobel(cvb, oracle, rng, ksize):
    img = rand_u8(rng, 97, 131)
    for dx, dy in ((1, 0), (0, 1), (1, 1), (2, 0)):
        if ksize == 1 and dx + dy > 1:
            continue
        assert_exact(cpu(cvb.Sobel(gpu(img), 3, dx, dy, ksize)), oracle.Sobel(img, 3, dx, dy, ksize), "Sobel s16 k%d %d%d" % (ksize, dx, dy))
        a = cpu(cvb.Sobel(gpu(img), 5, dx, dy, ksize, scale=1 / 2040.)); b = oracle.Sobel(img, 5, dx, dy, ksize, scale=1 / 2040.)
        assert_exact_body(a, b, 32, atol=1e-4, rtol=2e-5, what="Sobel u8->f32 k%d %d%d" % (ksize, dx, dy))
        ff = (img.astype(np.float32) + 0.37) * 0.731
        assert_exact_body(cpu(cvb.Sobel(gpu(ff), 5, dx, dy, ksize, scale=0.37, delta=1.5)), oracle.Sobel(ff, 5, dx, dy, ksize, scale=0.37, delta=1.5), 8,
                          atol=2e-2, rtol=1e-4, what="Sobel f32 k%d %d%d" % (ksize, dx, dy))


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("border", [4, 1, 0, 2])
def test_box_filter(cvb, oracle, rng, cn, border):
    """cv::boxFilter / cv::blur (box_filter.simd.hpp): 8U->8U with 16-bit sums + integer divide (area <= 256), 8U->8U with int sums
    (float scale in the SIMD body, double in the last w*cn % 8 elements), 8U->32F (w*cn % 4), 32F->32F with double sums: all bit-exact"""
    for (h, w) in ((97, 131), (64, 200), (33, 37)):
        u8 = rand_u8(rng, h, w, cn)
        f32 = (rng.random(u8.shape, dtype=np.float32) * 255).astype(np.float32)
        for ks in ((3, 3), (5, 5), (7, 3), (2, 4), (16, 16), (17, 17), (20, 20), (1, 1), (31, 9)):
            for norm in (True, False):
                anchor = (-1, -1) if ks != (7, 3) else (6, 0)
                what = "boxFilter %%s cn=%d %s ks=%s norm=%d border=%d" % (cn, (h, w), ks, norm, border)
                assert_exact(cpu(cvb.boxFilter(gpu(u8), -1, ks, anchor, norm, border)), oracle.boxFilter(u8, -1, ks, anchor, norm, border), what % "8U")
                assert_exact(cpu(cvb.boxFilter(gpu(u8), 5, ks, anchor, norm, border)), oracle.boxFilter(u8, 5, ks, anchor, norm, border), what % "8U->32F")
                assert_exact(cpu(cvb.boxFilter(gpu(f32), -1, ks, anchor, norm, border)), oracle.boxFilter(f32, -1, ks, anchor, norm, border), what % "32F")
    assert_exact(cpu(cvb.blur(gpu(u8), (9, 9))), oracle.blur(u8, (9, 9)), "blur")


def test_box_filter_both_u8_kernels(cvb, oracle, rng, monkeypatch):
    """odd, centred 8U->8U boxes run on the TMA + IDP4A/IDP2A kernel (epilogue modes 2 / 3); B200CV_BOX_PATH=generic keeps them on the
    shared-memory kernel of boxfilter.cu: both must return the reference's bytes, 16-bit-sum and int-sum cases, every channel count"""
    for cn in (1, 3, 4):
        img = rand_u8(rng, 203, 331, cn)                       # 331 * cn % 8 != 0: the double-scaled remainder columns exist
        for ks in ((3, 3), (5, 5), (15, 15), (9, 3), (17, 17), (31, 31), (21, 13)):
            for norm in (True, False):
                for border in (4, 0, 1):
                    want = oracle.boxFilter(img, -1, ks, (-1, -1), norm, border)
                    for path in ("", "generic"):
                        monkeypatch.setenv("B200CV_BOX_PATH", path)
                        assert_exact(cpu(cvb.boxFilter(gpu(img), -1, ks, (-1, -1), norm, border)), want,
                                     "boxFilter path=%r cn=%d ks=%s norm=%d border=%d" % (path, cn, ks, norm, border))


def test_box_filter_batch_4k(cvb, ref, rng):
    """4 frames of 3840x2160 8UC1 in one launch, 5x5 and 21x21 (both sum types), unaligned destination pitch handled by the byte-store path"""
    base = rand_u8(rng, 2160, 3840)
    batch = np.stack([np.roll(base, 7 * i, axis=1) for i in range(4)])[..., None]
    for ks in ((5, 5), (21, 21)):
        out = cpu(cvb.blur(gpu(batch), ks))
        for f in (0, 3):
            assert_exact(out[f, :, :, 0], ref.blur(batch[f, :, :, 0], ks), "blur 4K frame %d %s" % (f, ks))
    odd = rand_u8(rng, 301, 1001)
    assert_exact(cpu(cvb.blur(gpu(odd), (3, 3))), ref.blur(odd, (3, 3)), "blur 1001-wide")


def test_scharr(cvb, oracle, rng):
    """cv::Scharr = cv::Sobel(ksize = FILTER_SCHARR): 3/10/3 smoothing, -1/0/1 derivative (deriv.cpp:468-510)"""
    img = rand_u8(rng, 97, 131); img3 = rand_u8(rng, 61, 77, 3)
    for dx, dy in ((1, 0), (0, 1)):
        for im in (img, img3):
            assert_exact(cpu(cvb.Scharr(gpu(im), 3, dx, dy)), oracle.Sobel(im, 3, dx, dy, -1), "Scharr s16 %d%d" % (dx, dy))
        assert_exact_body(cpu(cvb.Scharr(gpu(img), 5, dx, dy, scale=1 / 4080., delta=0.5)), oracle.Sobel(img, 5, dx, dy, -1, scale=1 / 4080., delta=0.5), 32,
                          atol=1e-4, rtol=2e-5, what="Scharr u8->f32 %d%d" % (dx, dy))
        ff = (img.astype(np.float32) + 0.37) * 0.731
        assert_exact_body(cpu(cvb.Scharr(gpu(ff), 5, dx, dy, scale=0.11)), oracle.Sobel(ff, 5, dx, dy, -1, scale=0.11), 8, atol=1e-2, rtol=1e-4, what="Scharr f32 %d%d" % (dx, dy))


@pytest.mark.parametrize("k", [3, 5, 7, 9, 11, 13, 15, 21, 31])
def test_filter2d(cvb, oracle, rng, k):
    img = rand_u8(rng, 97, 131); f = img.astype(np.float32)
    ker = rng.random((k, k)).astype(np.float32); ker /= ker.sum()
    for b in (0, 1, 2, 4):
        got = cpu(cvb.filter2D(gpu(img), -1, ker, borderType=b)); want = oracle.filter2D(img, -1, ker, borderType=b)
        if k * k < 130:     # the reference evaluates the direct float sum: same operation order here, bit-exact
            assert_exact(got, want, "filter2D u8 k=%d b=%d" % (k, b))
        else:               # the reference switches to a float DFT (filter.dispatch.cpp:1288): +-1 LSB at ties
            assert_close(got, want, atol=1, what="filter2D u8 k=%d b=%d" % (k, b))
        gotf = cpu(cvb.filter2D(gpu(f), -1, ker, borderType=b)); wantf = oracle.filter2D(f, -1, ker, borderType=b)
        if k * k < 130:     # direct sum on both sides: bit-exact outside the reference's scalar remainder columns
            assert_exact_body(gotf, wantf, 8, atol=5e-4, rtol=1e-5, what="filter2D f32 k=%d b=%d" % (k, b))
            assert_exact(cpu(cvb.filter2D(gpu(img), 5, ker, delta=0.75, borderType=b)), oracle.filter2D(img, 5, ker, delta=0.75, borderType=b), "filter2D u8->f32 k=%d" % k) \
                if k * k < 50 else None
        else:               # reference = float DFT, GPU = 3 x BF16 on the tensor cores: the reference's own bar for this regime, 1e-4 of the range (test_filter.cpp:420-425)
            assert_close(gotf, wantf, atol=1e-4 * float(np.abs(wantf).max()), what="filter2D f32 k=%d b=%d" % (k, b))
            assert float(np.abs(gotf - wantf).mean()) <= 2e-5 * float(np.abs(wantf).max()), "filter2D f32 k=%d b=%d: mean error" % (k, b)


def test_filter2d_tensor_core(cvb, oracle, rng, monkeypatch):
    """8-bit filter2D with >= 11x11 taps runs on the tensor-core correlation engine (three base-256 digit planes of the fixed-point
    taps, exact integer MMA).  Checked against the CPU (DFT path) and against our own direct-sum kernel; ragged sizes, several
    M/N tiles and frames, signed taps, off-centre anchor, delta, every destination depth."""
    import os
    img = rng.integers(0, 256, (3, 301, 263, 1), dtype=np.uint8)       # batch of 3 frames, > 1 M-tile pair and > 4 N-tiles
    for (kh, kw), anchor, delta in (((11, 13), (-1, -1), 0.0), ((13, 17), (2, 9), 3.5), ((31, 31), (-1, -1), 0.0), ((5, 33), (30, 1), -2.0)):
        ker = (rng.random((kh, kw)).astype(np.float32) - 0.25); ker /= np.abs(ker).sum() * 0.5
        for b in (0, 1, 2, 4):
            got = cpu(cvb.filter2D(gpu(img), -1, ker, anchor=anchor, delta=delta, borderType=b))
            monkeypatch.setenv("B200CV_FILTER2D_PATH", "direct")
            direct = cpu(cvb.filter2D(gpu(img), -1, ker, anchor=anchor, delta=delta, borderType=b))
            monkeypatch.delenv("B200CV_FILTER2D_PATH")
            assert_close(got, direct, atol=1, what="filter2D tc vs direct %dx%d b=%d" % (kh, kw, b))
            assert (got != direct).mean() < 1e-3          # only exact .5 ties may differ
            for i in range(img.shape[0]):
                assert_close(got[i, :, :, 0], oracle.filter2D(img[i, :, :, 0], -1, ker, anchor=anchor, delta=delta, borderType=b), atol=1,
                             what="filter2D tc vs cpu %dx%d b=%d" % (kh, kw, b))
        im0 = np.ascontiguousarray(img[0, :, :, 0])
        ref = oracle.filter2D(im0, 5, ker, anchor=anchor, delta=delta)
        assert_close(cpu(cvb.filter2D(gpu(im0), 5, ker, anchor=anchor, delta=delta)), ref, atol=2e-3, rtol=1e-5, what="filter2D tc u8->f32")
        assert_close(cpu(cvb.filter2D(gpu(im0), 3, ker * 64, anchor=anchor, delta=delta)), oracle.filter2D(im0, 3, ker * 64, anchor=anchor, delta=delta),
                     atol=1, what="filter2D tc u8->s16")


def test_filter2d_tensor_core_f32(cvb, oracle, rng, monkeypatch):
    """float filter2D with >= 130 taps runs 3 x BF16 on the tensor cores (wgmma, FP32 accumulators).  Checked against the CPU (its DFT path) at the
    reference's own bar for that regime (1e-4 of the value range, test_filter.cpp:420-425) and, much tighter on average, against our own
    direct FP32 sum; ragged sizes, several M/N tiles and frames, signed taps, off-centre anchors, delta, non-integer and negative data."""
    img = ((rng.random((3, 301, 263, 1)) - 0.3) * 300).astype(np.float32)
    for (kh, kw), anchor, delta in (((15, 13), (-1, -1), 0.0), ((17, 17), (2, 9), 3.5), ((31, 31), (-1, -1), 0.0), ((21, 33), (30, 1), -2.0), ((33, 5), (1, 30), 0.25),
                                    ((11, 13), (-1, -1), 0.0), ((5, 33), (30, 1), 1.0), ((13, 13), (-1, -1), 0.0), ((33, 33), (0, 32), 0.0), ((19, 1 + 6), (-1, -1), 0.0)):
        ker = (rng.random((kh, kw)).astype(np.float32) - 0.25); ker /= np.abs(ker).sum() * 0.5
        for b in (0, 1, 2, 4):
            got = cpu(cvb.filter2D(gpu(img), -1, ker, anchor=anchor, delta=delta, borderType=b))
            monkeypatch.setenv("B200CV_FILTER2D_PATH", "direct")
            direct = cpu(cvb.filter2D(gpu(img), -1, ker, anchor=anchor, delta=delta, borderType=b))
            monkeypatch.delenv("B200CV_FILTER2D_PATH")
            if kh < 14:         # fewer than 14 kernel rows: the direct FP32 sum is faster and stays (bit-exact path)
                assert_exact(got, direct, "filter2D f32 %dx%d b=%d stays on the direct sum" % (kh, kw, b))
                continue
            scale = float(np.abs(direct).max())
            assert_close(got, direct, atol=1e-4 * scale, what="filter2D f32 tensor cores vs direct %dx%d b=%d" % (kh, kw, b))
            assert float(np.abs(got - direct).mean()) <= 1e-5 * scale, "filter2D f32 tensor cores vs direct %dx%d b=%d: mean error" % (kh, kw, b)
            assert (got != direct).mean() > 0.5, "the tensor-core path did not run (results identical to the direct sum)"
            for i in range(img.shape[0]):
                assert_close(got[i, :, :, 0], oracle.filter2D(img[i, :, :, 0], -1, ker, anchor=anchor, delta=delta, borderType=b), atol=1e-4 * scale,
                             what="filter2D f32 tensor cores vs cpu %dx%d b=%d" % (kh, kw, b))


@pytest.mark.parametrize("ksz", [(3, 3), (5, 5), (9, 9), (7, 3), (3, 13), (21, 21)])
def test_filter2d_tma_path(cvb, oracle, rng, ksz, monkeypatch):
    """single-channel filter2D on TMA-addressable rows (16-byte aligned pitch) runs the TMA tile kernel; identical arithmetic to the
    generic kernels (must agree bit for bit with them) and within the reference's own tolerance of the CPU."""
    import torch
    kw, kh = ksz
    H, W = 131, 421
    buf = torch.from_numpy(rng.integers(0, 256, (2, H, 432, 1), dtype=np.uint8)).cuda()
    view = buf[:, :, :W]
    img = view.cpu().numpy().copy()
    fbuf = torch.from_numpy((rng.random((H, 432)) * 255).astype(np.float32)).cuda()
    fview = fbuf[:, :W]
    fimg = fview.cpu().numpy().copy()
    ker = (rng.random((kh, kw)).astype(np.float32) - 0.2); ker /= np.abs(ker).sum()
    for b in (0, 1, 2, 4):
        got = cpu(cvb.filter2D(view, -1, ker, delta=1.25, borderType=b))
        gotf = cpu(cvb.filter2D(fview, -1, ker, delta=1.25, borderType=b))
        got32 = cpu(cvb.filter2D(view, 5, ker, borderType=b))
        monkeypatch.setenv("B200CV_FILTER2D_PATH", "v1")
        if kw * kh < 130:       # larger 8-bit kernels take the tensor-core path unless told otherwise
            assert_exact(got, cpu(cvb.filter2D(view, -1, ker, delta=1.25, borderType=b)), "filter2D tma vs v1 u8 %s b=%d" % (ksz, b))
            assert_exact(got32, cpu(cvb.filter2D(view, 5, ker, borderType=b)), "filter2D tma vs v1 u8->f32 %s b=%d" % (ksz, b))
        v1f = cpu(cvb.filter2D(fview, -1, ker, delta=1.25, borderType=b))
        if kw * kh < 130:
            assert_exact(gotf, v1f, "filter2D tma vs v1 f32 %s b=%d" % (ksz, b))
        else:               # float images with >= 130 taps run 3 x BF16 on the tensor cores: against our own direct FP32 sum
            assert_close(gotf, v1f, atol=1e-4 * float(np.abs(v1f).max()), what="filter2D tensor cores vs v1 f32 %s b=%d" % (ksz, b))
        monkeypatch.delenv("B200CV_FILTER2D_PATH")
        for i in range(2):
            want = oracle.filter2D(img[i, :, :, 0], -1, ker, delta=1.25, borderType=b)
            if kw * kh < 130:
                assert_exact(got[i, :, :, 0], want, "filter2D tma u8 %s b=%d" % (ksz, b))
            else:
                assert_close(got[i, :, :, 0], want, atol=1, what="filter2D tma u8 %s b=%d" % (ksz, b))
        wantf = oracle.filter2D(fimg, -1, ker, delta=1.25, borderType=b)
        if kw * kh < 130:
            assert_exact_body(gotf, wantf, 8, atol=5e-4, rtol=1e-5, what="filter2D tma f32 %s b=%d" % (ksz, b))
        else:
            assert_close(gotf, wantf, atol=1e-4 * float(np.abs(wantf).max()), what="filter2D tensor cores f32 %s b=%d" % (ksz, b))
        if kw * kh < 50:
            assert_exact(got32[0, :, :, 0], oracle.filter2D(img[0, :, :, 0], 5, ker, borderType=b), "filter2D tma u8->f32 %s b=%d" % (ksz, b))


def test_filter2d_generic(cvb, oracle, rng):
    img3 = rand_u8(rng, 61, 77, 3)
    ker = rng.random((4, 6)).astype(np.float32) - 0.3
    assert_exact(cpu(cvb.filter2D(gpu(img3), -1, ker, anchor=(1, 2), delta=7)), oracle.filter2D(img3, -1, ker, anchor=(1, 2), delta=7), "filter2D generic")
    assert_exact(cpu(cvb.filter2D(gpu(img3), 5, ker)), oracle.filter2D(img3, 5, ker), "filter2D u8->f32 (24 taps: direct sum, scalar order)")


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("width", [32, 48, 131, 512, 528, 1022, 2064])
def test_gaussian_u8_binomial_kernel(cvb, oracle, rng, k, width):
    """3 x 3 / 5 x 5 sigma = 0 on one channel, on views of a wider buffer (16-byte aligned rows): widths that are multiples of 16 run the
    packed 16-bit binomial kernel (gauss_u8_binomial.cu), the others (131, 1022) the TMA tile kernel; every border mode the binomial kernel
    takes; part-filled last warps (48, 528, 2064); equal to the oracle"""
    import torch
    h = 70
    base = gpu(rand_u8(rng, h, ((width + 15) // 16) * 16 + 16))
    view = base[:, :width]
    img = cpu(view)
    outb = torch.zeros_like(base)
    for b in (0, 1, 2, 4):
        want = oracle.GaussianBlur(img, (k, k), 0, 0, b)
        got = cpu(cvb.GaussianBlur(view, (k, k), 0, 0, b, dst=outb[:, :width]))
        assert_exact(got, want, "binomial k=%d w=%d border=%d" % (k, width, b))
