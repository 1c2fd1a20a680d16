"""GPU: cv::matchTemplate (no mask) against the exact reference of tests/mt_reference.py, at the tile, size, alignment and accumulator
edges of the two 8-bit numerator kernels (tensor-core ccorr_u8_tc_kernel, IDP4A ccorr_u8_kernel), the two normalisations of 8-bit
results (fused window sums mt_fused_u8_kernel, f64 "planes") and the float numerator (ccorr_f32_kernel).

Which kernels run.  Each case states the numerator kernel it is meant for, and the launch count proves it: TM_CCORR launches two
kernels on the tensor-core path (Toeplitz builder + MMA kernel), one on the IDP4A and float paths; the fused normalisation adds two
(template statistics + fused kernel), the planes one four.  8-bit images reach the tensor-core kernel when base, row step and frame
step are 16-byte aligned, w <= 65, h <= 512 and w h <= 33025; the fused normalisation when they are 4-byte aligned.

Bars.
  8-bit TM_CCORR: bit equality with float32(R), R the exact integer correlation.  Both kernels accumulate exactly (s32 sums stay
      below 2^31 for w h <= 33025, u32 sums below 2^32 for w h <= 66051) and convert to float by rounding to nearest, as the
      reference's (float) cast does.  No tolerance.
  Tensor-core vs IDP4A numerator, fused vs planes normalisation: bit equality, all six methods.  The same integers enter the same
      device code.
  8-bit, the other five methods: the device evaluates common_matchTemplate's f64 formula on the same float32(R) and the same integer
      window and template sums as the reference, in the same order.  The evaluations can differ only where nvcc contracts a multiply
      and an add into one FMA (num - S mean, Q - S^2/n, sum T^2/n - mean^2, ...), which changes that operation by at most one
      rounding of its largest term, 2^-53 |term|.  Let `big` be the largest term magnitude of the numerator formula (R, S mean, Q,
      templSum2) and c = 8 a generous count of such roundings per term.  Then
        non-normed methods:  |d num| <= c 2^-53 big
        normed methods:      r = num / t with t = sqrt(d2) templNorm, d2 = Q - S^2/n.  d2 loses relative accuracy Q / d2 to
                             cancellation, and the CCOEFF template norm loses kappa = (sum T^2/n) / var(T), so
                             |d r| <= c 2^-53 (big / t + |r| (1 + Q / d2 + kappa)).
      Both sides then round to float32, which adds at most one float32 ulp of the result.  Where the threshold
      d2 <= min(0.5, 10 FLT_EPSILON Q) gives t = 0, the result is a constant (0, or 1 for SQDIFF_NORMED) and must match exactly.
      For the windows here, d2 lies far from that threshold compared with its rounding.
  float32 images: the numerator is a chain of n = w h FFMAs, so |R_dev - R| <= gamma_n A per element, where
      A = sum |T| |I| and gamma_n = n 2^-24 / (1 - n 2^-24).  The reference rounds its own f64 sum (within n 2^-53 A of R) to
      float, which adds 2^-24 |R|.  This numerator bound dnum enters the normalisation as above: x1 for CCORR and CCOEFF, x2 for
      SQDIFF (Q - 2R + templSum2), divided by t for the normed methods.  The device's f64 window sums of float data are sliding sums,
      so c grows to 8 (w + h + 64).
mt_reference.allowance computes these bars per element.
"""
import numpy as np
import pytest
import torch

import mt_reference as mt
import opencv_b200 as C
from util import assert_exact, gpu

pytestmark = pytest.mark.gpu

METHODS = range(6)
NUMER_LAUNCHES = {"tc": 2, "dp4a": 1, "f32": 1}
NORM_LAUNCHES = {"fused": 2, "planes": 4}


def _device(frames, off=0, fpad=0):
    """frames (N, H, W) -> a (N, H, W, 1) CUDA view into a wider buffer: each row starts `off` elements into a buffer row whose step is
    a multiple of 16 bytes with at least 4 elements of padding, and each frame starts H rows plus `fpad` elements after the last.
    Everything outside the view holds 255 (8-bit) or 1e6 (float), so a kernel that reads past the image changes the answer."""
    n, h, w = frames.shape
    step = -(-(off + w + 4) // 16) * 16
    fstep = h * step + fpad
    fill = 255 if frames.dtype == np.uint8 else 1e6
    buf = torch.full((n * fstep + step,), fill, dtype=torch.uint8 if frames.dtype == np.uint8 else torch.float32, device="cuda")
    view = buf.as_strided((n, h, w, 1), (fstep, step, 1, 1), off)
    view.copy_(torch.from_numpy(np.ascontiguousarray(frames[..., None])).cuda())
    return view


def _norm_path(off, fpad):
    return "fused" if (off | fpad) % 4 == 0 else "planes"


def _run(cvb, monkeypatch, img, templ, method, force_dp4a=False, planes=False, result=None):
    """result (N, oh, ow) as numpy, and the number of kernels the call launched"""
    with monkeypatch.context() as m:
        if force_dp4a:
            m.setenv("B200CV_MATCHTEMPLATE_PATH", "dp4a")
        if planes:
            m.setenv("B200CV_MATCHTEMPLATE_NORM", "planes")
        torch.cuda.synchronize()
        n0 = cvb.launch_count()
        out = cvb.matchTemplate(img, templ, method, result=result)
        torch.cuda.synchronize()
        n = cvb.launch_count() - n0
    return out[..., 0].cpu().numpy(), n


def _expect_launches(method, numer, norm):
    return NUMER_LAUNCHES[numer] + (0 if method == mt.CCORR else NORM_LAUNCHES[norm])


def _check(got, ref, what, dnum=0.0, ulps=8):
    if ref.method == mt.CCORR and np.ndim(dnum) == 0 and dnum == 0:
        assert_exact(got, ref.res, what)
        return
    assert got.shape == ref.res.shape, "%s: shape %s vs %s" % (what, got.shape, ref.res.shape)
    lim = mt.allowance(ref, dnum, ulps)
    d = np.abs(got.astype(np.float64) - ref.res.astype(np.float64))
    bad = ~(d <= lim)
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d/%d elements beyond the bar, first at %s: got %r want %r (bar %g, t %g)" % (
            what, bad.sum(), d.size, i, got[i], ref.res[i], lim[i], ref.t[i]))


def _u8_case(cvb, monkeypatch, frames, templ, numer, off=0, fpad=0, planes_too=True, what=""):
    """all six methods on the path the layout selects (asserting it), against the reference; then the same with the IDP4A numerator
    forced, and with the planes normalisation, which must be bit-identical; returns the references"""
    img = _device(frames, off, fpad)
    t = gpu(templ)
    norm = _norm_path(off, fpad if frames.shape[0] > 1 else 0)      # one frame: its frame step does not enter the dispatch
    r = mt.ccorr_exact(frames, templ)
    refs = []
    for method in METHODS:
        w = "%s method=%d %s+%s" % (what, method, numer, norm)
        got, n = _run(cvb, monkeypatch, img, t, method)
        assert n == _expect_launches(method, numer, norm), "%s: %d launches, not the %s numerator with the %s normalisation" % (w, n, numer, norm)
        refs.append(mt.match_template_ref(frames, templ, method, r=r))
        _check(got, refs[-1], w)
        if numer == "tc":
            alt, n = _run(cvb, monkeypatch, img, t, method, force_dp4a=True)
            assert n == _expect_launches(method, "dp4a", norm), w + ": the IDP4A numerator did not run"
            assert_exact(alt, got, w + ": IDP4A numerator vs tensor-core numerator")
        if planes_too and norm == "fused" and method != mt.CCORR:
            alt, n = _run(cvb, monkeypatch, img, t, method, planes=True)
            assert n == _expect_launches(method, numer, "planes"), w + ": the planes normalisation did not run"
            assert_exact(alt, got, w + ": planes vs fused normalisation")
    return refs


def _frames(rng, n, oh, ow, h, w):
    return rng.integers(0, 256, (n, oh + h - 1, ow + w - 1), dtype=np.uint8)


# template widths across the tensor-core band (w + 63 <= 128, so w <= 65) and the fixed-width fused kernels (16, 32, 64, 128); ow and oh
# cover mod 64 / mod 256 in {0, 1, ragged}, ow mod 4 in {0, 1, 2, 3}, one result column or row, more than one 128-thread fused block
# (ow > 512), more than one 256-row MMA tile and one 128-row fused segment
WIDTH_CASES = [  # (frames, oh, ow, h, w, numerator)
    (1, 300, 128, 5, 1, "tc"), (1, 256, 129, 1, 2, "tc"), (2, 257, 130, 9, 3, "tc"), (1, 1, 131, 2, 15, "tc"),
    (1, 40, 515, 13, 16, "tc"), (1, 513, 64, 5, 17, "tc"), (1, 129, 77, 1, 31, "tc"), (3, 2, 517, 9, 32, "tc"),
    (1, 260, 1, 2, 33, "tc"), (1, 7, 193, 13, 63, "tc"), (1, 385, 66, 5, 64, "tc"), (2, 64, 3, 1, 65, "tc"),
    (1, 131, 200, 9, 66, "dp4a"), (1, 200, 518, 2, 128, "dp4a"),
]
# template heights: TMA boxes per column chunk go 1 -> 2 -> 3 and the box height drops below 256 (176 rows at h = 258); h = 513 and
# 65 x 509 (w h = 33085 > 33025) fall back to the IDP4A kernel
HEIGHT_CASES = [
    (1, 256, 100, 1, 33, "tc"), (1, 1, 1, 2, 64, "tc"), (1, 257, 1, 255, 7, "tc"), (1, 300, 129, 256, 65, "tc"),
    (1, 600, 65, 257, 1, "tc"), (2, 40, 200, 258, 17, "tc"), (1, 129, 3, 511, 64, "tc"), (1, 1, 66, 512, 40, "tc"),
    (1, 70, 130, 513, 16, "dp4a"), (1, 30, 64, 509, 65, "dp4a"),
]


@pytest.mark.parametrize("case", WIDTH_CASES + HEIGHT_CASES, ids=lambda c: "n%d_o%dx%d_t%dx%d" % (c[0], c[2], c[1], c[4], c[3]))
def test_match_template_u8_shapes(cvb, rng, monkeypatch, case):
    n, oh, ow, h, w, numer = case
    frames = _frames(rng, n, oh, ow, h, w)
    templ = rng.integers(0, 256, (h, w), dtype=np.uint8)
    if n == 1:
        templ = frames[0, oh // 3:oh // 3 + h, ow // 2:ow // 2 + w].copy()      # an exact match somewhere
    _u8_case(cvb, monkeypatch, frames, templ, numer, what="shape %s" % (case,))


# image layouts: (row offset in elements, frame-step padding); row steps are multiples of 16 bytes.  16-byte aligned: tensor-core
# numerator; 4-aligned: IDP4A numerator with the fused normalisation; odd: IDP4A with the planes normalisation.  With the planes hook on
# the aligned layouts (done inside _u8_case), all four pairs of numerator and normalisation run.
LAYOUTS = [((0, 0), "tc"), ((0, 4), "dp4a"), ((0, 1), "dp4a"), ((16, 0), "tc"), ((4, 0), "dp4a"), ((1, 0), "dp4a")]


@pytest.mark.parametrize("layout,numer", LAYOUTS, ids=["aligned", "fstep4", "fstep1", "off16", "off4", "off1"])
@pytest.mark.parametrize("n", [1, 3])
def test_match_template_u8_layouts(cvb, rng, monkeypatch, layout, numer, n):
    frames = _frames(rng, n, 300, 131, 21, 33)
    templ = frames[n - 1, 100:121, 40:73].copy()
    off, fpad = layout
    if n == 1 and off % 16 == 0:
        numer = "tc"                                    # one frame: its frame step does not enter the dispatch
    _u8_case(cvb, monkeypatch, frames, templ, numer, off, fpad, what="layout off=%d fpad=%d n=%d" % (off, fpad, n))


def test_match_template_u8_result_window(cvb, rng, monkeypatch):
    """a result that is a column window of a wider float buffer (rows 4 bytes off 16-byte alignment): the stores stay inside it"""
    n, oh, ow, h, w = 2, 270, 133, 17, 29
    frames = _frames(rng, n, oh, ow, h, w)
    templ = frames[1, 50:50 + h, 60:60 + w].copy()
    img, t = _device(frames), gpu(templ)
    r = mt.ccorr_exact(frames, templ)
    for method in METHODS:
        for force in (False, True):
            base = torch.full((n, oh, ow + 5, 1), -7.0, dtype=torch.float32, device="cuda")
            got, k = _run(cvb, monkeypatch, img, t, method, force_dp4a=force, result=base[:, :, 1:ow + 1])
            numer = "dp4a" if force else "tc"
            assert k == _expect_launches(method, numer, "fused")
            _check(got, mt.match_template_ref(frames, templ, method, r=r), "result window method=%d %s" % (method, numer))
            rest = base.cpu().numpy()
            assert (rest[:, :, 0] == -7).all() and (rest[:, :, ow + 1:] == -7).all(), "stores outside the result window"


@pytest.mark.parametrize("w,h,numer", [(65, 508, "tc"), (257, 257, "dp4a"), (179, 369, "dp4a")])
def test_match_template_u8_accumulator_limit(cvb, monkeypatch, w, h, numer):
    """all-255 image and template: R = 65025 w h, the largest sum each kernel's accumulator must hold (65 x 508: 2 147 125 500 < 2^31
    in s32; 179 x 369 = 66051 pixels: 4 294 966 275 < 2^32 in u32, float 4 294 966 272)"""
    frames = np.full((1, h + 70, w + 67), 255, np.uint8)
    templ = np.full((h, w), 255, np.uint8)
    got, k = _run(cvb, monkeypatch, _device(frames), gpu(templ), mt.CCORR)
    assert k == _expect_launches(mt.CCORR, numer, "fused")
    assert (got == np.float32(65025 * w * h)).all(), "all-255 %dx%d: got %r, want %r" % (w, h, got.flat[0], np.float32(65025 * w * h))
    _u8_case(cvb, monkeypatch, frames, templ, numer, what="all-255 %dx%d" % (w, h))


@pytest.mark.parametrize("w,h", [(257, 258), (196, 337)])
def test_match_template_u8_beyond_accumulator(cvb, w, h):
    """one pixel past w h = 66051 (196 x 337) and beyond: the u32 sums could wrap, so the call is refused and writes nothing"""
    frames = np.full((1, h + 3, w + 5), 255, np.uint8)
    res = torch.full((1, 4, 6, 1), -7.0, dtype=torch.float32, device="cuda")
    with pytest.raises(C.NotImplementedOnDevice):
        cvb.matchTemplate(_device(frames), gpu(np.full((h, w), 255, np.uint8)), mt.CCORR, result=res)
    torch.cuda.synchronize()
    assert (res.cpu().numpy() == -7).all()


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_match_template_template_larger_than_image(cvb, dtype):
    img = gpu(np.zeros((40, 50), dtype))
    res = torch.empty((1, 1), dtype=torch.float32, device="cuda")
    for th, tw in ((41, 10), (10, 51), (41, 51)):
        with pytest.raises(C.NotImplementedOnDevice):
            cvb.matchTemplate(img, gpu(np.ones((th, tw), dtype)), mt.CCORR_NORMED, result=res)


def test_match_template_u8_content(cvb, rng, monkeypatch):
    """content edges: constant image regions (t = 0 by the threshold), a constant template (CCOEFF_NORMED = 1 everywhere), an all-zero
    template, templates cut from the image (exact matches: SQDIFF ~ 0, the normed methods at 1 and through the 1.125 clamp), an inverted
    crop (CCOEFF_NORMED at -1, through the clamp's negative branch), noise"""
    frames = rng.integers(0, 256, (1, 300, 340), dtype=np.uint8)
    frames[0, 40:200, 60:260] = 201
    frames[0, 220:290, 10:120] = 0
    img = frames[0]
    templs = [img[100:124, 20:60], img[230:254, 150:190], img[110:134, 270:310], img[90:114, 40:80],
              img[30:54, 50:90], np.full((24, 40), 77, np.uint8), np.zeros((24, 40), np.uint8),
              rng.integers(0, 256, (24, 40), dtype=np.uint8), img[5:11, 300:305], 255 - img[150:174, 280:320], 255 - img[10:30, 5:45]]
    clamped = clamped_neg = zero_t = 0
    for templ in templs:
        templ = np.ascontiguousarray(templ)
        refs = _u8_case(cvb, monkeypatch, frames, templ, "tc", planes_too=False, what="content templ %s mean %.1f" % (templ.shape, templ.mean()))
        for ref in refs:
            clamped += int(ref.clamp.sum())
            clamped_neg += int((ref.clamp & (ref.res < 0)).sum())
            zero_t += int((ref.t == 0).sum())
    # the cases must reach the special branches of the normalisation
    assert clamped > clamped_neg > 0 and zero_t > 0, (clamped, clamped_neg, zero_t)


def test_match_template_u8_host_api(cvb, rng):
    """the host API: numpy in and out through the upload buffers of the host pipeline (a batch of odd-width frames, uploaded to
    256-byte pitched device rows: the tensor-core numerator)"""
    from opencv_b200 import hal
    frames = rng.integers(0, 256, (3, 211, 337), dtype=np.uint8)
    templ = frames[2, 60:91, 100:143].copy()
    batch = np.empty(frames.shape + (1,), np.uint8)     # (N, H, W, 1) with a dense channel stride
    batch[..., 0] = frames
    r = mt.ccorr_exact(frames, templ)
    for method in (mt.CCORR, mt.SQDIFF, mt.CCOEFF_NORMED):
        n0 = cvb.launch_count()
        got = hal.matchTemplate(batch, templ, method)[..., 0]
        k = cvb.launch_count() - n0
        assert k == _expect_launches(method, "tc", "fused"), "host API method=%d: %d launches" % (method, k)
        _check(got, mt.match_template_ref(frames, templ, method, r=r), "host API method=%d" % method)


def _mixed(rng, shape):
    """non-integer values over four decades, both signs"""
    return ((rng.random(shape) - 0.3) * 10.0 ** rng.uniform(-2, 2, shape)).astype(np.float32)


# (frames, H, W, h, w, row offset): the shape of test_gpu_features' f32 test, ragged multi-frame, more than one 64 x 64 CTA tile
# of ccorr_f32_kernel in each direction, and a template taller than a tile (h > 64)
F32_CASES = [(1, 128, 160, 19, 33, 0), (3, 157, 203, 23, 29, 1), (1, 300, 150, 9, 12, 0), (2, 170, 120, 80, 21, 3)]


@pytest.mark.parametrize("case", F32_CASES, ids=lambda c: "n%d_%dx%d_t%dx%d" % (c[0], c[2], c[1], c[4], c[3]))
def test_match_template_f32(cvb, rng, monkeypatch, case):
    n, H, W, h, w, off = case
    frames = _mixed(rng, (n, H, W))
    templ = _mixed(rng, (h, w))
    if n == 1:
        templ = frames[0, 7:7 + h, 11:11 + w].copy()
    img, t = _device(frames, off), gpu(templ)
    r, a = mt.ccorr_f64(frames, templ)
    k = w * h
    gamma = k * 2.0 ** -24 / (1 - k * 2.0 ** -24)
    dnum = gamma * a + k * 2.0 ** -53 * a + 2.0 ** -24 * np.abs(r)
    for method in METHODS:
        got, nl = _run(cvb, monkeypatch, img, t, method)
        assert nl == _expect_launches(method, "f32", "planes")
        _check(got, mt.match_template_ref(frames, templ, method, r=r), "f32 %s method=%d" % (case, method), dnum=dnum, ulps=8 * (w + h + 64))
