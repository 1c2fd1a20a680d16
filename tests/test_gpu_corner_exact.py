"""GPU: cornerHarris / cornerMinEigenVal and goodFeaturesToTrack held bit for bit to the numpy restatement of harris.cu
(tests/corner_reference.py, itself checked against the plain-C port in tests/test_corner_reference.py).  No reference build is needed.

Response.  Every destination starts as NaN, so a pixel no kernel writes shows up.  The kernels and their switch points (harris.cu):
  - the tile kernel covers 128 x 16 output tiles: the BS = 2 / 3 four-wide path, BS = 5 and the generic run-time box size; it zeroes a
    border product whose interpolated position falls outside its own region, which is safe by a margin of 0 - 1 column at bs 30 / 31
    with REFLECT / REFLECT_101 on a last tile of one column;
  - the register-marching kernel (3-tap Sobel, bs 2 and 3) covers interior 128 x 64 segments: a tile qualifies when x0 >= 128,
    W >= 256 + bs + 6, y0 >= 64 and H >= 128 + bs + 2 (harris_fast_tile); B200CV_HARRIS_PATH=tile puts every tile on the tile kernel.
Both paths are compared with the restatement, not only with each other.

Selection.  gftt_select runs on the device's own cornerHarris / cornerMinEigenVal map (REFLECT_101, the map goodFeaturesToTrack
computes), which the response cases hold exact; positions, order and qualities must all be equal, with the top-K preselection on and
off (B200CV_GFTT_PRESELECT=0).  The 8K noise frames have more than 2^20 local maxima above the quality level: the candidate list must
keep every one of them.
"""
import numpy as np
import pytest
import torch

import corner_reference as cr
from util import assert_exact, cpu

pytestmark = pytest.mark.gpu

BORDERS = [cr.BORDER_CONSTANT, cr.BORDER_REPLICATE, cr.BORDER_REFLECT, cr.BORDER_REFLECT_101]
KSIZES = [1, 3, 5, 7]
BLOCKS = [1, 2, 3, 4, 5, 7, 30, 31]
HF_W, HF_SEG = 128, 64


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _img(rng, shape, dt):
    """smooth structure plus noise, so that responses span many magnitudes; float sources in [0, 1]"""
    n, h, w = shape
    base = np.kron(rng.random((n, h // 6 + 2, w // 6 + 2)), np.ones((1, 6, 6)))[:, :h, :w]
    img = np.clip(base * 200 + rng.random(shape) * 55, 0, 255)
    if dt == np.uint8:
        return img.astype(np.uint8)
    return (img / 255).astype(np.float32)


def _dev(img, col_off=0, extra=0):
    """(N, H, W) numpy -> (N, H, W, 1) device tensor; col_off / extra > 0 make it a column window of a wider buffer (row pitch
    W + col_off + extra elements) whose other columns hold 255 / 7"""
    t = torch.from_numpy(np.ascontiguousarray(img[..., None])).cuda()
    if col_off or extra:
        n, h, w = img.shape
        base = torch.full((n, h, w + col_off + extra, 1), 255 if img.dtype == np.uint8 else 7, dtype=t.dtype, device="cuda")
        base[:, :, col_off:col_off + w] = t
        t = base[:, :, col_off:col_off + w]
    return t


def _nan_dst(n, h, w, col_off=0, extra=0):
    """(buffer, view): a NaN float32 buffer (N, H, W + col_off + extra, 1) and its window at column col_off"""
    buf = torch.full((n, h, w + col_off + extra, 1), float("nan"), dtype=torch.float32, device="cuda")
    return buf, buf[:, :, col_off:col_off + w]


def _call(cvb, op, src, dst, bs, ksize, border):
    if op == 0:
        cvb.cornerHarris(src, bs, ksize, 0.04, border, dst=dst)
    else:
        cvb.cornerMinEigenVal(src, bs, ksize, border, dst=dst)
    torch.cuda.synchronize()


def _check(cvb, img, bs, ksize, border, what="", col_off=0, extra=0, dst_off=0):
    """both responses of img (N, H, W) on the device equal the restatement bit for bit; guard columns of the destination stay NaN"""
    n, h, w = img.shape
    ref = cr.corner_response(img, bs, ksize, border, 0, 0.04)
    src = _dev(img, col_off, extra)
    for op in (0, 1):
        want = ref.res if op == 0 else cr.response32(*ref.sums, 1)
        buf, view = _nan_dst(n, h, w, dst_off, 3 if dst_off else 0)
        _call(cvb, op, src, view, bs, ksize, border)
        got = cpu(buf)[..., 0]
        tag = "%s op %d %s %s bs %d ksize %d border %d %s" % ("Harris" if op == 0 else "MinEig", op, img.dtype, img.shape, bs, ksize, border, what)
        assert not np.isnan(got[:, :, dst_off:dst_off + w]).any(), tag + ": pixels left unwritten"
        assert_exact(_bits(got[:, :, dst_off:dst_off + w]), _bits(want), tag)
        if dst_off:
            assert np.isnan(got[:, :, :dst_off]).all() and np.isnan(got[:, :, dst_off + w:]).all(), tag + ": guard columns written"


def _fast_tiles(w, h, bs):
    """how many 128 x 64 segments harris_fast_kernel owns (harris_fast_tile)"""
    r = bs + 2
    return sum(1 for x0 in range(0, w, HF_W) for y0 in range(0, h, HF_SEG)
               if x0 - r - 4 >= 0 and x0 + HF_W + r + 4 <= w and y0 - r >= 0 and y0 + HF_SEG + r <= h)


# ---- response: tile kernel paths and sizes -------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", [np.uint8, np.float32])
@pytest.mark.parametrize("ksize", KSIZES)
def test_widths(cvb, rng, dt, ksize):
    """widths 1, 2, 3, 127, 128, 129 and 257 (a last tile of one column) at every block size and border: the BS = 2 / 3 four-wide
    path, BS = 5, the generic path, and the bs 30 / 31 product-border margin"""
    for w in (1, 2, 3, 127, 128, 129, 257):
        img = _img(rng, (1, 19, w), dt)
        for bs in BLOCKS:
            for border in BORDERS:
                _check(cvb, img, bs, ksize, border)


@pytest.mark.parametrize("dt", [np.uint8, np.float32])
@pytest.mark.parametrize("ksize", KSIZES)
def test_heights(cvb, rng, dt, ksize):
    """heights 1, 2, 15, 16, 17 and 33 (a last tile of one row)"""
    for h in (1, 2, 15, 16, 17, 33):
        img = _img(rng, (1, h, 131), dt)
        for bs in (1, 2, 3, 5, 7, 31):
            for border in BORDERS:
                _check(cvb, img, bs, ksize, border)


@pytest.mark.parametrize("dt", [np.uint8, np.float32])
@pytest.mark.parametrize("bs", [2, 3])
def test_fast_kernel_thresholds(cvb, rng, monkeypatch, dt, bs):
    """each side of the register-marching kernel's size thresholds (W = 262 + bs, H = 128 + bs + 2), with and without it"""
    ws, hs = (262 + bs - 1, 262 + bs, 262 + bs + 1), (128 + bs + 1, 128 + bs + 2, 128 + bs + 3)
    assert _fast_tiles(ws[0], hs[2], bs) == 0 and _fast_tiles(ws[2], hs[0], bs) == 0 and _fast_tiles(ws[1], hs[1], bs) == 1
    for w in ws:
        for h in hs:
            img = _img(rng, (1, h, w), dt)
            for border in BORDERS:
                _check(cvb, img, bs, 3, border, "W %d H %d" % (w, h))
    monkeypatch.setenv("B200CV_HARRIS_PATH", "tile")
    img = _img(rng, (1, hs[1], ws[1]), dt)
    for border in BORDERS:
        _check(cvb, img, bs, 3, border, "tile path")


@pytest.mark.parametrize("dt", [np.uint8, np.float32])
@pytest.mark.parametrize("bs", [2, 3])
@pytest.mark.parametrize("path", ["default", "tile"])
def test_fast_kernel_frames(cvb, rng, monkeypatch, dt, bs, path):
    """several fast segments in x and y, partial tiles on both edges, 3 frames of different content, and one 600 x 800 frame"""
    if path == "tile":
        monkeypatch.setenv("B200CV_HARRIS_PATH", "tile")
    img = _img(rng, (3, 333, 517), dt)
    assert _fast_tiles(517, 333, bs) > 4
    for border in BORDERS:
        _check(cvb, img, bs, 3, border, path)
    _check(cvb, _img(rng, (1, 600, 800), dt), bs, 3, cr.BORDER_REFLECT_101, path)


@pytest.mark.parametrize("ksize", [3, 5])
def test_order_of_sums(cvb, rng, ksize):
    """faint float texture with isolated pixels of 2^30: around a spike the dx dy products of a box are of order 2^58 and cancel, so
    whether the faint products are added before or after the large ones decides B; the box must be summed in the stated order (rows
    left to right, then top to bottom) on the fast, four-wide and generic paths"""
    for shape in ((1, 40, 300), (1, 150, 300)):
        img = rng.random(shape, dtype=np.float32)
        img[:, 3::9, 4::11] = np.float32(2.0 ** 30)
        for bs in (2, 3, 4, 5, 7, 31):
            for border in BORDERS:
                _check(cvb, img, bs, ksize, border, "spikes")


# ---- response: layout ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", [np.uint8, np.float32])
@pytest.mark.parametrize("bs", [2, 3, 5])
def test_layout(cvb, rng, dt, bs):
    """sources at a column offset of 1 with a row pitch that is not a multiple of 4 (the fast kernel's byte path for 8-bit rows),
    destinations at a column offset into a wider NaN buffer (the scalar store path), both at once, and a batch"""
    img = _img(rng, (3, 200, 300), dt)
    assert _fast_tiles(300, 200, bs) > 0 or bs == 5
    for border in (cr.BORDER_REFLECT_101, cr.BORDER_CONSTANT):
        _check(cvb, img, bs, 3, border, "src +1, pitch 305", col_off=1, extra=4)
        _check(cvb, img, bs, 3, border, "dst +1", dst_off=1)
        _check(cvb, img, bs, 3, border, "src +3 pitch 307, dst +1", col_off=3, extra=4, dst_off=1)
    _check(cvb, img[:, :37, :45], bs, 5, cr.BORDER_REFLECT, "small, src +1", col_off=1, extra=2, dst_off=1)


def test_host_api(cvb, rng):
    """one call through the host API (opencv_b200.hal): numpy in, numpy out, same kernels"""
    from opencv_b200 import hal
    img = _img(rng, (1, 150, 333), np.uint8)[0]
    dst = np.full(img.shape, np.nan, np.float32)
    got = hal.cornerHarris(img, 3, 3, 0.04, cr.BORDER_REFLECT, dst=dst)
    assert_exact(_bits(got), _bits(cr.corner_harris(img, 3, 3, 0.04, cr.BORDER_REFLECT)), "hal.cornerHarris")


def test_refusals(cvb, rng):
    """WRAP, bs 32, Scharr (ksize -1) and even ksize are not implemented; bs 0 is a bad argument; the destination stays untouched"""
    src = _dev(_img(rng, (1, 40, 50), np.uint8))
    for bs, ksize, border in ((3, 3, 3), (32, 3, 4), (3, -1, 4), (3, 2, 4), (3, 4, 4), (3, 9, 4)):
        for op in (0, 1):
            buf, view = _nan_dst(1, 40, 50)
            with pytest.raises(cvb.NotImplementedOnDevice):
                _call(cvb, op, src, view, bs, ksize, border)
            assert np.isnan(cpu(buf)).all(), "bs %d ksize %d border %d: destination written" % (bs, ksize, border)
    buf, view = _nan_dst(1, 40, 50)
    with pytest.raises(cvb.B200cvError) as e:
        _call(cvb, 0, src, view, 0, 3, 4)
    assert not isinstance(e.value, cvb.NotImplementedOnDevice)
    assert np.isnan(cpu(buf)).all()


# ---- goodFeaturesToTrack -----------------------------------------------------------------------------------------------------

def _maps(cvb, src, harris):
    fn = (lambda s: cvb.cornerHarris(s, 3, 3, 0.04, cr.BORDER_REFLECT_101)) if harris else (lambda s: cvb.cornerMinEigenVal(s, 3, 3, cr.BORDER_REFLECT_101))
    return cpu(fn(src))[..., 0]


def _gftt(cvb, monkeypatch, img, mc, q, md, harris, max_out=None, wants=None, check_map=True):
    """goodFeaturesToTrack of img (N, H, W) with the preselection on and off against gftt_select on the device's map; returns the
    selections"""
    src = _dev(img)
    maps = _maps(cvb, src, harris)
    if check_map:
        assert_exact(_bits(maps), _bits(cr.corner_response(img, 3, 3, cr.BORDER_REFLECT_101, 0 if harris else 1).res), "map")
    if wants is None:
        wants = [cr.gftt_select(m, mc, q, md) for m in maps]
    for pre in ("1", "0"):
        monkeypatch.setenv("B200CV_GFTT_PRESELECT", pre)
        got = cvb.goodFeaturesToTrack(src, mc, q, md, 3, 3, harris, 0.04, max_out=max_out, with_quality=True)
        monkeypatch.delenv("B200CV_GFTT_PRESELECT")
        for f, ((gp, gq), (wp, wq)) in enumerate(zip(got, wants)):
            if max_out is not None:
                wp, wq = wp[:max_out], wq[:max_out]
            what = "frame %d of %s harris %s mc %d q %r md %g preselect %s" % (f, img.shape, harris, mc, q, md, pre)
            assert_exact(gp, wp, "corners " + what)
            assert_exact(_bits(gq), _bits(wq), "qualities " + what)
    return wants


@pytest.mark.parametrize("harris", [True, False])
@pytest.mark.parametrize("kind", ["smooth", "noise", "tiled", "mirrored"])
def test_gftt_exact(cvb, rng, monkeypatch, harris, kind):
    """smooth, noise, tiled (exact ties: larger address first, acceptance at exactly min_distance) and mirrored frames; min_distance
    0, 1, 5, 10.5; max_corners 0, 1, 1000 and more than there are candidates; max_out below the count.  A frame mirrored about the
    line between rows 119 and 120 has dx equal and dy negated exactly on the two rows, so their responses tie: local maxima that
    equal a neighbour, which only the non-strict 3x3 test keeps"""
    if kind == "tiled":
        img = np.tile(rng.integers(0, 256, (1, 5, 5), dtype=np.uint8), (1, 48, 64))
    elif kind == "mirrored":
        half = rng.integers(0, 256, (1, 120, 320), dtype=np.uint8)
        img = np.concatenate([half, half[:, ::-1]], axis=1)
    else:
        img = _img(rng, (1, 240, 320), np.uint8) if kind == "smooth" else rng.integers(0, 256, (1, 240, 320), dtype=np.uint8)
    resp = cr.corner_response(img[0], 3, 3, cr.BORDER_REFLECT_101, 0 if harris else 1).res
    vals, pos = cr.gftt_candidates(resp, 0.01)
    ncand = len(vals)
    assert ncand > 100
    if kind == "mirrored":
        assert len(np.intersect1d(pos, pos + 320)) > 5, "candidates with an equal neighbour"
    for md in (0, 1, 5, 10.5):
        for mc in (0, 1, 1000, ncand + 7):
            _gftt(cvb, monkeypatch, img, mc, 0.01, md, harris, check_map=(md == 0 and mc == 0))
    w = _gftt(cvb, monkeypatch, img, 0, 0.01, 5, harris, check_map=False)
    assert len(w[0][0]) > 20
    _gftt(cvb, monkeypatch, img, 0, 0.01, 5, harris, max_out=17, wants=w, check_map=False)


@pytest.mark.parametrize("harris", [True, False])
def test_gftt_threshold_equality(cvb, rng, monkeypatch, harris):
    """a quality level that puts the threshold exactly on a local maximum's value: that maximum is not a corner (TOZERO keeps only
    values strictly above the threshold), while a hair lower level keeps it"""
    img = _img(rng, (1, 240, 320), np.uint8)
    resp = cr.corner_response(img[0], 3, 3, cr.BORDER_REFLECT_101, 0 if harris else 1).res
    mx, _ = cr.gftt_threshold(resp, 0.01)
    vals, pos = cr.gftt_candidates(resp, 0.01)
    found = None
    for v, p in zip(vals[len(vals) // 3:], pos[len(vals) // 3:]):
        q0 = float(v) / float(mx)
        for q in (q0, np.nextafter(q0, 0), np.nextafter(q0, 1), np.nextafter(np.nextafter(q0, 1), 1)):
            if np.float32(float(mx) * q) == v:
                found = (v, p, float(q))
                break
        if found:
            break
    assert found, "no quality level puts the threshold on a candidate"
    v, p, q = found
    assert p not in cr.gftt_candidates(resp, q)[1] and p in cr.gftt_candidates(resp, q * (1 - 1e-6))[1]
    _gftt(cvb, monkeypatch, img, 0, q, 0, harris)
    _gftt(cvb, monkeypatch, img, 0, q * (1 - 1e-6), 0, harris, check_map=False)


def test_gftt_no_corners_and_thin_frames(cvb, rng, monkeypatch):
    """all-zero, constant and ramp frames (max <= 0: no corners); frames of 1 - 3 rows or columns"""
    ramp = np.tile((np.arange(100) * 2).astype(np.uint8), (60, 1))[None]
    for img in (np.zeros((1, 60, 100), np.uint8), np.full((1, 60, 100), 128, np.uint8), ramp):
        for harris in (True, False):
            w = _gftt(cvb, monkeypatch, img, 0, 0.01, 0, harris)
            assert len(w[0][0]) == 0
    for shape in ((1, 1, 40), (1, 2, 40), (1, 3, 40), (1, 40, 1), (1, 40, 2), (1, 40, 3), (1, 3, 3)):
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        for harris in (True, False):
            _gftt(cvb, monkeypatch, img, 0, 0.01, 0, harris)
            _gftt(cvb, monkeypatch, img, 5, 0.01, 1.5, harris, check_map=False)


def test_gftt_batch(cvb, rng, monkeypatch):
    """frames with very different maxima in one batch, and an all-zero frame next to textured ones"""
    img = np.stack([rng.integers(0, 256, (120, 160), dtype=np.uint8), np.zeros((120, 160), np.uint8),
                    (_img(rng, (1, 120, 160), np.uint8)[0] // 16).astype(np.uint8), _img(rng, (1, 120, 160), np.uint8)[0]])
    for harris in (True, False):
        for mc, md in ((50, 5), (0, 0), (300, 10.5)):
            w = _gftt(cvb, monkeypatch, img, mc, 0.01, md, harris, check_map=(mc == 50))
            assert len(w[1][0]) == 0 and all(len(w[f][0]) > 0 for f in (0, 2, 3))


@pytest.mark.parametrize("case", ["prefix runs out", "top cap overflow"])
def test_gftt_4k_preselection(cvb, rng, monkeypatch, case):
    """4K frames: the preselected prefix runs out before max_corners corners are accepted (6000 corners 60 apart on noise), and the
    bins above the preselection threshold hold more than GF_TOP_CAP = 2^17 candidates (a 4 x 4 tiled frame: every tile ties)"""
    if case == "prefix runs out":
        img, mc, md = rng.integers(0, 256, (1, 2160, 3840), dtype=np.uint8), 6000, 60
    else:
        img, mc, md = np.tile(rng.integers(0, 256, (1, 4, 4), dtype=np.uint8), (1, 540, 960)), 1000, 10
    maps = _maps(cvb, _dev(img), True)
    vals, _ = cr.gftt_candidates(maps[0], 0.01)
    if case == "top cap overflow":
        assert (vals == vals[0]).sum() > 2 ** 17
    w = _gftt(cvb, monkeypatch, img, mc, 0.01, md, True, check_map=False)
    assert 0 < len(w[0][0]) < mc if case == "prefix runs out" else len(w[0][0]) == mc


@pytest.mark.parametrize("harris", [True, False])
@pytest.mark.parametrize("frames", [1, 2])
def test_gftt_8k_candidate_overflow(cvb, rng, monkeypatch, harris, frames):
    """7680 x 4320 noise: more than 2^20 local maxima above the quality level in every frame, more than the first candidate list
    holds; every candidate must be kept, so the corners are those of the full list"""
    img = rng.integers(0, 256, (frames, 4320, 7680), dtype=np.uint8)
    maps = _maps(cvb, _dev(img), harris)
    wants = []
    for m in maps:
        assert len(cr.gftt_candidates(m, 0.01)[0]) > 2 ** 20, "the frame no longer overflows the first candidate list"
        wants.append(cr.gftt_select(m, 1000, 0.01, 10))
        assert len(wants[-1][0]) == 1000
    _gftt(cvb, monkeypatch, img, 1000, 0.01, 10, harris, wants=wants, check_map=False)
