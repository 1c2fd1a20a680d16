"""Canny on the device (opencv_b200/csrc/canny.cu) against the numpy restatement (tests/canny_reference.py), bit for bit.

Every dst is prefilled with 0x5A so a pixel that nothing writes shows up.  The HAL cases need the compiled reference (oracle/_ref) and
skip without it; everything else needs only the GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import canny_reference as cr

pytestmark = pytest.mark.gpu
FILL = 0x5A
TW, TH = 32, 16                                      # canny.cu's tile


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _edges_like(h, w, frames=None):
    import torch
    shape = (h, w) if frames is None else (frames, h, w, 1)
    return torch.full(shape, FILL, dtype=torch.uint8, device="cuda")


def _run(cvb, img, t1, t2, ap=3, l2=False):
    s = _dev(img)
    e = _edges_like(img.shape[0], img.shape[1])
    cvb.Canny(s, t1, t2, e, ap, l2)
    return e.cpu().numpy()


def _check(cvb, img, t1, t2, ap=3, l2=False):
    got = _run(cvb, img, t1, t2, ap, l2)
    want = cr.canny(img, t1, t2, ap, l2)
    assert np.array_equal(got, want), "mismatch %d px (shape %s ap %d l2 %s thr %s %s)" % (int((got != want).sum()), img.shape, ap, l2, t1, t2)


def _thr(ap, lo=40.0, hi=120.0):
    return (lo * 16, hi * 16) if ap == 7 else (lo, hi)


@pytest.mark.parametrize("ap", [3, 5, 7, -1])
@pytest.mark.parametrize("l2", [False, True])
@pytest.mark.parametrize("cn", [1, 2, 3, 4])
def test_matrix(cvb, ap, l2, cn):
    for k, (h, w) in enumerate([(37, 71), (16, 32), (17, 33), (131, 257)]):
        img = cr.test_image(100 + 10 * ap + cn + k, h, w, cn)
        t1, t2 = _thr(ap)
        if ap == -1 and not l2:
            # aperture -1 carries bit 31, which cv::Canny takes for the legacy L2 flag when L2gradient is false: refused
            e = _edges_like(h, w)
            with pytest.raises(cvb.B200cvError):
                cvb.Canny(_dev(img), t1, t2, e, ap, l2)
            assert (e.cpu().numpy() == FILL).all()
            continue
        _check(cvb, img, t1, t2, ap, l2)


def test_small_sizes(cvb):
    for w in range(1, 71):
        for h in (1, 2, 3, 5, 8, 13, 16, 17, 20):
            _check(cvb, cr.test_image(w * 31 + h, h, w, 1), 30, 90, 3, (w + h) % 2 == 1)
    for h in range(1, 21):
        for w in (1, 4, 31, 32, 33):
            _check(cvb, cr.test_image(h * 7 + w, h, w, 3), 30, 90, 5, h % 2 == 0)


def test_tile_boundaries(cvb):
    for h in (TH - 1, TH, TH + 1, 2 * TH - 1, 2 * TH, 2 * TH + 1, 3 * TH + 1):
        for w in (TW - 1, TW, TW + 1, 2 * TW + 1, 3 * TW):
            for ap in (3, 7):
                _check(cvb, cr.test_image(h * 100 + w + ap, h, w, 1), *_thr(ap, 20, 60), ap=ap, l2=ap == 7)


def test_4k_frames(cvb):
    for cn, ap, l2 in ((1, 3, False), (3, 5, True)):
        img = cr.test_image(4000 + cn, 2160, 3840, cn)
        _check(cvb, img, *_thr(ap, 30, 90), ap=ap, l2=l2)


def test_tall_frames(cvb):
    # more tile rows (and final-kernel block rows) than a grid's y dimension could hold: the tiles run along grid x
    img = cr.test_image(4100, 1_100_000, 2, 1)
    _check(cvb, img, 30, 90, 3, False)
    _check(cvb, img[:600_000], 30, 90, 5, True)


@pytest.mark.parametrize("frames", [1, 3, 16])
def test_batches(cvb, frames):
    h, w = 70, 150
    imgs = []
    for f in range(frames):
        kind = f % 4
        if kind == 0:
            a = cr.test_image(500 + f, h, w, 1)
        elif kind == 1:
            a = np.zeros((h, w), np.uint8)                       # blank
        elif kind == 2:
            a = np.full((h, w), 200, np.uint8)
            a[:, w // 2:] = 10
        else:
            a = (np.indices((h, w)).sum(0) % 2 * 255).astype(np.uint8)
        imgs.append(a)
    src = _dev(np.stack(imgs)[..., None])
    e = _edges_like(h, w, frames)
    cvb.Canny(src, 25, 80, e, 3, False)
    got = e.cpu().numpy()[..., 0]
    for f in range(frames):
        assert np.array_equal(got[f], cr.canny(imgs[f], 25, 80, 3, False)), "frame %d" % f


def test_unaligned_source_and_dst_window(cvb):
    import torch
    h, w = 45, 67
    img = cr.test_image(91, h, w, 3)
    big = torch.zeros((h, w + 5, 3), dtype=torch.uint8, device="cuda")
    big[:, 1:w + 1] = _dev(img)
    src = big[:, 1:w + 1]                                     # starts 3 bytes in, rows of (w + 5) * 3 bytes
    dbig = torch.full((h, w + 7), FILL, dtype=torch.uint8, device="cuda")
    dst = dbig[:, 3:w + 3]
    cvb.Canny(src, 30, 100, dst, 3, True)
    out = dbig.cpu().numpy()
    assert np.array_equal(out[:, 3:w + 3], cr.canny(img, 30, 100, 3, True))
    assert (out[:, :3] == FILL).all() and (out[:, w + 3:] == FILL).all()


def test_in_place_8uc1(cvb):
    img = cr.test_image(92, 77, 101, 1)
    t = _dev(img)
    cvb.Canny(t, 30, 100, t, 5, False)
    assert np.array_equal(t.cpu().numpy(), cr.canny(img, 30, 100, 5, False))


def test_checkerboards_and_plateaus(cvb):
    yy, xx = np.mgrid[0:48, 0:80]
    cases = [((xx + yy) % 2 * 255), ((xx // 2 + yy // 2) % 2 * 200), ((xx // 3) % 2 * 180 + 20),
             np.where((xx > 20) & (xx < 50) & (yy > 10) & (yy < 30), 150, 60), np.full((48, 80), 77)]
    for k, c in enumerate(cases):
        img = c.astype(np.uint8)
        for ap in (3, 5, 7, -1):
            for l2 in (False, True):
                if ap == -1 and not l2:
                    continue
                _check(cvb, img, *_thr(ap, 10 + k, 100), ap=ap, l2=l2)


def test_threshold_corner_cases(cvb):
    # swapped, equal, zero, negative and fractional thresholds, L2 thresholds above 32767, and 1e10 (INT_MIN after cvFloor)
    special = [(150.0, 50.0), (100.0, 100.0), (0.0, 0.0), (-5.0, 40.0), (20.5, 70.25), (-30.0, -10.0), (1e10, 1e10), (20.0, 1e10),
               (40000.0, 50000.0), (10.0, 40000.0), (437.0, 131.0)]
    for k, (t1, t2) in enumerate(special):
        for ap in (3, 7):
            for l2 in (False, True):
                _check(cvb, cr.test_image(900 + k, 48, 64, 1), t1, t2, ap, l2)
    img = cr.test_image(950, 30, 40, 3)
    _check(cvb, img, 30, 90, 3 | (1 << 31), False)                # the legacy CV_CANNY_L2_GRADIENT bit


def test_strong_pixels_on_the_border(cvb):
    img = np.full((40, 64), 30, np.uint8)
    img[0, :] = 250
    img[:, 0] = 250
    img[-1, 10:50] = 0
    img[5:35, -1] = 255
    for ap in (3, 7):
        _check(cvb, img, *_thr(ap, 20, 200), ap=ap, l2=True)


# ---- hysteresis through Canny(dx, dy): derivative images that draw exact candidate patterns ---------------------------------------------
def _draw(h, w, pts, strong, weak_val=50, strong_val=100, s=1):
    """derivative images whose NMS ridges are exactly the given points (an L1 magnitude of 2v on each).
    s = 0: pts is an ordered one-pixel path; the gradient is across the path (dy on rows, dx on columns, diagonal at turns).
    s = +-1: every point gets dx = s*v, dy = v (a diagonal direction), for straight diagonal lines."""
    dx = np.zeros((h, w), np.int16)
    dy = np.zeros((h, w), np.int16)
    big = set(strong)
    for i, (y, x) in enumerate(pts):
        v = strong_val if (y, x) in big else weak_val
        if s:
            dx[y, x], dy[y, x] = s * v, v
            continue
        nb = [pts[j] for j in (i - 1, i + 1) if 0 <= j < len(pts)]
        if all(q[0] == y for q in nb):
            dy[y, x] = 2 * v
        elif all(q[1] == x for q in nb):
            dx[y, x] = 2 * v
        else:
            dx[y, x], dy[y, x] = v, v
    return dx, dy


def _derivs(cvb, dx, dy, t1, t2, l2=False):
    e = _edges_like(dx.shape[0], dx.shape[1])
    cvb.Canny(_dev(dx), _dev(dy), t1, t2, e, l2)
    return e.cpu().numpy()


def _spiral(n):
    """square spiral with one empty line between its arms, as an ordered list of points"""
    pts = [(0, 0)]
    t, l, b, r = 0, 0, n - 1, n - 1
    y = x = 0
    while True:
        if l > r or t > b:
            break
        while x < r:
            x += 1; pts.append((y, x))
        while y < b:
            y += 1; pts.append((y, x))
        if b - t < 4 or r - l < 4:
            break
        while x > l:
            x -= 1; pts.append((y, x))
        while y > t + 2:
            y -= 1; pts.append((y, x))
        t += 2; l += 2; b -= 2; r -= 2
    return pts


def test_spiral_across_many_tiles(cvb):
    n = 300
    pts = _spiral(n)
    mask = np.zeros((n, n), np.uint8)
    for p in pts:
        mask[p] = 255
    assert len(set(pts)) == len(pts) and len(pts) > 40000
    dx, dy = _draw(n, n, pts, [pts[-1]], s=0)
    got = _derivs(cvb, dx, dy, 60, 150)
    assert np.array_equal(got, cr.canny_derivs(dx, dy, 60, 150))
    assert np.array_equal(got, mask), "the whole spiral hangs on one strong pixel at its far end"
    # cut once on a straight stretch: exactly the part still joined to the strong pixel stays
    c = len(pts) // 3
    straight = lambda c: (pts[c - 1][0] == pts[c + 1][0] and abs(pts[c - 1][1] - pts[c + 1][1]) == 2) or \
        (pts[c - 1][1] == pts[c + 1][1] and abs(pts[c - 1][0] - pts[c + 1][0]) == 2)
    while not straight(c):
        c += 1
    dx[pts[c]] = dy[pts[c]] = 0
    got = _derivs(cvb, dx, dy, 60, 150)
    want = np.zeros((n, n), np.uint8)
    for p in pts[c + 1:]:
        want[p] = 255
    assert np.array_equal(got, want)
    assert np.array_equal(got, cr.canny_derivs(dx, dy, 60, 150))


def test_weak_components_meeting_at_a_tile_corner(cvb):
    h, w = 3 * TH, 3 * TW
    # down-right diagonal through the corner (TW-1, TH-1) -> (TW, TH): only a diagonal step joins the two tiles
    pts = [(TH - 1 - k, TW - 1 - k) for k in range(8)] + [(TH + k, TW + k) for k in range(8)]
    dx, dy = _draw(h, w, pts, [pts[7]], s=-1)
    got = _derivs(cvb, dx, dy, 60, 150)
    want = np.zeros((h, w), np.uint8)
    for p in pts:
        want[p] = 255
    assert np.array_equal(got, want)
    # the other diagonal: (TW, TH-1) -> (TW-1, TH) across the corner of four tiles
    pts = [(TH - 1 - k, TW + k) for k in range(8)] + [(TH + k, TW - 1 - k) for k in range(8)]
    dx, dy = _draw(h, w, pts, [pts[-1]], s=1)
    got = _derivs(cvb, dx, dy, 60, 150)
    want = np.zeros((h, w), np.uint8)
    for p in pts:
        want[p] = 255
    assert np.array_equal(got, want)
    assert np.array_equal(got, cr.canny_derivs(dx, dy, 60, 150))


def test_derivatives_with_wrap_values(cvb):
    rng = np.random.default_rng(3)
    ext = np.array([-32768, -32767, 32767, 27146, 27147, -27147, 0, 1, -1, 100], np.int16)
    for k in range(24):
        cn = 1 if k % 2 else 3
        h, w = int(rng.integers(1, 60)), int(rng.integers(1, 90))
        shape = (h, w) if cn == 1 else (h, w, cn)
        dx = rng.choice(ext, size=shape) if k % 3 else rng.integers(-32768, 32768, size=shape).astype(np.int16)
        dy = rng.choice(ext, size=shape) if k % 3 else rng.integers(-32768, 32768, size=shape).astype(np.int16)
        l2 = k % 4 >= 2
        t1, t2 = float(rng.uniform(-100, 40000)), float(rng.uniform(-100, 40000))
        assert np.array_equal(_derivs(cvb, dx, dy, t1, t2, l2), cr.canny_derivs(dx, dy, t1, t2, l2)), (k, shape, l2)


def test_image_equals_derivatives_of_device_sobel(cvb):
    for ap in (3, 5, 7, -1):
        for cn in (1, 3):
            img = cr.test_image(300 + ap + cn, 53, 77, cn)
            s = _dev(img)
            scale = 1 / 16.0 if ap == 7 else 1.0
            dx = cvb.Sobel(s, cvb.CV_16S, 1, 0, ap, scale, 0.0, cvb.BORDER_REPLICATE)
            dy = cvb.Sobel(s, cvb.CV_16S, 0, 1, ap, scale, 0.0, cvb.BORDER_REPLICATE)
            t1, t2 = _thr(ap, 30, 90)
            a = _run(cvb, img, t1, t2, ap, True)
            e = _edges_like(53, 77)
            cvb.Canny(dx, dy, t1 / 16 if ap == 7 else t1, t2 / 16 if ap == 7 else t2, e, True)
            assert np.array_equal(a, e.cpu().numpy()), (ap, cn)


def test_launch_count_does_not_depend_on_content(cvb):
    import torch
    n = 300
    pts = _spiral(n)
    dx, dy = _draw(n, n, pts, [pts[-1]], s=0)
    blank = np.zeros((n, n), np.int16)
    counts = []
    for a, b in ((blank, blank), (dx, dy)):
        e = _edges_like(n, n)
        da, db = _dev(a), _dev(b)
        torch.cuda.synchronize()
        n0 = cvb.launch_count()
        cvb.Canny(da, db, 60, 150, e, False)
        counts.append(cvb.launch_count() - n0)
    img_counts = []
    for img in (np.zeros((n, n), np.uint8), cr.test_image(9, n, n, 1)):
        s, e = _dev(img), _edges_like(n, n)
        n0 = cvb.launch_count()
        cvb.Canny(s, 30, 90, e)
        img_counts.append(cvb.launch_count() - n0)
    assert counts[0] == counts[1] == img_counts[0] == img_counts[1] == 4


def test_refusals_leave_dst_untouched(cvb):
    import torch
    L = cvb.lib()
    img = _dev(cr.test_image(1, 20, 30, 1))
    e = _edges_like(20, 30)
    ms, md = cvb.describe(img), cvb.describe(e)
    st = cvb._stream_ptr(None)
    for ap in (0, 1, 2, 4, 9, -3):
        assert L.b200cv_canny(ctypes.byref(ms), ctypes.byref(md), ctypes.c_double(10), ctypes.c_double(20), ap, 0, st) == -2
    assert L.b200cv_canny(ctypes.byref(ms), ctypes.byref(md), ctypes.c_double(10), ctypes.c_double(20), -1, 0, st) == -2
    wrong = torch.full((20, 31), FILL, dtype=torch.uint8, device="cuda")
    mw = cvb.describe(wrong)
    assert L.b200cv_canny(ctypes.byref(ms), ctypes.byref(mw), ctypes.c_double(10), ctypes.c_double(20), 3, 0, st) == -2
    d16 = torch.full((20, 30), FILL, dtype=torch.int16, device="cuda")
    m16 = cvb.describe(d16)
    assert L.b200cv_canny(ctypes.byref(ms), ctypes.byref(m16), ctypes.c_double(10), ctypes.c_double(20), 3, 0, st) == -2
    f32 = cvb.describe(torch.zeros((20, 30), dtype=torch.float32, device="cuda"))
    assert L.b200cv_canny(ctypes.byref(f32), ctypes.byref(md), ctypes.c_double(10), ctypes.c_double(20), 3, 0, st) == 1
    c5 = cvb.describe(torch.zeros((20, 30, 5), dtype=torch.uint8, device="cuda"))
    assert L.b200cv_canny(ctypes.byref(c5), ctypes.byref(md), ctypes.c_double(10), ctypes.c_double(20), 3, 0, st) == 1
    dx = torch.zeros((20, 30), dtype=torch.int16, device="cuda")
    dy_bad = cvb.describe(torch.zeros((20, 29), dtype=torch.int16, device="cuda"))
    mdx = cvb.describe(dx)
    assert L.b200cv_canny_derivs(ctypes.byref(mdx), ctypes.byref(dy_bad), ctypes.byref(md), ctypes.c_double(10), ctypes.c_double(20), 0, st) == -2
    c2 = cvb.describe(torch.zeros((20, 30, 2), dtype=torch.int16, device="cuda"))
    assert L.b200cv_canny_derivs(ctypes.byref(c2), ctypes.byref(c2), ctypes.byref(md), ctypes.c_double(10), ctypes.c_double(20), 0, st) == 1
    torch.cuda.synchronize()
    assert (e.cpu().numpy() == FILL).all() and (wrong.cpu().numpy() == FILL).all() and (d16.cpu().numpy() == FILL).all()


# ---- host entries ---------------------------------------------------------------------------------------------------------------------
def test_host_frames_in_one_call(cvb):
    from opencv_b200 import hal
    imgs = np.stack([cr.test_image(600 + f, 61, 93, 3) for f in range(5)])
    imgs[2] = 0
    out = hal.Canny(imgs, 40, 110, None, 3, True)
    assert out.shape == (5, 61, 93, 1)
    for f in range(5):
        assert np.array_equal(out[f, :, :, 0], cr.canny(imgs[f], 40, 110, 3, True)), f


def test_hal_routes_cv_canny_without_a_second_divide(cvb):
    if not (cr.ref_available("ref") and cr.ref_available("ref_hal")):
        pytest.skip("the reference's Canny wrappers are not built (oracle/_ref)")
    ref, hal = cr.RefCanny("ref"), cr.RefCanny("ref_hal")
    for cn in (1, 3):
        img = cr.test_image(700 + cn, 83, 129, cn)
        # aperture-7 magnitudes of these images are ~1500-4600 after Sobel's 1/16: with one /16 these thresholds cut through them, with a
        # second /16 every maximum would be strong (none of them is a multiple of 16 either)
        for t1, t2 in ((38291.0, 62513.0), (62513.0, 38291.0), (50003.0, 50003.0)):
            want = ref.Canny(img, t1, t2, 7, False)
            n0 = cvb.launch_count()
            got = hal.Canny(img, t1, t2, 7, False)
            assert cvb.launch_count() - n0 >= 4, "cv::Canny did not reach the HAL"
            assert np.array_equal(got, want), (cn, t1, t2)
            assert np.array_equal(got, cr.canny(img, t1, t2, 7, False))
            assert not np.array_equal(got, cr.canny_prepared(img, *sorted((t1 / 256, t2 / 256)), 7, False))
    img = cr.test_image(710, 40, 50, 1)
    assert np.array_equal(hal.Canny(img, 20, 60, 3, True), ref.Canny(img, 20, 60, 3, True))


def test_cpp_gpumat_canny(cvb, tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_canny_host")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "cpp", "test_canny_host.cpp"),
                        "-L" + os.path.join(root, "opencv_b200", "lib"), "-lb200cv", "-Wl,-rpath," + os.path.join(root, "opencv_b200", "lib")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
