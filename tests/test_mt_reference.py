"""CPU: the numpy matchTemplate reference of tests/mt_reference.py against the plain-C port (oracle/port/port_features.c) and against
values computed by hand.  The GPU tests of tests/test_gpu_match_template_exact.py hold the device to this reference bit for bit, so it
is checked here first, on every machine.

8-bit images: the port sums the numerator in double (exact for 8-bit data), rounds it to float and normalises it with the same f64
operations in the same order, compiled without FMA contraction: the two must agree bit for bit.  Float images: the port and the
reference add the same f64 products in different orders, so they may differ by one float32 ulp, plus the f64 cancellation that the
normed methods can amplify (bounded with the same terms the GPU bars use)."""
import numpy as np
import pytest

import mt_reference as mt
from util import assert_exact

METHODS = range(6)


def _cases(rng):
    """(image, template) pairs: white noise, a constant template, an exact crop, an all-zero template, a constant image region"""
    img = rng.integers(0, 256, (37, 45), dtype=np.uint8)
    flat = img.copy()
    flat[5:30, 4:28] = 201
    yield img, rng.integers(0, 256, (6, 9), dtype=np.uint8)
    yield img, np.full((5, 7), 77, np.uint8)
    yield img, img[11:19, 20:33].copy()
    yield img, np.zeros((4, 3), np.uint8)
    yield flat, flat[2:9, 1:12].copy()
    yield img, img[:, :].copy()                  # template as large as the image: one result
    yield img[:1], img[:1, 3:9].copy()           # one image row


@pytest.mark.parametrize("method", METHODS)
def test_reference_vs_port_u8(port, rng, method):
    for img, templ in _cases(rng):
        want = port.matchTemplate(img, templ, method)
        got = mt.match_template_ref(img, templ, method).res
        assert_exact(got, want, "mt_reference u8 method=%d image %s templ %s" % (method, img.shape, templ.shape))


@pytest.mark.parametrize("method", METHODS)
def test_reference_vs_port_f32(port, rng, method):
    for img8, templ8 in _cases(rng):
        img = ((img8.astype(np.float32) - 90.5) * np.float32(0.37)).astype(np.float32)
        templ = ((templ8.astype(np.float32) - 90.5) * np.float32(0.37)).astype(np.float32)
        want = port.matchTemplate(img, templ, method)
        ref = mt.match_template_ref(img, templ, method)
        r, a = mt.ccorr_f64(img, templ)
        # both sum the same f64 products in their own order (each within n 2^-53 A of the exact sum), then round to float
        dnum = 2 * templ.size * 2.0 ** -53 * a + 2.0 ** -23 * np.abs(r)
        lim = mt.allowance(ref, dnum, ulps=64)
        bad = np.abs(ref.res.astype(np.float64) - want) > lim
        assert not bad.any(), "mt_reference f32 method=%d image %s templ %s: %d elements differ beyond the bar, first at %s (%r vs %r)" % (
            method, img.shape, templ.shape, bad.sum(), tuple(np.argwhere(bad)[0]), ref.res[bad][0], want[bad][0])


def test_reference_hand_values():
    """known answers: all-255 data, a single pixel template, a perfect match"""
    for w, h in ((1, 1), (65, 508), (179, 369)):
        img = np.full((h + 2, w + 1), 255, np.uint8)
        templ = np.full((h, w), 255, np.uint8)
        r = mt.ccorr_exact(img, templ)
        assert r.shape == (3, 2) and (r == 65025 * w * h).all()
    assert 65025 * 65 * 508 == 2147125500 < 2 ** 31
    assert 65025 * 179 * 369 == 4294966275 < 2 ** 32 and float(np.float32(4294966275)) == 4294966272.0     # w h = 66051
    img = np.arange(12, dtype=np.uint8).reshape(3, 4)
    assert_exact(mt.ccorr_exact(img, np.array([[2]], np.uint8)), 2 * img.astype(np.int64), "1x1 template")
    assert_exact(mt.ccorr_exact(img, np.array([[1, 1]], np.uint8)), img[:, :-1].astype(np.int64) + img[:, 1:], "1x2 template")
    s, q = mt.window_sums(img, 2, 2)
    assert s[0, 0] == 0 + 1 + 4 + 5 and q[2 - 1, 2] == 6 * 6 + 7 * 7 + 10 * 10 + 11 * 11
    # perfect match: SQDIFF 0, CCORR_NORMED and CCOEFF_NORMED 1, SQDIFF_NORMED 0 at the match
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (30, 40), dtype=np.uint8)
    templ = img[7:17, 12:25].copy()
    assert mt.match_template_ref(img, templ, mt.SQDIFF).res[7, 12] == 0
    assert mt.match_template_ref(img, templ, mt.SQDIFF_NORMED).res[7, 12] == 0
    assert mt.match_template_ref(img, templ, mt.CCORR_NORMED).res[7, 12] == 1
    assert mt.match_template_ref(img, templ, mt.CCOEFF_NORMED).res[7, 12] == 1
    # a constant template: CCOEFF_NORMED is 1 everywhere (the reference's flat-template rule); CCOEFF is 0 everywhere
    assert (mt.match_template_ref(img, np.full((3, 3), 9, np.uint8), mt.CCOEFF_NORMED).res == 1).all()
    assert (mt.match_template_ref(img, np.full((3, 3), 9, np.uint8), mt.CCOEFF).res == 0).all()
    # a constant image: every window's variance is 0, so the threshold sets t = 0 and CCOEFF_NORMED gives 0
    img = np.full((20, 20), 40, np.uint8)
    templ = rng.integers(0, 256, (4, 5), dtype=np.uint8)
    assert (mt.match_template_ref(img, templ, mt.CCOEFF_NORMED).res == 0).all()
    assert (mt.match_template_ref(img, templ, mt.CCORR).res == 40 * int(templ.astype(np.int64).sum())).all()


def test_reference_batch(rng):
    """a batch is its frames one by one, and the FFT numerator equals a direct integer sum"""
    imgs = rng.integers(0, 256, (3, 50, 61), dtype=np.uint8)
    templ = rng.integers(0, 256, (9, 14), dtype=np.uint8)
    for method in METHODS:
        b = mt.match_template_ref(imgs, templ, method).res
        for f in range(3):
            assert_exact(b[f], mt.match_template_ref(imgs[f], templ, method).res, "batch frame %d method %d" % (f, method))
    r = mt.ccorr_exact(imgs[0], templ)
    d = sum(int(templ[v, u]) * imgs[0, 5 + v, 7 + u].astype(np.int64) for v in range(9) for u in range(14))
    assert r[5, 7] == d
