"""The numpy restatement of cv::Canny (tests/canny_reference.py) against the reference: its recorded answers everywhere, the compiled
reference where oracle/_ref holds it, and a few cases worked out by hand.  CPU only."""
import os

import numpy as np
import pytest

import canny_reference as cr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "canny_ref.npz")


def _golden_cases():
    z = np.load(GOLDEN)
    P, R, K, O = z["params"], z["refused"], z["packed"], z["offsets"]
    for i, (seed, h, w, cn, t1, t2, ap, l2) in enumerate(P):
        h, w = int(h), int(w)
        out = None if R[i] else np.unpackbits(K[O[i]:O[i + 1]])[:h * w].reshape(h, w)
        yield (int(seed), h, w, int(cn), float(t1), float(t2), int(ap), bool(l2)), out


def test_golden_file_is_small_and_covers_the_matrix():
    assert os.path.getsize(GOLDEN) < 500_000
    seen = {(c[6], c[7], c[3]) for c, _ in _golden_cases()}
    for ap in (3, 5, 7, -1):
        for l2 in (False, True):
            for cn in (1, 3):
                assert (ap, l2, cn) in seen


def test_restatement_equals_recorded_reference():
    n = 0
    for (seed, h, w, cn, t1, t2, ap, l2), want in _golden_cases():
        img = cr.test_image(seed, h, w, cn)
        if want is None:
            with pytest.raises(cr.CannyArgError):
                cr.canny(img, t1, t2, ap, l2)
            continue
        got = cr.canny(img, t1, t2, ap, l2)
        assert np.array_equal((got > 0).astype(np.uint8), want), (seed, h, w, cn, t1, t2, ap, l2)
        assert set(np.unique(got)) <= {0, 255}
        n += 1
    assert n > 150


def test_scharr_needs_l2():
    # aperture -1 has bit 31 set, which the legacy CV_CANNY_L2_GRADIENT test (canny.cpp:839-844) strips when L2gradient is false
    with pytest.raises(cr.CannyArgError):
        cr.user_args(10, 20, -1, False)
    assert cr.user_args(10, 20, -1, True) == (10.0, 20.0, -1, True)
    assert cr.user_args(10, 20, 3 | (1 << 31), False) == (10.0, 20.0, 3, True)
    assert cr.user_args(160, 32, 7, False) == (2.0, 10.0, 7, False)


def test_cv_floor_model():
    assert cr.cv_floor_x86(2.5) == 2 and cr.cv_floor_x86(-2.5) == -3
    assert cr.cv_floor_x86(1e10) == cr.INT_MIN and cr.cv_floor_x86(-1e10) == cr.INT_MIN
    assert cr.cv_floor_x86(float("nan")) == cr.INT_MIN
    assert cr.cv_floor_x86(2147483647.9) == 2147483647
    assert cr.int_thresholds(40000.0, 50000.0, True) == (32767 * 32767, 32767 * 32767)
    assert cr.int_thresholds(-3.0, 2.5, True) == (-3, 6)


def test_hysteresis_labels_equal_the_stack_flood_fill():
    rng = np.random.default_rng(5)
    for _ in range(40):
        h, w = rng.integers(1, 60, 2)
        cls = rng.choice([0, 1, 2], size=(h, w), p=[0.45, 0.5, 0.05]).astype(np.uint8)
        assert np.array_equal(cr.hysteresis_stack(cls), cr.hysteresis_labels(cls))


def test_hand_step_edge():
    img = np.zeros((8, 10), np.uint8)
    img[:, 5:] = 200
    e = cr.canny(img, 100, 300)
    # |dx| = 800 on columns 4 and 5; the left one wins the NMS tie (m > left, m >= right)
    want = np.zeros((8, 10), np.uint8)
    want[:, 4] = 255
    assert np.array_equal(e, want)


def test_hand_strong_pixel_on_weak_line():
    cls = np.zeros((5, 9), np.uint8)
    cls[2, 1:8] = 1
    cls[2, 7] = 2
    cls[4, 0:3] = 1                       # a second line with no strong pixel stays off
    want = np.zeros((5, 9), np.uint8)
    want[2, 1:8] = 255
    assert np.array_equal(cr.hysteresis_stack(cls), want)


def test_hand_diagonal_only_connection():
    cls = np.zeros((6, 6), np.uint8)
    cls[0, 0] = 2
    for i in range(1, 6):
        cls[i, i] = 1
    cls[5, 0] = 1                         # not connected
    out = cr.hysteresis_stack(cls)
    assert all(out[i, i] == 255 for i in range(6)) and out[5, 0] == 0


# ---- the compiled reference -------------------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not cr.ref_available("ref"), reason="oracle/_ref/libcannyref.so not built (the reference is not available)")


@needs_ref
def test_restatement_equals_live_reference():
    ref = cr.RefCanny("ref")
    rng = np.random.default_rng(11)
    for k in range(120):
        h, w = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        cn = int(rng.choice([1, 2, 3, 4]))
        ap = int(rng.choice([3, 5, 7, -1]))
        l2 = bool(rng.integers(0, 2))
        t1, t2 = float(rng.uniform(-20, 300)), float(rng.uniform(-20, 300))
        if ap == 7:
            t1, t2 = t1 * 16, t2 * 16
        img = cr.test_image(1000 + k, h, w, cn)
        want = ref.Canny(img, t1, t2, ap, l2)
        if want is None:
            with pytest.raises(cr.CannyArgError):
                cr.canny(img, t1, t2, ap, l2)
        else:
            assert np.array_equal(cr.canny(img, t1, t2, ap, l2), want), (k, h, w, cn, ap, l2, t1, t2)


@needs_ref
def test_restatement_equals_live_reference_on_derivatives():
    ref = cr.RefCanny("ref")
    rng = np.random.default_rng(12)
    ext = np.array([-32768, -32767, 32767, 27146, 27147, -27147, 0, 1, -1], np.int16)
    for k in range(60):
        h, w = int(rng.integers(1, 50)), int(rng.integers(1, 50))
        cn = int(rng.choice([1, 3]))
        shape = (h, w) if cn == 1 else (h, w, cn)
        if k % 2:
            dx = rng.choice(ext, size=shape)
            dy = rng.choice(ext, size=shape)
        else:
            dx = rng.integers(-32768, 32768, size=shape).astype(np.int16)
            dy = rng.integers(-32768, 32768, size=shape).astype(np.int16)
        l2 = bool(k % 4 >= 2)
        if not l2:
            # the reference's 128-bit L1 loop takes |-32768| as -32768 and its scalar tail as 32768 (canny.cpp:456-470): the answer
            # depends on where the pixel falls in the row, so -32768 is only checked with L2, where both paths agree
            dx[dx == -32768] = -32767
            dy[dy == -32768] = -32767
        t1, t2 = float(rng.uniform(-100, 40000)), float(rng.uniform(-100, 40000))
        want = ref.CannyDerivs(dx, dy, t1, t2, l2)
        assert np.array_equal(cr.canny_derivs(dx, dy, t1, t2, l2), want), (k, h, w, cn, l2, t1, t2)


def test_gradient_equals_oracle_sobel():
    from oracle.api import Oracle, available
    kind = "ref" if available("ref") else "port" if available("port") else None
    if kind is None:
        pytest.skip("no Sobel oracle built")
    orc = Oracle(kind)
    for ap in (3, 5, 7, -1):
        for cn in (1, 3):
            img = cr.test_image(77 + ap, 37, 53, cn)
            dx, dy = cr.sobel16(img, ap)
            scale = 1 / 16.0 if ap == 7 else 1.0
            ox = orc.Sobel(img, 3, 1, 0, ap, scale, 0.0, 1)
            oy = orc.Sobel(img, 3, 0, 1, ap, scale, 0.0, 1)
            assert np.array_equal(dx.reshape(ox.shape), ox), (ap, cn)
            assert np.array_equal(dy.reshape(oy.shape), oy), (ap, cn)
