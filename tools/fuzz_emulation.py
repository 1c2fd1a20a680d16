"""Randomised differential test of the host-emulated kernels (tests/test_kernel_emulation.py) against the port: random sizes, channel counts and
codes for ~150 s.  python tools/fuzz_emulation.py   (CPU only; last runs: 33 316 and 22 955 iterations, all outputs equal)"""
import sys, os, numpy as np, ctypes, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import test_kernel_emulation as T
from oracle.api import Oracle
port = Oracle("port")
rng = np.random.default_rng(int(time.time()))
def fx(f):  # unwrap pytest fixture
    return f.__wrapped__() if hasattr(f, "__wrapped__") else f()
two = fx(T.two_plane_emu); mtm = fx(T.mtmask_emu)
yuv = fx(T.yuv_emu); area = fx(T.area_emu); exact = fx(T.exact_emu); lz = fx(T.lanczos_emu); bayer = fx(T.bayer_emu); lab = fx(T.lab_emu)
t0 = time.time(); n = 0
while time.time() - t0 < 150:
    h = int(rng.integers(1, 40)) * 2; w = int(rng.integers(1, 60)) * 2
    img = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    code = int(rng.integers(90, 107))
    assert np.array_equal(yuv(img, code), port.cvtColorYUV(img, code)), ("420", h, w, code)
    y2 = rng.integers(0, 256, (h, w, 2), dtype=np.uint8); code = int(rng.choice([107,108,111,112,115,116,117,118,119,120,121,122,123,124]))
    assert np.array_equal(yuv(y2, code), port.cvtColorYUV(y2, code)), ("422", h, w, code)
    scn = int(rng.choice([3, 4])); b = rng.integers(0, 256, (h, w, scn), dtype=np.uint8)
    code = int(rng.integers(127, 135)); assert np.array_equal(yuv(b, code), port.cvtColorYUV(b, code)), ("to420", h, w, code)
    code = int(rng.integers(143, 155)); assert np.array_equal(yuv(b, code), port.cvtColorYUV(b, code)), ("to422", h, w, code)
    # resizers
    sh, sw = int(rng.integers(1, 90)), int(rng.integers(1, 90)); dh, dw = int(rng.integers(1, 120)), int(rng.integers(1, 120))
    cn = int(rng.choice([1, 3, 4])); shape = (sh, sw) if cn == 1 else (sh, sw, cn)
    u8 = rng.integers(0, 256, shape, dtype=np.uint8); f32 = (rng.random(shape, dtype=np.float32) * 255).astype(np.float32)
    if (dh, dw) != (sh, sw):
        assert np.array_equal(exact(u8, (dw, dh), 5), port.resize(u8, (dw, dh), 5)) or (sh == 2 * dh and sw == 2 * dw), ("lin_exact", sh, sw, dh, dw, cn)
        for im in (u8, f32):
            assert np.array_equal(exact(im, (dw, dh), 6), port.resize(im, (dw, dh), 6)), ("nn_exact", sh, sw, dh, dw, cn)
            assert np.array_equal(lz(im, (dw, dh)), port.resize(im, (dw, dh), 4)), ("lanczos", im.dtype, sh, sw, dh, dw, cn)
            if dh <= sh and dw <= sw and not (sh == 2 * dh and sw == 2 * dw):
                assert np.array_equal(area(im, (dw, dh)), port.resize(im, (dw, dh), 3)), ("area", im.dtype, sh, sw, dh, dw, cn)
    g = rng.integers(0, 256, (max(sh, 3), max(sw, 3)), dtype=np.uint8)
    code = int(rng.choice([46, 47, 48, 49, 139, 140, 141, 142])); assert np.array_equal(bayer(g, code), port.cvtColorYUV(g, code)), ("bayer", g.shape, code)
    c3 = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8); code = int(rng.choice([32,33,34,35,44,45,74,75,56,57,78,79]))
    assert np.array_equal(lab(c3, code), port.cvtColorLab(c3, code)), ("lab", code)
    # two-plane NV12 / NV21, masked matchTemplate
    yp = rng.integers(0, 256, (h, w), dtype=np.uint8); uvp = rng.integers(0, 256, (h // 2, w // 2, 2), dtype=np.uint8); code = int(rng.integers(90, 98))
    assert np.array_equal(two(yp, uvp, code), port.cvtColorTwoPlane(yp, uvp, code)), ("two-plane", h, w, code)
    ih, iw = int(rng.integers(8, 40)), int(rng.integers(8, 40)); th, tw = int(rng.integers(1, ih + 1)), int(rng.integers(1, iw + 1))
    im = rng.integers(0, 256, (ih, iw), dtype=np.uint8); tt = rng.integers(0, 256, (th, tw), dtype=np.uint8)
    mk = (rng.random((th, tw)) > 0.3).astype(np.uint8) if rng.random() < 0.5 else rng.random((th, tw)).astype(np.float32)
    if mk.sum() > 0:
        meth = int(rng.integers(0, 6))
        a, b2 = mtm(im, tt, mk, meth), port.matchTemplateMasked(im, tt, meth, mk)
        assert np.array_equal(a, b2, equal_nan=True), ("masked MT", ih, iw, th, tw, meth)
    n += 1
print("fuzz iterations", n, "all equal")
