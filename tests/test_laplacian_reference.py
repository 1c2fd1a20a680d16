"""The plain-C restatement of cv::Laplacian (port_laplacian, oracle/port/port_laplacian.c) against the reference over the whole table of
tests/laplacian_cases.py, bit for bit: always against the SHA-256 of the reference's answers recorded in tests/golden/laplacian_ref.json
by tools/make_laplacian_golden.py, and against the live reference where oracle/_ref/liblapref.so is built.  Bit for bit outside one
region: where the reference's float rows fall into a scalar remainder loop (the last cols*cn mod 8 elements of a row for float sources
at ksize 1, 3 and >= 7, mod 32 for 8-bit sources at ksize >= 7; laplacian_cases.remainder_start), its rounding there depends on how
its compiler contracted each loop, which the port does not restate; those elements are zeroed on both sides.  The float ksize 5
remainder, which the fused kernel's own row formulas cover, is restated and compared.

It also checks, on the CPU, that the restatement is composed as the reference composes it: ksize 1 / 3 is the port's filter2D with the
scaled 3x3 kernel, and ksize >= 5 is sepFilter2D(kd, ks) + sepFilter2D(ks, kd) in the working depth followed by convertTo.
tests/test_gpu_laplacian.py holds the CUDA kernel to the restatement.
"""
import ctypes
import ctypes.util
import json
import os

import numpy as np
import pytest

import laplacian_cases as lc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "laplacian_ref.json")
IMAGES = sorted({c.image.id: c.image for c in lc.CASES}.values(), key=lambda i: i.id)
_fmaf = ctypes.CDLL(ctypes.util.find_library("m")).fmaf          # one rounding, as the reference's v_fma
_fmaf.restype, _fmaf.argtypes = ctypes.c_float, (ctypes.c_float, ctypes.c_float, ctypes.c_float)
K3 = {1: np.array([[0, 1, 0], [1, -4, 1], [0, 1, 0]], np.float32), 3: np.array([[2, 0, 2], [0, -8, 0], [2, 0, 2]], np.float32)}


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)["laplacian"]


def test_golden_covers_the_table(golden):
    assert set(golden) == {c.id for c in lc.CASES}
    for c in lc.CASES:
        assert (golden[c.id] == "refused") == (c.ddepth < 0), c.id


@pytest.mark.parametrize("image", IMAGES, ids=lambda i: i.id)
def test_port_vs_reference(port, golden, image):
    img = lc.image_of(image)
    for c in (c for c in lc.CASES if c.image.id == image.id):
        got = lc.run("port", img, c.ddepth, c.ksize, c.scale, c.delta, c.border)
        if lc.ref_available():
            want = lc.masked(image, c.ksize, lc.run("ref", img, c.ddepth, c.ksize, c.scale, c.delta, c.border))
            assert (got is None) == (want is None), c.id
            if want is not None:
                assert lc.same_bits(lc.masked(image, c.ksize, got), want), "%s: differs from the live reference" % c.id
        assert lc.digest(lc.masked(image, c.ksize, got)) == golden[c.id], "%s: the port's result is not the one recorded from the reference" % c.id


def _convert(v, ddepth, scale, delta):
    """convertTo(ddepth, scale, delta) of a 16S or 32F plane: saturate_cast, or saturate_cast(fma(v, scale, delta))"""
    v = v.astype(np.float32)
    if not (scale == 1 and delta == 0):
        a, b = float(np.float32(scale)), float(np.float32(delta))
        v = np.array([_fmaf(float(x), a, b) for x in v.reshape(-1)], np.float32).reshape(v.shape)
    if ddepth == lc.CV_32F:
        return v
    with np.errstate(invalid="ignore"):
        ok = (v >= -2147483648.0) & (v < 2147483648.0)
        r = np.where(ok, np.rint(np.where(ok, v, 0)), -2147483648.0)
    lo, hi = (0, 255) if ddepth == lc.CV_8U else (-32768, 32767)
    return np.clip(r, lo, hi).astype(lc.NP[ddepth])


def _sobel(n, d):
    p = np.array([1], np.int64)
    for _ in range(n - d - 1):
        p = np.convolve(p, [1, 1])
    for _ in range(d):
        p = np.convolve(p, [-1, 1])
    return p.astype(np.float32)


@pytest.mark.parametrize("image", [i for i in IMAGES if i.fill != "special" and i.shape[0] * i.shape[1] < 1 << 20], ids=lambda i: i.id)
def test_port_is_composed_as_the_reference(port, image):
    img = lc.image_of(image)
    for c in (c for c in lc.CASES if c.image.id == image.id and c.ddepth >= 0):
        got = lc.run("port", img, c.ddepth, c.ksize, c.scale, c.delta, c.border)
        if c.ksize <= 3:
            k = K3[c.ksize] * np.float32(c.scale) if c.scale != 1 else K3[c.ksize]
            want = port.filter2D(img, c.ddepth, k, (-1, -1), c.delta, c.border)
        else:
            kd, ks = _sobel(c.ksize, 2), _sobel(c.ksize, 0)
            w = lc.CV_16S if image.depth == lc.CV_8U and c.ksize <= 5 else lc.CV_32F
            d2x = port.sepFilter2D(img, w, kd, ks, (-1, -1), 0.0, c.border)
            d2y = port.sepFilter2D(img, w, ks, kd, (-1, -1), 0.0, c.border)
            s = np.clip(d2x.astype(np.int32) + d2y, -32768, 32767).astype(np.int16) if w == lc.CV_16S else d2x + d2y
            if c.scale == 1 and c.delta == 0 and lc.NP[c.ddepth] == s.dtype:
                want = s
            else:
                want = _convert(s, c.ddepth, c.scale, c.delta)
        if image.depth == lc.CV_32F and c.ksize == 5:
            # the port's sepFilter2D keeps the general order in the last (w*cn mod 8) elements of a row; port_laplacian restates the
            # reference's scalar remainder there (SymmRowSmallFilter), which test_port_vs_reference holds to the reference
            we = got.shape[1] * image.cn
            v = we - we % 8
            got, want = got.reshape(got.shape[0], we)[:, :v], want.reshape(want.shape[0], we)[:, :v]
        assert lc.same_bits(got, want), c.id
