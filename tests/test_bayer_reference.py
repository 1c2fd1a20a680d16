"""The numpy restatement of Bayer VNG and Bayer-to-GRAY (tests/bayer_reference.py) against the reference over the whole table of
tests/bayer_cases.py, bit for bit: against the live reference where oracle/_ref is built, and always against the SHA-256 of the
reference's answers recorded in tests/golden/bayer_ref.json by tools/make_bayer_golden.py.

tests/test_gpu_bayer_vng.py holds the CUDA kernels to the restatement.  This file also checks, on the CPU, the claims the table is built
on (the `ties` cases put ng == 7 ties in both arms of every pattern, and the arms' factors matter there), and runs the host builds of
bayer_gray_kernel (demosaic.cu, whole) and of the VNG per-pixel core (demosaic_vng.cu: vng_planes, vng_pixel, vng_simd_arm) against the
restatement.
"""
import ctypes
import json
import os

import numpy as np
import pytest

import bayer_cases as bc
import bayer_reference as br
from oracle.api import Oracle, available
from test_kernel_emulation import Mat, build_emulation, build_emulation_raw, mat_of

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bayer_ref.json")
SMALL = [c for c in bc.CASES if c.shape[0] * c.shape[1] <= 10000]


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)["bayer"]


@pytest.fixture(scope="module")
def live_ref():
    return Oracle("ref") if available("ref") else None


def restated(case):
    m = bc.mosaic_of(case)
    return br.vng(m, case.code)[0] if case.kind == "vng" else br.gray(m, case.code)


def test_golden_covers_the_table(golden):
    assert set(golden) == {c.id for c in bc.CASES}


@pytest.mark.parametrize("case", bc.CASES, ids=lambda c: c.id)
def test_restatement_vs_reference(live_ref, golden, case):
    got = restated(case)
    if live_ref is not None:
        want = live_ref.cvtColor(bc.mosaic_of(case), case.code, 3 if case.kind == "vng" else 1)
        bad = np.argwhere(got != want)
        assert len(bad) == 0, "%s: %d elements differ, first at %s" % (case.id, len(bad), tuple(bad[0]))
    assert bc.digest(got) == golden[case.id], "%s: the restatement's result is not the one recorded from the reference" % case.id


# ---- the claims the table is built on ------------------------------------------------------------------------------------------
def test_arm_factors_differ_only_at_seven():
    for ng in range(1, 9):
        assert (br.SCALE_SCALAR[ng] == br.SCALE_SIMD[ng]) == (ng != 7), ng
    d = np.arange(-4080, 4081)
    differ = d[np.rint(d.astype(np.float32) * br.SCALE_SCALAR[7]) != np.rint(d.astype(np.float32) * br.SCALE_SIMD[7])]
    assert len(differ) == 130 and (differ % 7 == 0).all() and ((differ // 7) % 2 == 1).all()


@pytest.mark.parametrize("pat", sorted(bc.PAT))
def test_ties_reach_head_body_and_tail(golden, pat):
    """each `ties` case has pixels where the scalar factor rounds differently in the head (column 2 of a row whose column 2 is green) and
    in the tail, and pixels where the vector-body factor does; swapping the arms' factors changes the digest"""
    case = bc.BY_ID["ties-vng-%s-s%d" % (pat, bc.TIE_SEEDS[pat])]
    m = bc.mosaic_of(case)
    vals, ng, arm = br.vng_sites(m, case.code)
    scalar_ties = np.argwhere((br.vng_sites(m, case.code, scale_scalar=br.SCALE_SIMD)[0] != vals).any(-1))
    simd_ties = np.argwhere((br.vng_sites(m, case.code, scale_simd=br.SCALE_SCALAR)[0] != vals).any(-1))
    assert len(simd_ties) and all(arm[r, x] == br.SIMD and ng[r, x] == 7 for r, x in simd_ties)
    assert all(arm[r, x] == br.SCALAR and ng[r, x] == 7 for r, x in scalar_ties)
    assert any(x == 0 for _, x in scalar_ties), "no tie in a head column"
    assert any(x > 0 for _, x in scalar_ties), "no tie in a tail column"
    swapped = br.vng(m, case.code, scale_scalar=br.SCALE_SIMD, scale_simd=br.SCALE_SCALAR)[0]
    assert bc.digest(swapped) != golden[case.id]


def test_table_reaches_every_arm_start():
    """widths 8-13 and 26-41 give no vector block and a first one for both start columns, and every residue of W - 10 modulo 8"""
    widths = {c.shape[1] for c in bc.CASES if c.kind == "vng" and min(c.shape) >= 8}
    for green_at_2 in (False, True):
        spans = {w: br.simd_columns(w, green_at_2) for w in widths}
        assert any(a == b for a, b in spans.values()) and any(b - a == 8 for a, b in spans.values())
    assert {(w - 10) % 8 for w in widths if 26 <= w <= 41} == set(range(8))
    assert {7, 8} <= {min(c.shape) for c in bc.CASES if c.kind == "vng"}


def test_small_vng_ignores_the_pattern(golden):
    """below 8 pixels the reference demosaics every VNG code as COLOR_BayerRG2BGR: the four patterns' answers are one answer"""
    m = bc.mosaic_of(bc.BY_ID["fb-vng-bg-7x20-rand"])
    outs = {bc.digest(br.vng(m, code)[0]) for code in br.VNG_CODES}
    assert outs == {bc.digest(br.bilinear(m, 1, 0))}
    assert golden["fb-vng-bg-7x20-rand"] == bc.digest(br.bilinear(m, 1, 0))


# ---- the kernels' arithmetic, built for the host -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gray_emu():
    lib = build_emulation("demosaic.cu", "int emu_demosaic_gray(const b200cvMat* s, const b200cvMat* d, int code)",
                          "    return b200cv::demosaic_gray(s, d, code, nullptr);")
    lib.emu_demosaic_gray.argtypes = [ctypes.POINTER(Mat), ctypes.POINTER(Mat), ctypes.c_int]

    def run(m, code):
        dst = np.full(m.shape, 0xCD, m.dtype)
        ms, md = mat_of(m), mat_of(dst)
        depth = 0 if m.dtype == np.uint8 else 2
        ms.type = depth; md.type = depth
        assert lib.emu_demosaic_gray(ctypes.byref(ms), ctypes.byref(md), code) == 0
        return dst
    return run


@pytest.mark.parametrize("case", [c for c in SMALL if c.kind == "gray"], ids=lambda c: c.id)
def test_emulated_gray_kernel_vs_restatement(gray_emu, case):
    m = bc.mosaic_of(case)
    assert np.array_equal(gray_emu(m, case.code), br.gray(m, case.code))


VNG_EMU_BODY = r"""
    using namespace b200cv;
    // the kernel's evaluation order without its tiles: planes of every interior site, then every pixel from its clamped site, whose
    // mosaic row is two below the destination row
    const int green0 = (code - 62) & 1, blue0 = code < 64 ? 0 : 2;
    unsigned short* P = (unsigned short*)calloc((size_t)7 * H * W, sizeof(unsigned short));
    for (int r = 1; r < H - 1; r++)
        for (int c = 1; c < W - 1; c++) vng_planes(m + (size_t)r * W + c, W, P + (size_t)r * W + c, H * W);
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) {
            const int cy = min(max(y, 2), H - 5), cx = min(max(x, 2), W - 3);
            const bool green_at_2 = (((cy - 2) & 1) != 0) != (green0 != 0);
            const bool green = green_at_2 != (((cx - 2) & 1) != 0);
            const int blue = ((cy - 2) & 1) ? blue0 ^ 2 : blue0;
            int c, g, o;
            const bool simd = vng_simd_arm(cx, green_at_2, W);
            vng_pixel(m + (size_t)(cy + 2) * W + cx, W, P + (size_t)(cy + 2) * W + cx, W, H * W, green, simd, c, g, o);
            unsigned char* d = out + ((size_t)y * W + x) * 3;
            d[blue] = (unsigned char)o; d[1] = (unsigned char)g; d[blue ^ 2] = (unsigned char)c;
            arm[(size_t)y * W + x] = simd;
        }
    free(P);
    return 0;"""


@pytest.fixture(scope="module")
def vng_emu():
    lib = build_emulation_raw("demosaic_vng.cu", "int emu_vng(const unsigned char* m, int W, int H, int code, unsigned char* out, int* arm)", VNG_EMU_BODY)

    def run(m, code):
        H, W = m.shape
        out = np.zeros((H, W, 3), np.uint8)
        arm = np.zeros((H, W), np.int32)
        m = np.ascontiguousarray(m)
        assert lib.emu_vng(m.ctypes.data_as(ctypes.c_void_p), W, H, code, out.ctypes.data_as(ctypes.c_void_p), arm.ctypes.data_as(ctypes.c_void_p)) == 0
        return out, arm
    return run


@pytest.mark.parametrize("case", [c for c in SMALL if c.kind == "vng" and min(c.shape) >= 8], ids=lambda c: c.id)
def test_emulated_vng_core_vs_restatement(vng_emu, case):
    m = bc.mosaic_of(case)
    want, _, want_arm = br.vng(m, case.code)
    got, arm = vng_emu(m, case.code)
    assert np.array_equal(arm, want_arm), "arm chosen by vng_simd_arm"
    assert np.array_equal(got, want)
