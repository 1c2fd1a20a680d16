"""GPU: cv::cvtColor for Bayer VNG (codes 62-65, demosaic_vng.cu) and Bayer to GRAY (86-89, demosaic.cu), bit for bit against the numpy
restatement of tests/bayer_reference.py (which tests/test_bayer_reference.py holds to the reference's recorded answers), over the whole
table of tests/bayer_cases.py; then views, batches, the host path, the launch count and the refusals."""
import numpy as np
import pytest

import bayer_cases as bc
import bayer_reference as br
import opencv_b200 as C
from util import assert_exact, cpu, gpu

pytestmark = [pytest.mark.gpu]


def restated(case, m=None):
    m = bc.mosaic_of(case) if m is None else m
    return br.vng(m, case.code)[0] if case.kind == "vng" else br.gray(m, case.code)


@pytest.mark.parametrize("case", bc.CASES, ids=lambda c: c.id)
def test_case(cvb, case):
    m = bc.mosaic_of(case)
    assert_exact(cpu(cvb.cvtColor(gpu(m), case.code)), restated(case, m), case.id)


VIEWED = [c for c in bc.CASES if c.shape[0] * c.shape[1] <= 10000 and min(c.shape) >= 3]


@pytest.mark.parametrize("case", VIEWED, ids=lambda c: c.id)
def test_views(cvb, case):
    """source and destination as views into larger buffers: rows padded, starting an odd number of pixels in; the elements around the
    destination window must come back unchanged"""
    m = bc.mosaic_of(case)
    want = restated(case, m)
    H, W = m.shape
    cn = 3 if case.kind == "vng" else 1
    for soff, doff in ((3, 1), (1, 5)):
        sbig = np.zeros((H + 2, W + 7), m.dtype)
        sbig[1:1 + H, soff:soff + W] = m
        src = gpu(sbig)[1:1 + H, soff:soff + W]
        expect = np.full((H + 2, (W + 7) * cn), 0x5A, m.dtype)
        expect[1:1 + H, doff * cn:(doff + W) * cn] = want.reshape(H, W * cn)
        dbig = gpu(np.full(expect.shape, 0x5A, m.dtype))
        dst = dbig[1:1 + H, doff * cn:(doff + W) * cn]
        cvb.cvtColor(src, case.code, dst=dst.view(H, W, cn) if cn > 1 else dst)
        assert_exact(cpu(dbig), expect, "%s, views %d / %d pixels in (the window and the elements around it)" % (case.id, soff, doff))


@pytest.mark.parametrize("code,dtype", [(62, np.uint8), (65, np.uint8), (87, np.uint8), (88, np.uint16)])
def test_batch_with_spare_rows(cvb, code, dtype):
    """three frames, each followed by 5 spare rows in both buffers: frame_step is not H * pitch"""
    rng = np.random.default_rng(code)
    H, W, N = 37, 45, 3
    frames = rng.integers(0, 256 if dtype == np.uint8 else 65536, (N, H, W)).astype(dtype)
    cn = 3 if code <= 65 else 1
    sbig = np.zeros((N, H + 5, W, 1), dtype)
    sbig[:, :H, :, 0] = frames
    dbig = gpu(np.full((N, H + 5, W, cn), 0x77, dtype))
    cvb.cvtColor(gpu(sbig)[:, :H], code, dst=dbig[:, :H])
    out = cpu(dbig)
    for f in range(N):
        want = br.vng(frames[f], code)[0] if cn == 3 else br.gray(frames[f], code)
        assert_exact(out[f, :H], want.reshape(H, W, cn), "code %d frame %d" % (code, f))
    assert (out[:, H:] == 0x77).all(), "spare rows between frames were written"


def test_4k_batch(cvb):
    """four 2160 x 3840 mosaics in one call; frames 0 and 3 checked"""
    rng = np.random.default_rng(4)
    batch = rng.integers(0, 256, (4, 2160, 3840, 1), dtype=np.uint8)
    out = cpu(cvb.cvtColor(gpu(batch), C.COLOR_BayerGR2BGR_VNG))
    assert out.shape == (4, 2160, 3840, 3)
    for f in (0, 3):
        assert_exact(out[f], br.vng(batch[f, :, :, 0], 65)[0], "VNG 4K batch frame %d" % f)
    g = cpu(cvb.cvtColor(gpu(batch), C.COLOR_BayerBG2GRAY))
    assert g.shape == (4, 2160, 3840, 1)
    assert_exact(g[2, :, :, 0], br.gray(batch[2, :, :, 0], 86), "GRAY 4K batch frame 2")


@pytest.mark.parametrize("case_id", ["r8-vng-gb-10x33-rand", "ties-vng-rg-s0", "fb-vng-gr-7x20-rand", "g-gray-gr-u16-9x31-rand", "g-gray-bg-u8-2x9-rand"])
def test_host_path(cvb, case_id):
    """hal.cvtColor on numpy arrays (b200cv_host_cvt_color: staged through the device)"""
    case = bc.BY_ID[case_id]
    m = bc.mosaic_of(case)
    assert_exact(cvb.cvtColor(m, case.code), restated(case, m), case_id)


def test_one_launch_per_call(cvb):
    import torch
    rng = np.random.default_rng(1)
    one = gpu(rng.integers(0, 256, (64, 96), dtype=np.uint8))
    batch = gpu(rng.integers(0, 256, (3, 64, 96, 1), dtype=np.uint8))
    small = gpu(rng.integers(0, 256, (7, 30), dtype=np.uint8))
    for src in (one, batch, small):
        for code in (C.COLOR_BayerBG2BGR_VNG, C.COLOR_BayerGR2GRAY):
            torch.cuda.synchronize()
            n0 = cvb.launch_count()
            cvb.cvtColor(src, code)
            assert cvb.launch_count() - n0 == 1, "code %d shape %s" % (code, tuple(src.shape))


def test_refusals_leave_the_destination_untouched(cvb):
    """16-bit VNG (the reference asserts 8-bit), VNG to 4 channels (the reference writes 3-byte pixels into 4-channel rows) and in-place
    calls are argument errors; mosaics under 3 pixels on a side are not implemented for VNG"""
    m8 = gpu(np.arange(20 * 24, dtype=np.uint8).reshape(20, 24))
    m16 = gpu(np.zeros((20, 24), np.uint16))
    calls = [(m16, gpu(np.full((20, 24, 3), 9, np.uint16)), C.COLOR_BayerBG2BGR_VNG),
             (m8, gpu(np.full((20, 24, 4), 9, np.uint8)), C.COLOR_BayerRG2BGR_VNG)]
    for src, dst, code in calls:
        with pytest.raises(C.B200cvError) as e:
            cvb.cvtColor(src, code, dst=dst)
        assert not isinstance(e.value, C.NotImplementedOnDevice)
        assert (cpu(dst) == 9).all(), "code %d: the destination was written" % code
    big = gpu(np.full((20, 72), 9, np.uint8))          # in place: the destination starts where the source does
    for code, src, dst in ((C.COLOR_BayerGB2BGR_VNG, big[:, :24], big.view(20, 24, 3)), (C.COLOR_BayerGB2GRAY, big[:, :24], big[:, :24])):
        with pytest.raises(C.B200cvError) as e:
            cvb.cvtColor(src, code, dst=dst)
        assert not isinstance(e.value, C.NotImplementedOnDevice)
        assert (cpu(big) == 9).all(), "code %d in place: the buffer was written" % code
    with pytest.raises(C.NotImplementedOnDevice):
        cvb.cvtColor(gpu(np.zeros((2, 24), np.uint8)), C.COLOR_BayerBG2BGR_VNG)
