"""GPU: cv::matchTemplate with a mask (all six methods; 8-bit binarised and float weight masks), against the reference at its own bar for
matchTemplate (1e-3 of the result range; the reference's numerators come from a float DFT, the device sums are direct and in double).

A failure here fails the suite."""
import numpy as np
import pytest

import opencv_b200 as C
from util import assert_close, cpu, gpu

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("method", range(6))
def test_masked_match_template(cvb, oracle, rng, method):
    img = rng.integers(0, 256, (200, 320), dtype=np.uint8)
    templ = img[60:92, 100:148].copy()
    m8 = (rng.random(templ.shape) > 0.3).astype(np.uint8) * 255
    mf = rng.random(templ.shape).astype(np.float32)
    for im, tt in ((img, templ), (img.astype(np.float32), templ.astype(np.float32))):
        for mk in (m8, mf):
            want = oracle.matchTemplateMasked(im, tt, method, mk)
            got = cpu(cvb.matchTemplate(gpu(im), gpu(tt), method, mask=gpu(mk)))
            assert_close(got, want, atol=1e-3 * max(1.0, float(np.abs(want).max())), what="masked matchTemplate %s mask %s method %d" % (im.dtype, mk.dtype, method))
    if method in (1, 3, 5):
        got = cpu(cvb.matchTemplate(gpu(img), gpu(templ), method, mask=gpu(m8)))
        assert np.unravel_index(got.argmin() if method == 1 else got.argmax(), got.shape) == (60, 100)


def test_masked_match_template_batch_1080p(cvb, ref, rng):
    base = rng.integers(0, 256, (1080, 1920), dtype=np.uint8)
    batch = np.stack([base, np.roll(base, 31, axis=1)])[..., None]
    templ = base[500:564, 800:864].copy(); mask = np.zeros(templ.shape, np.uint8); mask[8:56, 8:56] = 255
    out = cpu(cvb.matchTemplate(gpu(batch), gpu(templ), C.TM_CCOEFF_NORMED, mask=gpu(mask)))
    assert out.shape == (2, 1017, 1857, 1)
    want = ref.matchTemplateMasked(batch[1, :, :, 0], templ, C.TM_CCOEFF_NORMED, mask)
    assert_close(out[1, :, :, 0], want, atol=1e-3, what="masked CCOEFF_NORMED 1080p frame 1")
    assert np.unravel_index(out[1, :, :, 0].argmax(), want.shape) == (500, 831)
