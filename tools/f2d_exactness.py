"""how many pixels of 8-bit filter2D differ from the reference CPU result: direct FP32 kernel vs tensor-core fixed-point path"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
import opencv_b200 as cvb
from oracle.api import Oracle

cvb.init(0)
ref = Oracle("ref")
rng = np.random.default_rng(5)
img = rng.integers(0, 256, (1080, 1920), dtype=np.uint8)
g = torch.from_numpy(img).cuda()
for k in (3, 5, 7, 9, 11):
    ker = rng.random((k, k)).astype(np.float32); ker /= ker.sum()
    want = ref.filter2D(img, -1, ker)
    os.environ["B200CV_FILTER2D_PATH"] = "direct"
    a = cvb.filter2D(g, -1, ker).cpu().numpy()
    os.environ.pop("B200CV_FILTER2D_PATH")
    os.environ["B200CV_FILTER2D_TC_MIN_TAPS"] = "1"
    b = cvb.filter2D(g, -1, ker).cpu().numpy()
    os.environ.pop("B200CV_FILTER2D_TC_MIN_TAPS")
    print("k=%d  direct: %d differ (max %d)   tensor: %d differ (max %d)   of %d" % (
        k, (a != want).sum(), np.abs(a.astype(int) - want).max(), (b != want).sum(), np.abs(b.astype(int) - want).max(), want.size))

f = (rng.random((1080, 1920)) * 255).astype(np.float32)
gf = torch.from_numpy(f).cuda()
for k in (3, 5, 7, 9, 11):
    ker = rng.random((k, k)).astype(np.float32); ker /= ker.sum()
    want = ref.filter2D(f, -1, ker, delta=0.5)
    a = cvb.filter2D(gf, -1, ker, delta=0.5).cpu().numpy()
    w2 = ref.filter2D(img, 5, ker) if k * k < 50 else None
    a2 = cvb.filter2D(g, 5, ker).cpu().numpy() if w2 is not None else None
    body = (f.shape[1] // 8) * 8
    print("f32 k=%d: %d differ (max %.3g)%s" % (k, (a != want).sum(), np.abs(a - want).max(),
                                               "   u8->f32: %d differ" % (a2 != w2).sum() if w2 is not None else ""))
