"""float filter2D with >= 130 taps: tensor-core path (filter2d_tc_f32.cu) against the direct FP32 sum (filter2d_tma.cu), per kernel shape.
The tensor-core cost grows with the kernel rows, the direct sum's with the taps: this finds the row count from which the tensor cores win.
CUDA events around 20 launches on 8 3840x2160 CV_32FC1 frames, the two paths alternated.  Prints one line per (rows, cols) shape."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import opencv_b200 as cvb  # noqa: E402

cvb.init(0)
src = torch.rand((8, 2160, 3840, 1), device="cuda")
dst = torch.empty_like(src)
rng = np.random.default_rng(1)


def timed(ker, n=20):
    cvb.filter2D(src, -1, ker, dst=dst)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        cvb.filter2D(src, -1, ker, dst=dst)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


print(torch.cuda.get_device_name(0))
for kh, kw in ((5, 27), (7, 19), (9, 15), (11, 13), (12, 12), (13, 11), (15, 9), (17, 9)):
    ker = rng.random((kh, kw)).astype(np.float32)
    ker /= ker.sum()
    t = {"tc": [], "direct": []}
    for _ in range(3):
        os.environ.pop("B200CV_FILTER2D_PATH", None)
        os.environ["B200CV_FILTER2D_TC_MIN_TAPS"] = "130"      # tensor cores for every row count
        t["tc"].append(timed(ker))
        os.environ.pop("B200CV_FILTER2D_TC_MIN_TAPS")
        os.environ["B200CV_FILTER2D_PATH"] = "direct"
        t["direct"].append(timed(ker))
    os.environ.pop("B200CV_FILTER2D_PATH", None)
    print("%2d x %2d  tc %.3f ms  direct %.3f ms  (median of 3, per 8 frames)" % (kh, kw, np.median(t["tc"]), np.median(t["direct"])), flush=True)
