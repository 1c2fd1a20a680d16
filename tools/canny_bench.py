#!/usr/bin/env python3
"""Time cv::Canny on the device (b200cv_canny) over 4K frames and check its output against the reference.

    python tools/canny_bench.py [--reps 15] [--warmup 3] [--frames 16] [--frames-c3 4]

Workload: 16 smooth-plus-noise 4K 8UC1 frames and 4 4K 8UC3 frames (one launch set per batch); aperture 3 with L1 and with L2, aperture 5
with L2.  Each configuration is timed with CUDA events around one call, after warm-up; the median and range of the repeats are printed
beside the card's name and power limit (read-only nvidia-smi query).  For context, the same frames through the two 16S b200cv_sobel calls
that Canny's gradient stage replaces, and the compiled reference's CPU cv::Canny where oracle/_ref holds it.  The device output of the
timed frames is compared with the reference (or, without it, with the numpy restatement on two frames).  One JSON line per configuration.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:           # the timing itself does not depend on it
        return "unknown (%s)" % e


def smooth_frames(torch, n, cn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    low = torch.rand((n * cn, 1, 270, 480), device="cuda", generator=g)
    img = torch.nn.functional.interpolate(low, size=(2160, 3840), mode="bicubic").clamp(0, 1) * 235
    img = img + torch.rand(img.shape, device="cuda", generator=g) * 20
    return img.clamp(0, 255).to(torch.uint8).reshape(n, cn, 2160, 3840).permute(0, 2, 3, 1).contiguous()


def time_call(torch, fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--frames-c3", type=int, default=4)
    ap.add_argument("--t1", type=float, default=40.0)
    ap.add_argument("--t2", type=float, default=120.0)
    a = ap.parse_args()

    import torch
    import opencv_b200 as cvb
    import canny_reference as cr
    if not torch.cuda.is_available():
        sys.exit("canny_bench: no CUDA device")
    cvb.init(0)
    gpu = card()
    ref = cr.RefCanny("ref") if cr.ref_available("ref") else None
    batches = {"8UC1": smooth_frames(torch, a.frames, 1, 1), "8UC3": smooth_frames(torch, a.frames_c3, 3, 2)}
    configs = [(3, False), (3, True), (5, True)]
    for name, src in batches.items():
        n = src.shape[0]
        edges = torch.empty((n, 2160, 3840, 1), dtype=torch.uint8, device="cuda")
        host = src.cpu().numpy()
        for ksize, l2 in configs:
            call = lambda: cvb.Canny(src, a.t1, a.t2, edges, ksize, l2)
            med, lo, hi = time_call(torch, call, a.reps, a.warmup)
            dx = torch.empty(src.shape, dtype=torch.int16, device="cuda")
            dy = torch.empty(src.shape, dtype=torch.int16, device="cuda")
            sob = lambda: (cvb.Sobel(src, cvb.CV_16S, 1, 0, ksize, 1.0, 0.0, cvb.BORDER_REPLICATE, dst=dx),
                           cvb.Sobel(src, cvb.CV_16S, 0, 1, ksize, 1.0, 0.0, cvb.BORDER_REPLICATE, dst=dy))
            smed, slo, shi = time_call(torch, sob, a.reps, a.warmup)
            del dx, dy
            call()
            torch.cuda.synchronize()
            got = edges.cpu().numpy()[..., 0]
            frame = lambda f: host[f, :, :, 0] if host.shape[3] == 1 else host[f]
            cpu_ms, checked, mismatched = None, 0, 0
            if ref is not None:
                t0 = time.perf_counter()
                outs = [ref.Canny(frame(f), a.t1, a.t2, ksize, l2) for f in range(n)]
                cpu_ms = (time.perf_counter() - t0) * 1e3
                for f in range(n):
                    checked += 1
                    mismatched += int(not np.array_equal(got[f], outs[f]))
                checker = "reference"
            else:
                for f in range(min(2, n)):
                    checked += 1
                    mismatched += int(not np.array_equal(got[f], cr.canny(frame(f), a.t1, a.t2, ksize, l2)))
                checker = "restatement"
            px = n * 2160 * 3840
            print(json.dumps({"op": "Canny", "frames": n, "type": name, "ksize": ksize, "L2": l2, "thresholds": [a.t1, a.t2],
                              "ms_median": round(med, 3), "ms_min": round(lo, 3), "ms_max": round(hi, 3), "reps": a.reps,
                              "gpix_per_s": round(px / med / 1e6, 2), "edge_fraction": round(float((got > 0).mean()), 4),
                              "sobel16s_x2_ms_median": round(smed, 3), "sobel16s_x2_ms_range": [round(slo, 3), round(shi, 3)],
                              "reference_cpu_ms": None if cpu_ms is None else round(cpu_ms, 1),
                              "checked_frames": checked, "mismatched_frames": mismatched, "checked_against": checker, "gpu": gpu}), flush=True)
            if mismatched:
                sys.exit("canny_bench: device output differs from the %s" % checker)


if __name__ == "__main__":
    main()
