#!/usr/bin/env python3
"""Time cv::Laplacian on the device (opencv_b200.Laplacian) against what a user does without it: two device Sobel calls (dx = 2 and
dy = 2) into the same working depth plus a torch add, then a conversion where the destination depth asks for one.

Workloads: 16 frames of 2160 x 3840, 8UC1 -> 16S and -> 32F at ksize 1, 3, 5 and 7, and 32FC1 -> 32F at ksize 5 (Sobel covers ksize
up to 7, so the baseline exists for every row).  Each timing is the median of CUDA-event timings of one batched call, over --runs runs
of --reps repetitions; the card's name and power limit are read in the same run (read-only nvidia-smi query).  The HBM bound is the
bytes the call must move (source read once, destination written once) over 3.35 TB/s, the H100 SXM data-sheet bandwidth.

    python tools/laplacian_bench.py [--frames 16] [--reps 9] [--runs 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
CV_8U, CV_16S, CV_32F = 0, 3, 5
WORKLOADS = [(CV_8U, CV_16S, k) for k in (1, 3, 5, 7)] + [(CV_8U, CV_32F, k) for k in (1, 3, 5, 7)] + [(CV_32F, CV_32F, 5)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:           # the timing itself does not depend on it
        return "unknown (%s)" % e


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
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("laplacian_bench: no CUDA device")
    import opencv_b200 as cvb
    cvb.init(0)
    H, W, N = 2160, 3840, a.frames
    g = torch.Generator(device="cuda").manual_seed(5)
    u8 = torch.randint(0, 256, (N, H, W, 1), dtype=torch.uint8, device="cuda", generator=g)     # a batch of 1-channel frames
    f32 = u8.to(torch.float32) * 0.37
    esz = {CV_8U: 1, CV_16S: 2, CV_32F: 4}
    tdt = {CV_16S: torch.int16, CV_32F: torch.float32}
    print("card: %s" % card())
    for sd, dd, k in WORKLOADS:
        src = u8 if sd == CV_8U else f32
        dst = torch.empty((N, H, W, 1), dtype=tdt[dd], device="cuda")
        # the baseline's working depth is the Laplacian's: 16S for 8-bit sources up to ksize 5, 32F otherwise
        wd = CV_16S if sd == CV_8U and k <= 5 else CV_32F
        gx = torch.empty((N, H, W, 1), dtype=tdt[wd], device="cuda")
        gy = torch.empty_like(gx)

        def fused():
            cvb.Laplacian(src, dd, k, dst=dst)

        def two_sobels():
            cvb.Sobel(src, wd, 2, 0, k, dst=gx)
            cvb.Sobel(src, wd, 0, 2, k, dst=gy)
            if wd == dd:
                torch.add(gx, gy, out=dst)
            else:
                dst.copy_(gx + gy)

        t_fused, t_base = [], []
        for _ in range(a.runs):          # alternate the two so that clock drift hits both
            t_fused.append(time_call(torch, fused, a.reps, a.warmup))
            t_base.append(time_call(torch, two_sobels, a.reps, a.warmup))
        tf, tb = float(np.median(t_fused)), float(np.median(t_base))
        nbytes = N * H * W * (esz[sd] + esz[dd])
        bound_ms = nbytes / HBM_BYTES_PER_S * 1e3
        row = {"workload": "%s->%s k=%d" % ({0: "8UC1", 5: "32FC1"}[sd], {3: "16S", 5: "32F"}[dd], k), "frames": N,
               "laplacian_ms": round(tf, 3), "two_sobel_add_ms": round(tb, 3), "speedup": round(tb / tf, 2),
               "hbm_bound_ms": round(bound_ms, 3), "share_of_hbm_bound": round(bound_ms / tf, 3)}
        print(json.dumps(row))
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
