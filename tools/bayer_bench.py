#!/usr/bin/env python3
"""Time the Bayer demosaicing kernels on the device over 16 4K mosaics and check one output frame against the numpy restatement.

    python tools/bayer_bench.py [--reps 20] [--warmup 3] [--frames 16]

Workload: 16 random 2160 x 3840 8UC1 mosaics (and 16UC1 for GRAY), one call per batch.  Timed: VNG (COLOR_BayerRG2BGR_VNG), GRAY at
8 and 16 bits, and for context the bilinear (COLOR_BayerRG2BGR) and edge-aware (COLOR_BayerRG2BGR_EA) kernels.  Each is timed with CUDA
events around one call, `--reps` times, in two runs; the median and the range over both runs are printed beside the card's name and power
limit (read-only nvidia-smi query in the same process) and the HBM bound computed from the shapes (bytes read + written over 3.35 TB/s:
VNG and the bilinear kernels 4 B/px, GRAY 2 B/px at 8 bits and 4 B/px at 16 bits).  Where oracle/_ref holds the compiled reference, its
CPU time for the same call on one frame, times the frame count, is printed too.  One JSON line per kernel.
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

HBM = 3.35e12


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
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    a = ap.parse_args()
    import torch
    import opencv_b200 as C
    import bayer_reference as br
    from oracle.api import Oracle, available
    if not torch.cuda.is_available():
        sys.exit("bayer_bench: no CUDA device")
    C.init(0)
    H, W, N = 2160, 3840, a.frames
    g = torch.Generator(device="cuda").manual_seed(11)
    m8 = torch.randint(0, 256, (N, H, W, 1), device="cuda", generator=g, dtype=torch.uint8)
    m16 = (torch.randint(0, 65536, (N, H, W, 1), device="cuda", generator=g, dtype=torch.int32)).to(torch.int16).view(torch.uint16)
    out3 = torch.empty((N, H, W, 3), dtype=torch.uint8, device="cuda")
    out1 = torch.empty((N, H, W, 1), dtype=torch.uint8, device="cuda")
    out1w = torch.empty((N, H, W, 1), dtype=torch.uint16, device="cuda")
    configs = [("vng", m8, out3, C.COLOR_BayerRG2BGR_VNG, 4),
               ("gray_u8", m8, out1, C.COLOR_BayerRG2GRAY, 2),
               ("gray_u16", m16, out1w, C.COLOR_BayerRG2GRAY, 4),
               ("bilinear", m8, out3, C.COLOR_BayerRG2BGR, 4),
               ("edge_aware", m8, out3, C.COLOR_BayerRG2BGR_EA, 4)]
    name = card()
    runs = {k: [] for k, *_ in configs}
    for _ in range(2):
        for k, src, dst, code, _bpp in configs:
            runs[k] += time_call(torch, lambda: C.cvtColor(src, code, dst=dst), a.reps, a.warmup)
    ref = Oracle("ref") if available("ref") else None
    for k, src, dst, code, bpp in configs:
        C.cvtColor(src, code, dst=dst)
        f = N - 1
        host = src[f, :, :, 0].cpu().numpy()
        got = dst[f].cpu().numpy()
        if k == "vng":
            ok = np.array_equal(got, br.vng(host, code)[0])
        elif k.startswith("gray"):
            ok = np.array_equal(got[:, :, 0], br.gray(host, code))
        else:
            ok = None if ref is None else np.array_equal(got, ref.cvtColor(host, code, 3))
        ts = runs[k]
        bound = N * H * W * bpp / HBM * 1e3
        row = {"kernel": k, "code": code, "frames": N, "shape": [H, W], "median_ms": round(float(np.median(ts)), 4),
               "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4), "hbm_bound_ms": round(bound, 4),
               "share_of_hbm_bound": round(bound / float(np.median(ts)), 3), "exact_frame": ok, "card": name}
        if ref is not None:
            t0 = time.perf_counter()
            ref.cvtColor(host, code, 3 if dst.shape[-1] == 3 else 1)
            row["reference_cpu_ms_for_all_frames"] = round((time.perf_counter() - t0) * 1e3 * N, 1)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
