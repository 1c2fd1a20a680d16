#!/usr/bin/env python3
"""Time cv::distanceTransform on the device (b200cv_distance_transform) over 4K edge-distance frames and check it against the CPU oracles.

    python tools/dist_bench.py [--reps 9] [--warmup 2] [--frames 16] [--runs 2]

Workload: inverted edge maps (0 on one-pixel contours of a smooth random field, 255 elsewhere), 2160 x 3840 8UC1: a batch of 16 frames
and a single frame, for the 3x3 L2 chamfer, the 5x5 L2 chamfer, the precise transform and the 8-bit L1 call.  Each configuration is
timed with CUDA events around one call, after warm-up, in `--runs` separate passes over all configurations; each pass prints its
median.  The card's name and power limit are read in the same run (read-only nvidia-smi query).  The HBM bound is the bytes the call
must move (source read once, destination written once) over 3.35 TB/s; the chamfer's other bound is its 2 * H dependent row steps.
For context, the compiled reference's CPU call on the same frames where oracle/_ref/libdistref.so exists (timed over the first
--ref-frames frames and scaled to the batch).  The device output of two frames is compared with the reference, or the plain-C port
without it.  One JSON line per configuration and run.
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

HBM_BYTES_PER_S = 3.35e12
MODES = {"l2_3x3": (2, 3, 5), "l2_5x5": (2, 5, 5), "precise": (2, 0, 5), "l1_8u": (1, 3, 0)}
CASE_CALL = {"l2_3x3": "l2_3", "l2_5x5": "l2_5", "precise": "precise", "l1_8u": "l1_u8"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:           # the timing itself does not depend on it
        return "unknown (%s)" % e


def edge_frames(torch, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    low = torch.rand((n, 1, 180, 320), device="cuda", generator=g)
    field = torch.nn.functional.interpolate(low, size=(2160, 3840), mode="bilinear")[:, 0]
    inside = field > 0.5
    edge = torch.zeros_like(inside)
    edge[:, :, :-1] |= inside[:, :, :-1] != inside[:, :, 1:]
    edge[:, :-1, :] |= inside[:, :-1, :] != inside[:, 1:, :]
    return torch.where(edge, 0, 255).to(torch.uint8).unsqueeze(-1).contiguous()


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
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--ref-frames", type=int, default=2)
    a = ap.parse_args()

    import torch
    import opencv_b200 as cvb
    import dist_cases as dc
    if not torch.cuda.is_available():
        sys.exit("dist_bench: no CUDA device")
    cvb.init(0)
    gpu = card()
    batches = {a.frames: edge_frames(torch, a.frames, 1), 1: edge_frames(torch, 1, 2)}
    checker = "reference" if dc.ref_available() else "port"
    if checker == "port":
        from oracle import build_port
        build_port.build()
    H, W = 2160, 3840
    ref_ms = {}
    for run in range(a.runs):
        for n, src in batches.items():
            host = src.cpu().numpy()[..., 0]
            for mode, (dt, mask, dst_type) in MODES.items():
                dst = torch.empty((n, H, W, 1), dtype=torch.uint8 if dst_type == 0 else torch.float32, device="cuda")
                call = lambda: cvb.distanceTransform(src, dt, mask, dst=dst, dstType=dst_type)
                med, lo, hi = time_call(torch, call, a.reps, a.warmup)
                torch.cuda.synchronize()
                got = dst.cpu().numpy()[..., 0]
                mismatched = 0
                for f in sorted({0, n - 1}):
                    want = dc.run("ref" if checker == "reference" else "port", host[f], CASE_CALL[mode])[1]
                    mismatched += int(not np.array_equal(got[f].view(np.uint8 if dst_type == 0 else np.int32),
                                                         want.view(np.uint8 if dst_type == 0 else np.int32)))
                key = (n, mode)
                if checker == "reference" and run == 0:
                    k = min(a.ref_frames, n)
                    t0 = time.perf_counter()
                    for f in range(k):
                        dc.run("ref", host[f], CASE_CALL[mode])
                    ref_ms[key] = (time.perf_counter() - t0) * 1e3 * n / k
                nbytes = n * H * W * (1 + (1 if dst_type == 0 else 4))
                bound_ms = nbytes / HBM_BYTES_PER_S * 1e3
                print(json.dumps({"op": "distanceTransform", "mode": mode, "frames": n, "run": run, "ms_median": round(med, 3),
                                  "ms_min": round(lo, 3), "ms_max": round(hi, 3), "reps": a.reps,
                                  "hbm_bytes": nbytes, "hbm_bound_ms": round(bound_ms, 4), "share_of_hbm_bound": round(bound_ms / med, 4),
                                  "dependent_row_steps": 2 * H if mode != "precise" else None,
                                  "reference_cpu_ms": None if key not in ref_ms else round(ref_ms[key], 1),
                                  "zero_fraction": round(float((host == 0).mean()), 4),
                                  "checked_frames": len({0, n - 1}), "mismatched_frames": mismatched, "checked_against": checker,
                                  "gpu": gpu}), flush=True)
                del dst
                if mismatched:
                    sys.exit("dist_bench: device output differs from the %s" % checker)


if __name__ == "__main__":
    main()
