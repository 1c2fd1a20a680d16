#!/usr/bin/env python3
"""Time erode / dilate / morphologyEx on the device (opencv_b200) over 16 frames of 2160 x 3840 8UC1 and 8 frames of 32FC1.

Configurations: 3x3 rect erode, 5x5 ellipse dilate, 15x15 rect erode, 31x31 ellipse erode, 3x3 rect with 10 iterations (grown to a
21x21 rectangle, one pass), OPEN with a 5x5 ellipse, GRADIENT with a 3x3 rect, 32x32 and 33x33 rect erodes (the last size of the
fused kernel and the first of the van Herk path), and 3x3 rect with 40 iterations (81x81, van Herk).  Each device time is the median of CUDA-event timings of one batched call, over --runs runs of --reps repetitions; the median of
the runs is printed with each run's value.  The HBM bound is the bytes the call must move at least (the source read once and the
destination written once; GRADIENT / TOPHAT / BLACKHAT and OPEN / CLOSE also write and read one intermediate plane) over 3.35 TB/s, the
H100 SXM data-sheet bandwidth.  The reference's CPU time (oracle/_ref/libmorphref.so, where it was built) is a host clock around the
same frames, one reference call per frame (its own parallel_for_ threads within each frame).  The card's name and power limit are read
in the same run (a read-only nvidia-smi query).  One frame of
each configuration is checked against tests/morph_reference.py.

    python tools/morph_bench.py [--reps 9] [--runs 2]
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
# name, op, shape, size, iterations, planes moved (source + destination + intermediate writes and reads)
CONFIGS = [("3x3 rect erode", 0, 0, 3, 1, 2), ("5x5 ellipse dilate", 1, 2, 5, 1, 2), ("15x15 rect erode", 0, 0, 15, 1, 2),
           ("31x31 ellipse erode", 0, 2, 31, 1, 2), ("3x3 rect x10 erode", 0, 0, 3, 10, 2), ("OPEN 5x5 ellipse", 2, 2, 5, 1, 4),
           ("GRADIENT 3x3 rect", 4, 0, 3, 1, 4), ("32x32 rect erode", 0, 0, 32, 1, 2), ("33x33 rect erode", 0, 0, 33, 1, 2),
           ("3x3 rect x40 erode", 0, 0, 3, 40, 2)]


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
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("morph_bench: no CUDA device")
    import opencv_b200 as cvb
    import morph_cases as mc
    import morph_reference as mr
    cvb.init(0)
    H, W = 2160, 3840
    g = torch.Generator(device="cuda").manual_seed(5)
    # binary-looking frames (a thresholded smooth field with noise), as morphology usually sees
    field = torch.nn.functional.interpolate(torch.rand((16, 1, H // 16, W // 16), device="cuda", generator=g), size=(H, W), mode="bilinear")
    noise = torch.randint(0, 64, (16, 1, H, W), device="cuda", generator=g)
    u8 = torch.where(field > 0.5, torch.full_like(noise, 255), noise).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    f32 = u8[:8].to(torch.float32) * 0.37
    print("card: %s" % card())
    have_ref = mc.ref_available()
    for name, op, shape, k, it, planes in CONFIGS:
        kernel = cvb.getStructuringElement(shape, (k, k))
        for src in (u8, f32):
            dst = torch.empty_like(src)

            def run():
                cvb.morphologyEx(src, op, kernel, dst=dst, iterations=it)

            ts = [time_call(torch, run, a.reps, a.warmup) for _ in range(a.runs)]
            torch.cuda.synchronize()
            f0 = src[0].cpu().numpy()
            want = mr.morphology(f0, "mex", op, kernel, (-1, -1), it)
            ok = bool(np.array_equal(dst[0].cpu().numpy(), want))
            ref_ms = None
            if have_ref:
                call = mc.Call("mex", op, ("rect" if shape == 0 else "ellipse", k, k), (-1, -1), it, 0, None)
                frames = [np.ascontiguousarray(f[:, :, 0]) for f in src.cpu().numpy()]
                depth = "8U" if src.dtype == torch.uint8 else "32F"
                t0 = time.perf_counter()
                for f in frames:
                    mc.reference(f, depth, call)
                ref_ms = (time.perf_counter() - t0) * 1e3
            nbytes = src.numel() * src.element_size() * planes
            row = {"config": name, "type": "8UC1" if src.dtype == torch.uint8 else "32FC1", "frames": src.shape[0],
                   "device_ms": round(float(np.median(ts)), 3), "runs_ms": [round(t, 3) for t in ts],
                   "hbm_bound_ms": round(nbytes / HBM_BYTES_PER_S * 1e3, 3),
                   "reference_cpu_ms": None if ref_ms is None else round(ref_ms, 1), "frame0_matches_restatement": ok}
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
