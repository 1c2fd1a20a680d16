#!/usr/bin/env python3
"""Build the reference's cv::Laplacian wrapper (tests/cpp/laplacian_ref_shim.cpp) into oracle/_ref/liblapref.so, linked against
oracle/_ref/libocvref.so.  Needs the reference's headers and an oracle/_ref built by oracle/build_ref.py; without them it does nothing.
Test infrastructure only: the library never links it.  Usage: python tools/build_laplacian_ref.py [--reference DIR]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_ref")
SRC = os.path.join(ROOT, "tests", "cpp", "laplacian_ref_shim.cpp")


def _link(src, base_name, out, inc):
    base = os.path.join(OUT, base_name)
    if os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in (src, base)):
        return out
    cmd = ["g++", "-std=c++11", "-O1", "-shared", "-fPIC", "-w", "-o", out, src] + inc + ["-L" + OUT, "-l" + base_name[3:-3], "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("laplacian_ref_shim: compilation against the reference failed")
    return out


def build(ref="/root/reference"):
    """liblapref.so against the reference; liblapref_hal.so too where oracle/build_ref.py --hal built libocvref_hal.so (the reference
    with this project's HAL registered, tests/test_gpu_laplacian.py::test_hal_built_reference_sends_ksize_3_here)"""
    gen = os.path.join(OUT, "gen")
    if not os.path.isdir(os.path.join(ref, "modules", "imgproc", "include")) or not os.path.isdir(gen) or \
            not os.path.exists(os.path.join(OUT, "libocvref.so")):
        return None
    inc = ["-I" + gen] + ["-I" + os.path.join(ref, "modules", m, "include") for m in ("core", "imgproc")]
    out = _link(SRC, "libocvref.so", os.path.join(OUT, "liblapref.so"), inc)
    if os.path.exists(os.path.join(OUT, "libocvref_hal.so")):
        _link(SRC, "libocvref_hal.so", os.path.join(OUT, "liblapref_hal.so"), inc)
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    print(build(ap.parse_args().reference))
