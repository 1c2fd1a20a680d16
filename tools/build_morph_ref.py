#!/usr/bin/env python3
"""Build the reference's cv::erode / dilate / morphologyEx / getStructuringElement wrappers (tests/cpp/morph_ref_shim.cpp) into
oracle/_ref/libmorphref.so, linked against oracle/_ref/libocvref.so.  Needs the reference's headers and an oracle/_ref built by oracle/build_ref.py; without them it does nothing.
Test infrastructure only: the library never links it.  Usage: python tools/build_morph_ref.py [--reference DIR]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_ref")
SRC = os.path.join(ROOT, "tests", "cpp", "morph_ref_shim.cpp")


def build(ref="/root/reference"):
    gen = os.path.join(OUT, "gen")
    base = os.path.join(OUT, "libocvref.so")
    if not os.path.isdir(os.path.join(ref, "modules", "imgproc", "include")) or not os.path.isdir(gen) or not os.path.exists(base):
        return None
    out = os.path.join(OUT, "libmorphref.so")
    if os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in (SRC, base)):
        return out
    inc = ["-I" + gen] + ["-I" + os.path.join(ref, "modules", m, "include") for m in ("core", "imgproc")]
    cmd = ["g++", "-std=c++11", "-O1", "-shared", "-fPIC", "-w", "-o", out, SRC] + inc + ["-L" + OUT, "-locvref", "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("morph_ref_shim: compilation against the reference failed")
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    print(build(ap.parse_args().reference))
