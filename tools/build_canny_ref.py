#!/usr/bin/env python3
"""Build the reference's cv::Canny wrappers (tests/cpp/canny_ref_shim.cpp) into oracle/_ref/ next to the reference libraries:

    oracle/_ref/libcannyref.so       linked against libocvref.so      (the reference's own Canny)
    oracle/_ref/libcannyref_hal.so   linked against libocvref_hal.so  (the reference with hal/b200cv_hal_replacement.hpp: Canny -> b200cv_hal_canny)

Needs the reference's headers and an oracle/_ref built by oracle/build_ref.py --hal; without them it does nothing.  Test infrastructure
only: the library never links these.  Usage: python tools/build_canny_ref.py [--reference DIR]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_ref")
SRC = os.path.join(ROOT, "tests", "cpp", "canny_ref_shim.cpp")


def build(ref="/root/reference"):
    gen = os.path.join(OUT, "gen")
    if not os.path.isdir(os.path.join(ref, "modules", "imgproc", "include")) or not os.path.isdir(gen):
        return []
    inc = ["-I" + gen] + ["-I" + os.path.join(ref, "modules", m, "include") for m in ("core", "imgproc")]
    built = []
    for name, dep in (("libcannyref.so", "ocvref"), ("libcannyref_hal.so", "ocvref_hal")):
        out = os.path.join(OUT, name)
        if not os.path.exists(os.path.join(OUT, "lib%s.so" % dep)):
            continue
        deps = [SRC, os.path.join(OUT, "lib%s.so" % dep)]
        if os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps):
            built.append(out)
            continue
        cmd = ["g++", "-std=c++11", "-O1", "-shared", "-fPIC", "-w", "-o", out, SRC] + inc + ["-L" + OUT, "-l" + dep, "-Wl,-rpath,$ORIGIN"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("canny_ref_shim: compilation against the reference failed")
        built.append(out)
    return built


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    print("\n".join(build(ap.parse_args().reference)))
