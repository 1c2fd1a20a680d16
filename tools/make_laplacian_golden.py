#!/usr/bin/env python3
"""Write tests/golden/laplacian_ref.json: for every case of tests/laplacian_cases.py, the SHA-256 of the compiled reference's
cv::Laplacian answer (oracle/_ref/liblapref.so, built by tools/build_laplacian_ref.py), or "refused" where it rejects the arguments.
Elements the reference computes in a scalar remainder loop the port does not restate (laplacian_cases.remainder_start)
are zeroed before hashing.  Digests only: inputs are regenerated from the case ids, outputs are not stored.  The file also records which of the reference's
CPU-dispatched objects produced the answers: convertTo's cvt_32f and the separable filters are dispatched per instruction set
(SSE2 / AVX2), and the AVX2 objects, compiled with FMA, are the ones whose operation order the port and the device restate.

    python tools/make_laplacian_golden.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import laplacian_cases as lc  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "laplacian_ref.json")


def cpu_variant():
    flags = set()
    with open("/proc/cpuinfo") as fh:
        for line in fh:
            if line.startswith("flags"):
                flags = set(line.split(":", 1)[1].split())
                break
    return "AVX2+FMA3 objects (cvt_32f: v_fma)" if {"avx2", "fma"} <= flags else "baseline SSE2 objects (no FMA)"


def main():
    out, img_id, img = {}, None, None
    for c in lc.CASES:
        if c.image.id != img_id:
            img_id, img = c.image.id, lc.image_of(c.image)
        out[c.id] = lc.digest(lc.masked(c.image, c.ksize, lc.run("ref", img, c.ddepth, c.ksize, c.scale, c.delta, c.border)))
    with open(OUT, "w") as fh:
        json.dump({"dispatch": cpu_variant(), "laplacian": out}, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("%s: %d cases, %d bytes" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
