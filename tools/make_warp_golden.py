#!/usr/bin/env python3
"""Write tests/golden/warp_ref.json: the SHA-256 of the compiled reference's answer (oracle/_ref/libocvref.so, built by
oracle/build_ref.py) for every case of tests/warp_cases.py and for the fixed-point remap cases.
Digests only: inputs are regenerated from the case ids, outputs are not stored.

    python tools/make_warp_golden.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import warp_cases as wc  # noqa: E402
from oracle.api import Oracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "warp_ref.json")


def main():
    ref = Oracle("ref")
    warp = {c.id: wc.digest([wc.run(ref, c, f) for f in wc.frames_of(c)]) for c in wc.CASES}
    remap = {}
    for dtype, cn in wc.TYPES6:
        case = wc.remap_case(dtype, cn)
        src = wc.frames_of(case)[0]
        remap[case.id] = wc.digest([ref.remap(src, wc.fixed_maps(), None, wc.NEAREST, b, wc.BV4) for b in wc.BORDERS])
    with open(OUT, "w") as fh:
        json.dump({"warp": warp, "remap": remap}, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("%s: %d warp cases, %d remap cases, %d bytes" % (OUT, len(warp), len(remap), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
