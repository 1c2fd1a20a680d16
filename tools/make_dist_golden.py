#!/usr/bin/env python3
"""Write tests/golden/dist_ref.json: for every case of tests/dist_cases.py, the SHA-256 of the compiled reference's cv::distanceTransform
answer (oracle/_ref/libdistref.so, built by tools/build_dist_ref.py) prefixed with the depth it produced, or "refused" where it rejects
the arguments.  Digests only: inputs are regenerated from the case ids, outputs are not stored.

    python tools/make_dist_golden.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dist_cases as dc  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "dist_ref.json")


def main():
    images = {}
    out = {}
    for c in dc.CASES:
        if c.image not in images:
            images = {c.image: dc.image_of(c)}
        out[c.id] = dc.digest(*dc.run("ref", images[c.image], c.call))
    with open(OUT, "w") as fh:
        json.dump({"dist": out}, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("%s: %d cases, %d bytes" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
