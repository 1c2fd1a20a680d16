#!/usr/bin/env python3
"""Write tests/golden/resize_ref.json: the SHA-256 of the compiled reference's answer (oracle/_ref/libocvref.so, built by
oracle/build_ref.py) for every case of tests/resize_cases.py.  Digests only: inputs are regenerated from the case ids, outputs are not
stored; NaN is hashed in one canonical form (resize_cases.canonical).

    python tools/make_resize_golden.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import resize_cases as rc  # noqa: E402
from oracle.api import Oracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "resize_ref.json")


def main():
    ref = Oracle("ref")
    resize = {c.id: rc.digest([rc.run(ref, c, f) for f in rc.frames_of(c)]) for c in rc.CASES}
    with open(OUT, "w") as fh:
        json.dump({"resize": resize}, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("%s: %d resize cases, %d bytes" % (OUT, len(resize), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
