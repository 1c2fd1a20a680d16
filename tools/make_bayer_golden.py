#!/usr/bin/env python3
"""Write tests/golden/bayer_ref.json: the SHA-256 of the compiled reference's cv::cvtColor answer (oracle/_ref/libocvref.so, built by
oracle/build_ref.py) for every case of tests/bayer_cases.py (Bayer VNG, codes 62-65, and Bayer to GRAY, 86-89).  Digests only: inputs
are regenerated from the case ids, outputs are not stored.

    python tools/make_bayer_golden.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bayer_cases as bc  # noqa: E402
from oracle.api import Oracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "bayer_ref.json")


def main():
    ref = Oracle("ref")
    bayer = {c.id: bc.digest(ref.cvtColor(bc.mosaic_of(c), c.code, 3 if c.kind == "vng" else 1)) for c in bc.CASES}
    with open(OUT, "w") as fh:
        json.dump({"bayer": bayer}, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("%s: %d cases, %d bytes" % (OUT, len(bayer), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
