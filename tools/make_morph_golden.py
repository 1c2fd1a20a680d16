#!/usr/bin/env python3
"""Write tests/golden/morph_ref.json: for every call of every case of tests/morph_cases.py, the SHA-256 of the compiled reference's
answer (oracle/_ref/libmorphref.so, built by tools/build_morph_ref.py) with the 32F elements that tests/morph_reference.py excludes
zeroed, or "refused" where the reference rejects the arguments; and the reference's getStructuringElement for every shape and size
from 1x1 to 15x15 plus a few larger ones.  Digests only: inputs are regenerated from the case ids.

    python tools/make_morph_golden.py
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import morph_cases as mc  # noqa: E402
import morph_reference as mr  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "morph_ref.json")


def main():
    out = {}
    for case in mc.CASES:
        img = mc.image_of(case)
        for name, call in case.calls.items():
            want = mc.reference(img, case.depth, call)
            try:
                excl = mc.restated(img, call)[1]
            except mr.Refused:
                excl = None
            out["%s/%s" % (case.id, name)] = mc.digest(want, excl)
    se = {}
    for shape, w, h, anchor in mc.STRUCTURING:
        e = mc.ref_structuring_element(shape, w, h, anchor)
        se["%d-%dx%d-%d,%d" % (shape, w, h, anchor[0], anchor[1])] = "refused" if e is None else hashlib.sha256(e.tobytes()).hexdigest()
    with open(OUT, "w") as fh:
        json.dump({"morph": out, "structuring": se}, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("%s: %d calls, %d elements, %d bytes" % (OUT, len(out), len(se), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
