#!/usr/bin/env python3
"""Write tests/golden/canny_ref.npz: cv::Canny answers of the compiled reference (oracle/_ref/libcannyref.so, built by
tools/build_canny_ref.py) for the cases below.  Inputs are not stored: tests/canny_reference.test_image regenerates them from the seed.
Outputs are stored np.packbits-packed (edge = 1 bit).  Refused argument sets are stored as refusals.

    python tools/make_canny_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import canny_reference as cr  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "canny_ref.npz")
SIZES = [(1, 1), (1, 7), (7, 1), (2, 2), (3, 5), (16, 33), (48, 64), (131, 257)]    # (h, w)


def cases():
    out = []
    seed = 100
    # every aperture x L1/L2 x cn 1/3 over the sizes, with ordinary thresholds
    for ap in (3, 5, 7, -1):
        for l2 in (False, True):
            for cn in (1, 3):
                for (h, w) in SIZES:
                    t = (40.0, 120.0) if ap != 7 else (400.0, 1300.0)
                    out.append((seed, h, w, cn, t[0], t[1], ap, l2))
                    seed += 1
    # threshold corner cases at a mid size, aperture 3 and 7
    special = [(150.0, 50.0), (100.0, 100.0), (0.0, 0.0), (-5.0, 40.0), (20.5, 70.25), (-30.0, -10.0),
               (1e10, 1e10), (20.0, 1e10), (40000.0, 50000.0), (10.0, 40000.0), (32767.5, 32768.0)]
    for ap in (3, 7):
        for l2 in (False, True):
            for t1, t2 in special:
                out.append((seed, 48, 64, 1, t1, t2, ap, l2))
                seed += 1
    # the legacy CV_CANNY_L2_GRADIENT bit inside the aperture, and refused apertures
    out.append((seed, 48, 64, 3, 30.0, 90.0, 3 | (1 << 31), False)); seed += 1
    out.append((seed, 48, 64, 1, 30.0, 90.0, 5 | (1 << 31), False)); seed += 1
    for ap in (1, 2, 4, 9, 0):
        out.append((seed, 16, 16, 1, 30.0, 90.0, ap, False)); seed += 1
    return out


def main():
    ref = cr.RefCanny("ref")
    params, refused, packed, offsets = [], [], [], [0]
    for (seed, h, w, cn, t1, t2, ap, l2) in cases():
        img = cr.test_image(seed, h, w, cn)
        e = ref.Canny(img, t1, t2, ap, l2)
        params.append((seed, h, w, cn, t1, t2, float(int(cr.wrap32(ap))), float(l2)))
        refused.append(e is None)
        bits = np.packbits((e > 0).reshape(-1)) if e is not None else np.zeros(0, np.uint8)
        packed.append(bits)
        offsets.append(offsets[-1] + bits.size)
    np.savez_compressed(OUT, params=np.array(params, np.float64), refused=np.array(refused), packed=np.concatenate(packed),
                        offsets=np.array(offsets, np.int64))
    print("%s: %d cases (%d refused), %d bytes" % (OUT, len(params), sum(refused), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
