#!/usr/bin/env python3
"""Compare two `bench.py --dump-outputs` directories op by op (same arguments, two builds).

    python tools/compare_dumps.py OLD_DIR NEW_DIR [--float-tol 1e-4] [--json OUT]

Every op must be bit-identical, except that the ops named by --allow-diff (default: the float filter2D ops that run on the tensor cores,
whose per-element MMA order a kernel change may alter) may differ by at most --float-tol of that op's output range (max |old|).
Prints one line per op that is not identical and a summary; exits 1 if an op is missing or out of tolerance.
"""
import argparse
import glob
import json
import os
import re
import sys

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--allow-diff", default=r"^filter2D_f32_k(15|21|31)$", help="regex of op names that may differ within --float-tol")
    ap.add_argument("--float-tol", type=float, default=1e-4)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    allow = re.compile(a.allow_diff)
    names = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(a.old, "*.npy")))
    if not names:
        sys.exit("no .npy files in %s" % a.old)
    rows, bad = [], 0
    for name in names:
        pn = os.path.join(a.new, name + ".npy")
        if not os.path.exists(pn):
            rows.append(dict(op=name, status="missing"))
            bad += 1
            continue
        o, n = np.load(os.path.join(a.old, name + ".npy")), np.load(pn)
        if o.shape != n.shape:
            rows.append(dict(op=name, status="shape %s vs %s" % (o.shape, n.shape)))
            bad += 1
            continue
        same = np.array_equal(o, n, equal_nan=True)
        d = np.abs(o.astype(np.float64) - n.astype(np.float64))
        rng = float(np.abs(o.astype(np.float64)).max()) or 1.0
        r = dict(op=name, status="identical" if same else "differs", n=int(o.size), ndiff=int((o != n).sum()), max_abs=float(d.max()), max_rel_range=float(d.max()) / rng)
        if not same and not (allow.search(name) and r["max_rel_range"] <= a.float_tol):
            r["status"] = "FAIL"
            bad += 1
        rows.append(r)
    for r in rows:
        if r["status"] != "identical":
            print(json.dumps(r))
    print("%d ops: %d identical, %d differ within tolerance, %d failed" % (
        len(rows), sum(r["status"] == "identical" for r in rows), sum(r["status"] == "differs" for r in rows), bad))
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(rows, fh, indent=1)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
