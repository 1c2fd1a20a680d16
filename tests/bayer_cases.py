"""One table of cv::cvtColor cases for the Bayer VNG (codes 62-65) and Bayer-to-GRAY (86-89) codes, aimed at the places where the
reference's code changes arm or copies instead of computing (see tests/bayer_reference.py):

  fb     min(W, H) of 7 and 8 on either axis: the bilinear fallback and the first VNG size
  w      widths 8-13: no vector block, or a first one, for each start column (2 or 3 by row parity)
  r8     widths 26-41 at 10 rows: every residue of W - 10 modulo 8, both row parities in every image
  h      heights 8-10: the four copied bottom rows
  flat   constant and near-constant mosaics (maxGrad <= 1: T = minGrad + 1) and 0 / max checkerboards
  ties   mosaics whose ids were chosen so that ng == 7 meets a colour difference that is an odd multiple of 7 (where the two
         arms' factors round differently) in head, body and tail columns, for every pattern (test_bayer_reference.py checks it)
  g      GRAY: 1x1 to 3x3, 2-row and 2-column sizes, odd and even widths, 8- and 16-bit
  big    1080 x 1920 and 2160 x 3840

Every case is plain data; its pixels come from PCG64 seeded by the SHA-256 of its id, so every machine builds the same bytes.
"""
import hashlib
from collections import namedtuple

import numpy as np

Case = namedtuple("Case", "id kind code shape dtype fill")      # kind "vng" | "gray"; shape (H, W); dtype "u8" | "u16"

PAT = {"bg": 0, "gb": 1, "rg": 2, "gr": 3}
VNG = {p: 62 + i for p, i in PAT.items()}
GRAY = {p: 86 + i for p, i in PAT.items()}

# seeds of the `ties` group: the first seed per pattern whose mosaic puts such ties in the head, body and tail columns (any seed that
# meets the claim would do; tests/test_bayer_reference.py checks it)
TIE_SEEDS = {"bg": 0, "gb": 0, "rg": 0, "gr": 0}


def _cases():
    out = []

    def vng(group, shape, fill="rand", pats=PAT):
        for p in pats:
            out.append(Case("%s-vng-%s-%dx%d-%s" % (group, p, shape[0], shape[1], fill), "vng", VNG[p], shape, "u8", fill))

    def gray(group, shape, fill="rand", dtypes=("u8", "u16"), pats=PAT):
        for dt in dtypes:
            for p in pats:
                out.append(Case("%s-gray-%s-%s-%dx%d-%s" % (group, p, dt, shape[0], shape[1], fill), "gray", GRAY[p], shape, dt, fill))

    for shape in [(7, 7), (7, 20), (20, 7), (8, 8), (8, 20), (20, 8), (3, 3), (3, 12), (12, 3), (5, 6)]:
        vng("fb", shape)
    for w in range(8, 14):
        vng("w", (12, w))
    for w in range(26, 42):
        vng("r8", (10, w))
    for h in (8, 9, 10, 11):
        vng("h", (h, 24))
    for fill in ("const", "near", "checker"):
        vng("flat", (16, 37), fill)
    for p, seed in TIE_SEEDS.items():
        out.append(Case("ties-vng-%s-s%d" % (p, seed), "vng", VNG[p], (160, 25), "u8", "ties"))
    for shape in [(1, 1), (1, 2), (2, 1), (2, 2), (2, 3), (3, 2), (3, 3), (1, 9), (9, 1), (2, 9), (9, 2), (3, 4), (4, 3), (3, 17), (17, 3),
                  (5, 16), (9, 31), (16, 33)]:
        gray("g", shape)
    for fill in ("const", "checker"):
        gray("g", (9, 20), fill)
    vng("big", (1080, 1920), pats=("rg",))
    vng("big", (2160, 3840), pats=("gb",))
    gray("big", (1080, 1920), pats=("bg",))
    gray("big", (2160, 3840), pats=("gr",))
    return out


def rng_of(case_id):
    return np.random.Generator(np.random.PCG64(int.from_bytes(hashlib.sha256(case_id.encode()).digest()[:8], "little")))


def mosaic_of(case):
    """the case's source mosaic (H, W), uint8 or uint16"""
    H, W = case.shape
    dt = np.uint8 if case.dtype == "u8" else np.uint16
    top = 255 if case.dtype == "u8" else 65535
    g = rng_of(case.id)
    if case.fill == "rand":
        return g.integers(0, top + 1, (H, W), dtype=dt)
    if case.fill == "const":
        return np.full((H, W), int(g.integers(0, top + 1)), dt)
    if case.fill == "near":        # a constant with sparse +-1 pixels: gradients of 0, 1 and 2
        m = np.full((H, W), int(g.integers(1, top)), np.int64)
        m += (g.random((H, W)) < 0.1) * g.choice([-1, 1], (H, W))
        return m.astype(dt)
    if case.fill == "checker":
        y, x = np.mgrid[0:H, 0:W]
        return (((y + x) & 1) * top).astype(dt)
    if case.fill == "ties":        # triangle-wave ramps plus noise (integer arithmetic only): one excluded direction (ng == 7) is common
        y, x = np.mgrid[0:H, 0:W]
        px, py, ph = (int(v) for v in g.integers(4, 13, 3))
        tri = lambda t, p: np.abs(t % (2 * p) - p)
        base = 68 + tri(x + ph, px) * 120 // px + tri(y, py) * 60 // py
        return np.clip(base + g.integers(-20, 21, (H, W)), 0, 255).astype(dt)
    raise ValueError(case.fill)


CASES = _cases()
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
