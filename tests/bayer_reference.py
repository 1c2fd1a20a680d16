"""numpy restatement of the reference's Bayer VNG and Bayer-to-GRAY demosaicing (modules/imgproc/src/demosaicing.cpp):

* vng(mosaic, code) -- Bayer2RGB_VNG_8u (:1059-1587), codes 62-65, 8-bit, 3-channel destination.  It also returns, per output pixel,
  the number of directions taken (`ng`) and the arm that computed it (SCALAR or SIMD), both read at the evaluated site.
* gray(mosaic, code) -- Bayer2Gray_ (:652-792), codes 86-89, 8- and 16-bit.

VNG computes every pixel of rows 2 .. H-5 and columns 2 .. W-3 and copies the rest (columns 0-1 and W-2, W-1 from their row's
nearest computed column, then rows 0-1 and H-4 .. H-1 from rows 2 and H-5), so the pixel at (y, x) is the value computed for
(clamp(y, 2, H-5), clamp(x, 2, W-3)).  The reference advances its mosaic pointer by two rows before the loop (:1083) and indexes it
with the destination row, so destination row y is computed from the mosaic around row y + 2 (rows 4 .. H-3; 5 x 5 reads reach
rows 2 .. H-1), with the pattern of row y (same parity).  Each value comes from seven gradient planes of the 3 x 3 neighbourhood,
a threshold T = minGrad + max(maxGrad / 2, 1) over eight directional gradients, and the mean colour differences over the
directions below T, scaled by 1 / (2 ng) and rounded half to even.  The reference has two arms for that last step:
  the scalar loop (head and tail columns) multiplies by  scale[ng] = {0, 0.5f, 0.25f, 0.1666666666667f, 0.125f, 0.1f,
                                                                      0.08333333333f, 0.0714286f, 0.0625f}[ng],
  the 8-pixel vector body multiplies by 0.5f / (float)ng;
the two factors differ as float32 only at ng == 7.  The body starts at column 2 in a row whose column 2 is a red / blue site and
at column 3 where it is green, and runs while its first column is <= W - 10.  Images with min(W, H) < 8 take the bilinear
Bayer2RGB_ with the VNG code, which that function reads as COLOR_BayerRG2BGR whatever the pattern.

GRAY: the pixel at (y, x) is the interior value at (clamp(y, 1, H-2), clamp(x, 1, W-2)); an image with W <= 2 or H <= 2 is all zero.
"""
import numpy as np

SCALAR, SIMD = 0, 1
SCALE_SCALAR = np.array([0, 0.5, 0.25, 0.1666666666667, 0.125, 0.1, 0.08333333333, 0.0714286, 0.0625], np.float32)
SCALE_SIMD = np.array([0] + [np.float32(0.5) / np.float32(n) for n in range(1, 9)], np.float32)

VNG_CODES = (62, 63, 64, 65)            # COLOR_BayerBG2BGR_VNG, GB, RG, GR
GRAY_CODES = (86, 87, 88, 89)           # COLOR_BayerBG2GRAY, GB, RG, GR
R2Y, G2Y, B2Y = 4899, 9617, 1868


def vng_pattern(code):
    """(blueIdx, greenCell0) of the first computed row (demosaicing.cpp:1067-1068)"""
    return (0 if code in (62, 63) else 2), code not in (62, 64)


def simd_columns(W, green_at_2):
    """the columns [start, end) the reference's 8-pixel vector body computes in a row whose column 2 is (or is not) a green site"""
    s = 3 if green_at_2 else 2
    if W - 10 < s:
        return s, s
    return s, s + ((W - 10 - s) // 8 + 1) * 8


def bilinear(m, blue0, swg0):
    """Bayer2RGB_ (demosaicing.cpp:806-1056) on an 8-bit mosaic with W, H >= 3: the interior value at the nearest interior site"""
    H, W = m.shape
    s = m.astype(np.int32)
    yi = np.clip(np.arange(H), 1, H - 2)[:, None]
    xi = np.clip(np.arange(W), 1, W - 2)[None, :]
    i, k = yi - 1, xi - 1
    blue = np.where(i & 1, -blue0, blue0)
    swg = ((i & 1) != 0) != (swg0 != 0)
    green = ((k & 1) == 0) == swg
    at = lambda dy, dx: s[yi + dy, xi + dx]
    c_lo = np.where(green, (at(-1, 0) + at(1, 0) + 1) >> 1, (at(-1, -1) + at(-1, 1) + at(1, -1) + at(1, 1) + 2) >> 2)
    c_hi = np.where(green, (at(0, -1) + at(0, 1) + 1) >> 1, at(0, 0))
    g = np.where(green, at(0, 0), (at(-1, 0) + at(0, -1) + at(0, 1) + at(1, 0) + 2) >> 2)
    out = np.stack([np.where(blue > 0, c_lo, c_hi), g, np.where(blue > 0, c_hi, c_lo)], axis=-1)
    return out.astype(np.uint8)


def vng_planes(m):
    """the seven gradient planes (demosaicing.cpp:1138-1153) at every interior site; entries outside rows / columns 1 .. n-2 are 0"""
    s = m.astype(np.int32)
    H, W = s.shape
    P = np.zeros((7, H, W), np.int16)         # every plane value is <= 1020
    if H < 3 or W < 3:
        return P
    c = lambda dy, dx: s[1 + dy:H - 1 + dy, 1 + dx:W - 1 + dx]
    a = np.abs
    P[0, 1:-1, 1:-1] = a(c(-1, -1) - c(1, -1)) + a(c(-1, 0) - c(1, 0)) * 2 + a(c(-1, 1) - c(1, 1))
    P[1, 1:-1, 1:-1] = a(c(-1, -1) - c(-1, 1)) + a(c(0, -1) - c(0, 1)) * 2 + a(c(1, -1) - c(1, 1))
    P[2, 1:-1, 1:-1] = a(c(-1, 1) - c(1, -1)) * 2
    P[3, 1:-1, 1:-1] = a(c(-1, -1) - c(1, 1)) * 2
    P[4, 1:-1, 1:-1] = P[2, 1:-1, 1:-1] + a(c(-1, 0) - c(0, -1)) + a(c(1, 0) - c(0, 1))
    P[5, 1:-1, 1:-1] = P[3, 1:-1, 1:-1] + a(c(-1, 0) - c(0, 1)) + a(c(1, 0) - c(0, -1))
    P[6, 1:-1, 1:-1] = (c(-1, 0) + c(0, -1) + c(0, 1) + c(1, 0)) >> 1
    return P


def vng_sites(m, code, scale_scalar=SCALE_SCALAR, scale_simd=SCALE_SIMD, simd_start=None, band=256):
    """the computed block: (values (H-6, W-4, 3) for rows 2 .. H-5 and columns 2 .. W-3, ng, arm), in bands of rows.  `scale_scalar`,
    `scale_simd` and `simd_start` exist so that tests can show what a different factor or body start would change."""
    H, W = m.shape
    s = m.astype(np.int32)
    P = vng_planes(m)
    parts = [_vng_band(s, P, code, y, min(y + band, H - 4), scale_scalar, scale_simd, simd_start) for y in range(2, H - 4, band)]
    return tuple(np.concatenate(x) for x in zip(*parts))


def _vng_band(s, P, code, y0, y1, scale_scalar, scale_simd, simd_start):
    H, W = s.shape
    ys = np.arange(y0, y1)[:, None] + 2            # destination row y is computed from the mosaic around row y + 2
    xs = np.arange(2, W - 2)[None, :]
    blue0, green0 = vng_pattern(code)
    g_row = ((ys - 4) & 1).astype(bool) != green0
    green = g_row != ((xs - 2) & 1).astype(bool)
    blue_idx = np.where((ys - 4) & 1, blue0 ^ 2, blue0)
    S = lambda dy, dx: s[ys + dy, xs + dx]
    p = lambda k, dy, dx: P[k][ys + dy, xs + dx].astype(np.int32)

    gN = p(0, -1, 0) + p(0, 0, 0)
    gS = p(0, 0, 0) + p(0, 1, 0)
    gW = p(1, 0, -1) + p(1, 0, 0)
    gE = p(1, 0, 0) + p(1, 0, 1)
    gNE = np.where(green, p(2, -1, 0) + p(2, -1, 1) + p(2, 0, 0) + p(2, 0, 1), p(4, -1, 1) + p(4, 0, 0))
    gSW = np.where(green, p(2, 0, 0) + p(2, 0, -1) + p(2, 1, 0) + p(2, 1, -1), p(4, 0, 0) + p(4, 1, -1))
    gNW = np.where(green, p(3, -1, 0) + p(3, -1, -1) + p(3, 0, 0) + p(3, 0, -1), p(5, -1, -1) + p(5, 0, 0))
    gSE = np.where(green, p(3, 0, 0) + p(3, 0, 1) + p(3, 1, 0) + p(3, 1, 1), p(5, 0, 0) + p(5, 1, 1))
    grads = [gN, gS, gW, gE, gNE, gSW, gNW, gSE]
    mn = np.minimum.reduce(grads)
    mx = np.maximum.reduce(grads)
    T = mn + np.maximum(mx // 2, 1)

    c0 = S(0, 0)
    # per direction: (red/blue-site sums (Rs, Gs, Bs), green-site sums (Rs, Gs, Bs)), in the reference's order N S W E NE SW NW SE
    terms = [
        ((S(-2, 0) + c0, S(-1, 0) * 2, S(-1, -1) + S(-1, 1)), (S(-2, -1) + S(-2, 1), S(-2, 0) + c0, S(-1, 0) * 2)),
        ((S(2, 0) + c0, S(1, 0) * 2, S(1, -1) + S(1, 1)), (S(2, -1) + S(2, 1), S(2, 0) + c0, S(1, 0) * 2)),
        ((S(0, -2) + c0, S(0, -1) * 2, S(-1, -1) + S(1, -1)), (S(0, -1) * 2, S(0, -2) + c0, S(-1, -2) + S(1, -2))),
        ((S(0, 2) + c0, S(0, 1) * 2, S(-1, 1) + S(1, 1)), (S(0, 1) * 2, S(0, 2) + c0, S(-1, 2) + S(1, 2))),
        ((S(-2, 2) + c0, p(6, -1, 1), S(-1, 1) * 2), (S(-2, 1) + S(0, 1), S(-1, 1) * 2, S(-1, 0) + S(-1, 2))),
        ((S(2, -2) + c0, p(6, 1, -1), S(1, -1) * 2), (S(2, -1) + S(0, -1), S(1, -1) * 2, S(1, 0) + S(1, -2))),
        ((S(-2, -2) + c0, p(6, -1, -1), S(-1, -1) * 2), (S(-2, -1) + S(0, -1), S(-1, -1) * 2, S(-1, -2) + S(-1, 0))),
        ((S(2, 2) + c0, p(6, 1, 1), S(1, 1) * 2), (S(2, 1) + S(0, 1), S(1, 1) * 2, S(1, 2) + S(1, 0))),
    ]
    Rs = np.zeros_like(T); Gs = np.zeros_like(T); Bs = np.zeros_like(T); ng = np.zeros_like(T)
    for g, (nz, gz) in zip(grads, terms):
        take = g < T
        Rs += np.where(take, np.where(green, gz[0], nz[0]), 0)
        Gs += np.where(take, np.where(green, gz[1], nz[1]), 0)
        Bs += np.where(take, np.where(green, gz[2], nz[2]), 0)
        ng += take

    arm = np.zeros(green.shape, np.int32)
    for r in range(arm.shape[0]):
        a, b = simd_columns(W, bool(g_row[r, 0]))
        if simd_start is not None:
            a, b = simd_start, simd_start + max(0, (W - 10 - simd_start) // 8 + 1) * 8
        arm[r, max(a - 2, 0):max(b - 2, 0)] = SIMD
    f = np.where(arm == SIMD, scale_simd[ng], scale_scalar[ng]).astype(np.float32)
    rnd = lambda d: np.rint(d.astype(np.float32) * f).astype(np.int32)       # float32 product, round half to even
    # red / blue site: R = sample, G = R + round((Gs - Rs) f), B = R + round((Bs - Rs) f); green site mirrored
    R = np.where(green, c0 + rnd(Rs - Gs), c0)
    G = np.where(green, c0, c0 + rnd(Gs - Rs))
    B = np.where(green, c0 + rnd(Bs - Gs), c0 + rnd(Bs - Rs))
    R, G, B = (np.clip(v, 0, 255) for v in (R, G, B))
    out = np.empty(R.shape + (3,), np.int32)
    out[..., 1] = G
    out[..., 0] = np.where(blue_idx == 0, B, R)
    out[..., 2] = np.where(blue_idx == 0, R, B)
    return out.astype(np.uint8), ng, arm


def vng(m, code, **kw):
    """(dst (H, W, 3) uint8, ng (H, W), arm (H, W)) of cv::cvtColor(m, code) for code 62-65; ng = 0 and arm = SCALAR where the bilinear
    fallback ran"""
    assert m.dtype == np.uint8 and m.ndim == 2 and code in VNG_CODES
    H, W = m.shape
    assert min(H, W) >= 3, "the project refuses W < 3 or H < 3"
    if min(H, W) < 8:
        return bilinear(m, 1, 0), np.zeros((H, W), np.int32), np.zeros((H, W), np.int32)
    vals, ng, arm = vng_sites(m, code, **kw)
    yi = np.clip(np.arange(H), 2, H - 5)[:, None] - 2
    xi = np.clip(np.arange(W), 2, W - 3)[None, :] - 2
    return vals[yi, xi], ng[yi, xi], arm[yi, xi]


def gray(m, code):
    """cv::cvtColor(m, code) for code 86-89, 8- or 16-bit; the sums are unsigned (a 16-bit mosaic reaches 4 294 934 528 > INT_MAX)"""
    assert m.ndim == 2 and m.dtype in (np.uint8, np.uint16) and code in GRAY_CODES
    H, W = m.shape
    if H <= 2 or W <= 2:
        return np.zeros_like(m)
    s = m.astype(np.uint64)
    yi = np.clip(np.arange(H), 1, H - 2)[:, None]
    xi = np.clip(np.arange(W), 1, W - 2)[None, :]
    i, k = yi - 1, xi - 1
    b0, r0 = (B2Y, R2Y) if code in (86, 87) else (R2Y, B2Y)
    swg = ((i & 1) != 0) != (code in (87, 89))
    bco = np.where(i & 1, r0, b0).astype(np.uint64)
    rco = np.where(i & 1, b0, r0).astype(np.uint64)
    green = ((k & 1) == 0) == swg
    at = lambda dy, dx: s[yi + dy, xi + dx]
    t_rb = (at(-1, -1) + at(-1, 1) + at(1, -1) + at(1, 1)) * rco + (at(-1, 0) + at(0, -1) + at(0, 1) + at(1, 0)) * G2Y + at(0, 0) * (4 * bco)
    t_g = (at(-1, 0) + at(1, 0)) * rco + (at(0, -1) + at(0, 1)) * bco + at(0, 0) * (2 * G2Y)
    v = np.where(green, (t_g + (1 << 14)) >> 15, (t_rb + (1 << 15)) >> 16)
    return v.astype(m.dtype)
