// gauss_u8.cu -- the 8-bit single-channel GaussianBlur fast path: TMA tile loads + packed-integer (IDP4A) arithmetic.
//
// Same result as the reference's fixedSmoothInvoker (modules/imgproc/src/smooth.simd.hpp:1925-2197; evaluator
// modules/imgproc/test/test_smooth_bitexact.cpp:40-53):  dst = ((sum_j ky[j] * (sum_i kx[i] * src)) + 2^15) >> 16  with 8.8 taps
// (every tap <= 255 for ksize >= 3), bit for bit.
//
// Per CTA: one 192 x TH output tile (TH = 64-(K-1) rounded down to a multiple of 4).
//   1. ONE thread issues a 3-D TMA box load (cp.async.bulk.tensor) of the 256 x (TH+K-1) byte tile + apron into shared
//      memory; everybody waits on the mbarrier.  TMA zero-fills outside the image = BORDER_CONSTANT; for REPLICATE /
//      REFLECT / REFLECT_101 only CTAs on the image boundary patch their apron cells from the mirrored in-tile cells.
//   2. Row pass: each thread takes 4 columns x 4 rows.  4 taps per IDP4A (u8 x u8 -> u32); the unaligned windows of a
//      group come from PRMT of two aligned shared words.  The 16-bit row sums of vertically adjacent rows (2p, 2p+1) are
//      packed into one word per column (PRMT) and stored to shared memory.
//   3. Column pass: 2 taps per IDP2A (u16 x u8 -> u32) on those vertical pairs, with the tap words pre-shifted on the host
//      for each of the 4 row phases (zero padded) so no data realignment is needed; accumulators start at 2^15.
//      Epilogue: the result byte is bits 16..23 of the sum (never saturates: sum k = 256), picked by PRMT; 4 pixels per
//      32-bit store.
// Instruction budget (K=3): ~1 IDP4A + 2 IDP2A and ~6 other instructions per pixel, against ~46 for the generic float kernel.
#include <vector>
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "tma.cuh"

namespace b200cv {

constexpr int GU_TW = 192;      // output tile width
constexpr int GU_IW = 256;      // staged tile width (bytes) = TMA box width
constexpr int GU_RG = 16;       // row groups of 4 rows staged / processed per tile (64 rows)

struct GU8Params {
    uint32_t kxw[8];            // row taps, 4 per word
    uint32_t kyw[4][9];         // column taps for output row phase o (0..3) and row group g: byte i = ky[4g + i - o] or 0
    int W, H, TH, border;
    int sep_mode, even_limit;   // sepFilter2D's 8.8 fixed-point mode: columns < even_limit round half-to-even, the rest half-up (filter.simd.hpp:1011-1100)
    GU8Box box;                 // sep_mode 2 / 3: cv::boxFilter epilogues on the plain window sum (all taps 1)
};

__host__ __device__ constexpr bool gu_nz(int KB, int o, int g) { return 4 * g - o < KB; }

// Interleaved channels: a row of W pixels x CN channels is a row of W*CN byte ELEMENTS whose horizontal taps are CN elements apart;
// the column pass does not see channels at all.  Tile width in elements so that apron + tile + apron fits one 256-byte TMA box row.
template <int CN> struct GUTile { static constexpr int TW = CN == 1 ? 192 : CN == 3 ? 160 : 128; };

template <int KB, int CN, bool BOX>
__global__ void __launch_bounds__(256, 4) gauss_u8_dp4a_kernel(const __grid_constant__ CUtensorMap tmap, Img dst, const __grid_constant__ GU8Params p)
{
    constexpr int GU_TW = GUTile<CN>::TW;            // (shadows the single-channel constant)
    constexpr int RB = KB / 2;
    constexpr int RBE = RB * CN;                     // horizontal apron in elements
    constexpr int RA = ((RBE + 15) / 16) * 16;       // left apron staged: TMA needs the box to start on a 16-byte boundary
    constexpr int OFF = RA - RBE;                    // tile column of (output column 0, tap 0)
    constexpr int GH = (KB + 3) / 4;                 // tap groups per row
    constexpr int GV = (KB + 3 + 3) / 4;             // row groups touched by one 4-row output group
    static_assert(RA + GU_TW + RBE <= GU_IW, "apron + tile must fit the TMA box");
    __shared__ __align__(128) unsigned char s_in[GU_IW * GU_RG * 4];          // 256 x 64 bytes
    __shared__ __align__(16) uint32_t s_mid[GU_RG * 2 * GU_TW];               // [row pair][column]: (sum of row 2p, sum of row 2p+1) as 2 x u16
    __shared__ __align__(8) uint64_t s_bar;

    const int TH = p.TH, IH = TH + KB - 1;
    const int f = blockIdx.z, x0 = blockIdx.x * GU_TW, y0 = blockIdx.y * TH;
    const int tid = threadIdx.x;

    if (tid == 0) {
        mbar_init(&s_bar, 1);
        fence_barrier_init();
        mbar_arrive_expect_tx(&s_bar, (uint32_t)(GU_IW * IH));
        tma_load_3d(s_in, &tmap, x0 - RA, y0 - RB, f, &s_bar);
        // only this thread polls the barrier; the others sleep in bar.sync instead of spending issue slots on a spin loop
        mbar_wait(&s_bar, 0);
    }
    __syncthreads();

    // ---- border patch (only CTAs whose tile crosses the image boundary; BORDER_CONSTANT needs nothing) ----
    const int tx0 = x0 - RA;                            // image column of tile column 0
    const bool edge = (tx0 < 0) || (y0 - RB < 0) || (tx0 + GU_IW > p.W) || (y0 - RB + IH > p.H);
    if (edge && p.border != B200CV_BORDER_CONSTANT) {
        // rows first (whole rows from the mirrored source row), then columns
        for (int idx = tid; idx < IH * (GU_IW / 4); idx += 256) {
            int r = idx / (GU_IW / 4), c4 = idx - r * (GU_IW / 4);
            int gy = y0 - RB + r;
            if ((unsigned)gy < (unsigned)p.H) continue;
            int sr = border_interpolate(gy, p.H, p.border) - (y0 - RB);
            if ((unsigned)sr < (unsigned)IH)      // rows further than the apron below the image feed no valid output: leave them
                ((uint32_t*)s_in)[r * (GU_IW / 4) + c4] = ((const uint32_t*)s_in)[sr * (GU_IW / 4) + c4];
        }
        __syncthreads();
        {   // columns left of the image (tile columns [0, RA) of the first tile column) and right of it (from c_first on)
            const int c_first = p.W - tx0;
            const int nright = c_first < GU_IW ? min(GU_IW - c_first, RBE + 4) : 0;
            const int nleft = tx0 < 0 ? RA : 0;
            const int ncol = nleft + nright;
            for (int idx = tid; idx < IH * ncol; idx += 256) {
                int r = idx / ncol, k = idx - r * ncol;
                int c = k < nleft ? k : c_first + (k - nleft);
                int sc;
                if (CN == 1) sc = border_interpolate(tx0 + c, p.W, p.border) - tx0;
                else {      // element -> (pixel, channel); the border rule acts on pixels
                    const int e = tx0 + c, px = e >= 0 ? e / CN : -((-e + CN - 1) / CN), ch = e - px * CN;
                    sc = border_interpolate(px, p.W / CN, p.border) * CN + ch - tx0;
                }
                if ((unsigned)sc < (unsigned)GU_IW) s_in[r * GU_IW + c] = s_in[r * GU_IW + sc];
            }
        }
        __syncthreads();
    }

    // ---- row pass: item = 4 columns x 4 rows; (rg, cg) advance without divisions ----
    {
        constexpr int NCG = GU_TW / 4;                               // column groups (48 / 40 / 32)
        int rg = tid / NCG, cg = tid - rg * NCG;
#pragma unroll 1
        for (; rg < GU_RG; ) {
            uint32_t res[4][4];                                      // [row][col] 16-bit sums
            const uint32_t* wp0 = (const uint32_t*)(s_in + (rg * 4) * GU_IW + cg * 4);
#pragma unroll
            for (int r = 0; r < 4; r++) {
                const uint32_t* wp = wp0 + r * (GU_IW / 4);
                // last byte any (column b, tap) of this item touches: OFF + 3 + CN * (KB - 1)
                constexpr int W0 = OFF / 4, W1 = (OFF + 3 + CN * (KB - 1)) / 4 + (CN == 1 ? 1 : 0);
                uint32_t w[W1 - W0 + 1];
#pragma unroll
                for (int j = W0; j <= W1; j++) w[j - W0] = wp[j];
                uint32_t a[4] = {0, 0, 0, 0};
#pragma unroll
                for (int g = 0; g < GH; g++) {
                    const uint32_t t = p.kxw[g];
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        uint32_t win;
                        if constexpr (CN == 1) {
                            const int tot = OFF + b + 4 * g, wi = tot / 4 - W0, sh = tot % 4;     // compile-time after unrolling
                            win = sh == 0 ? w[wi] : __byte_perm(w[wi], w[wi + 1], sh == 1 ? 0x4321 : sh == 2 ? 0x5432 : 0x6543);
                        } else {
                            // taps 4g .. 4g+3 of output column b are CN bytes apart; taps beyond KB-1 carry zero weights: reuse the last real one
                            int pos[4];
#pragma unroll
                            for (int q = 0; q < 4; q++) pos[q] = OFF + b + CN * (4 * g + q < KB ? 4 * g + q : KB - 1);
                            const uint32_t lo = __byte_perm(w[pos[0] / 4 - W0], w[pos[1] / 4 - W0], (unsigned)((pos[0] & 3) | ((4 + (pos[1] & 3)) << 4)));
                            const uint32_t hi = __byte_perm(w[pos[2] / 4 - W0], w[pos[3] / 4 - W0], (unsigned)((pos[2] & 3) | ((4 + (pos[3] & 3)) << 4)));
                            win = __byte_perm(lo, hi, 0x5410);
                        }
                        a[b] = __dp4a(win, t, a[b]);
                    }
                }
                res[r][0] = a[0]; res[r][1] = a[1]; res[r][2] = a[2]; res[r][3] = a[3];
            }
            // vertical pairs: word = (row 2p, row 2p+1) of one column
            uint32_t* mp = s_mid + (rg * 2) * GU_TW + cg * 4;
            *(uint4*)mp = make_uint4(__byte_perm(res[0][0], res[1][0], 0x5410), __byte_perm(res[0][1], res[1][1], 0x5410),
                                     __byte_perm(res[0][2], res[1][2], 0x5410), __byte_perm(res[0][3], res[1][3], 0x5410));
            *(uint4*)(mp + GU_TW) = make_uint4(__byte_perm(res[2][0], res[3][0], 0x5410), __byte_perm(res[2][1], res[3][1], 0x5410),
                                               __byte_perm(res[2][2], res[3][2], 0x5410), __byte_perm(res[2][3], res[3][3], 0x5410));
            cg += 256 % NCG; rg += 256 / NCG;
            if (cg >= NCG) { cg -= NCG; rg += 1; }
        }
    }
    __syncthreads();

    // ---- column pass: item = 4 columns x 4 output rows ----
    {
        constexpr int NCG = GU_TW / 4;
        const bool vec_store = (((uintptr_t)dst.data | dst.step | dst.fstep) & 3) == 0;
        const bool full = vec_store && x0 + GU_TW <= p.W && y0 + TH <= p.H;      // interior tile: no bounds checks at all
        const int nq = TH / 4;
        int q = tid / NCG, cg = tid - q * NCG;
        uchar* dbase = dst.row<uchar>(f, y0) + x0;
        const size_t dstep = dst.step;
#pragma unroll 1
        for (; q < nq; ) {
            uint32_t acc[4][4];                                           // [output row][column], start at the rounding constant
#pragma unroll
            for (int o = 0; o < 4; o++)
#pragma unroll
                for (int c = 0; c < 4; c++) acc[o][c] = BOX ? 0u : p.sep_mode ? 32767u : 32768u;
            const uint32_t* mp0 = s_mid + (q * 2) * GU_TW + cg * 4;
#pragma unroll
            for (int g = 0; g < GV; g++) {
                // rows 4g, 4g+1 (pair 2g) and 4g+2, 4g+3 (pair 2g+1) of this item; tap word bytes 0..3 = taps of rows 4g..4g+3 for phase o
                const bool need_lo = 4 * g - 3 < KB, need_hi = 4 * g + 2 - 3 < KB;       // any phase o in 0..3 touches them
                uint4 m0 = make_uint4(0, 0, 0, 0), m1 = make_uint4(0, 0, 0, 0);
                if (need_lo) m0 = *(const uint4*)(mp0 + (2 * g) * GU_TW);
                if (need_hi) m1 = *(const uint4*)(mp0 + (2 * g + 1) * GU_TW);
                const uint32_t a0[4] = {m0.x, m0.y, m0.z, m0.w}, a1[4] = {m1.x, m1.y, m1.z, m1.w};
#pragma unroll
                for (int o = 0; o < 4; o++) {
                    const uint32_t t = p.kyw[o][g];
                    if (4 * g + 1 - o >= 0 && 4 * g - o < KB) {
#pragma unroll
                        for (int c = 0; c < 4; c++) acc[o][c] = __dp2a_lo(a0[c], t, acc[o][c]);
                    }
                    if (4 * g + 3 - o >= 0 && 4 * g + 2 - o < KB) {
#pragma unroll
                        for (int c = 0; c < 4; c++) acc[o][c] = __dp2a_hi(a1[c], t, acc[o][c]);
                    }
                }
            }
            if constexpr (BOX) {                                         // box filter: result byte goes to bits 16..23 for the pack below
                const bool body = x0 + cg * 4 < p.box.tail_from;         // uniform over the 4 columns: tail_from is a multiple of 8
#pragma unroll
                for (int o = 0; o < 4; o++)
#pragma unroll
                    for (int c = 0; c < 4; c++) {
                        const uint32_t s = acc[o][c];
                        uint32_t r;
                        if (!p.box.have_scale) r = min(s, 255u) << 16;
                        else if (p.sep_mode == 2) r = ((s + p.box.div_delta) * p.box.div_scale) >> 7;
                        else r = (uint32_t)min(body ? __float2int_rn(__fmul_rn(__uint2float_rn(s), p.box.scale_f)) : __double2int_rn(__dmul_rn((double)s, p.box.scale)), 255) << 16;
                        acc[o][c] = r;
                    }
            } else if (p.sep_mode) {
                const bool half_even = x0 + cg * 4 < p.even_limit;      // uniform over the 4 columns: even_limit is a multiple of 16
#pragma unroll
                for (int o = 0; o < 4; o++)
#pragma unroll
                    for (int c = 0; c < 4; c++) acc[o][c] += half_even ? (((acc[o][c] - 32767u) >> 16) & 1u) : 1u;
            }
            uint32_t packed[4];
#pragma unroll
            for (int o = 0; o < 4; o++)
                packed[o] = __byte_perm(__byte_perm(acc[o][0], acc[o][1], 0x0062), __byte_perm(acc[o][2], acc[o][3], 0x0062), 0x5410);
            uchar* dp = dbase + (size_t)(q * 4) * dstep + cg * 4;
            if (full) {
#pragma unroll
                for (int o = 0; o < 4; o++) *(uint32_t*)(dp + o * dstep) = packed[o];
            } else {
                const int gx = x0 + cg * 4;
#pragma unroll
                for (int o = 0; o < 4; o++) {
                    const int gy = y0 + q * 4 + o;
                    if (gy < p.H && gx < p.W) {
                        if (vec_store && gx + 4 <= p.W) *(uint32_t*)(dp + o * dstep) = packed[o];
                        else {
#pragma unroll
                            for (int c = 0; c < 4; c++) if (gx + c < p.W) dp[o * dstep + c] = (uchar)(packed[o] >> (8 * c));
                        }
                    }
                }
            }
            cg += 256 % NCG; q += 256 / NCG;
            if (cg >= NCG) { cg -= NCG; q += 1; }
        }
    }
}

template <int KB, int CN>
static int launch_gu8_cn(const CUtensorMap& tm, const Img& d, const GU8Params& p, int frames, cudaStream_t st)
{
    auto kern = p.sep_mode >= 2 ? gauss_u8_dp4a_kernel<KB, CN, true> : gauss_u8_dp4a_kernel<KB, CN, false>;
    dim3 grid(div_up((unsigned)p.W, GUTile<CN>::TW), div_up((unsigned)p.H, (unsigned)p.TH), (unsigned)frames);
    kern<<<grid, 256, 0, st>>>(tm, d, p);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

template <int KB>
static int launch_gu8(const CUtensorMap& tm, const Img& d, const GU8Params& p, int frames, int cn, cudaStream_t st)
{
    if (cn == 1) return launch_gu8_cn<KB, 1>(tm, d, p, frames, st);
    if (cn == 3) return launch_gu8_cn<KB, 3>(tm, d, p, frames, st);
    return launch_gu8_cn<KB, 4>(tm, d, p, frames, st);
}

// returns B200CV_NOT_IMPLEMENTED when the fast path does not apply (caller falls back to the generic kernel)
int gauss_u8_fast(const Img& s, const Img& d, int cn, const int64_t* fx, int kw, const int64_t* fy, int kh, int border, cudaStream_t st, int sep_mode, int even_limit,
                  const GU8Box* box)
{
    if (cn != 1 && cn != 3 && cn != 4) return B200CV_NOT_IMPLEMENTED;
    if (!(kw & 1) || !(kh & 1) || kw < 3 || kh < 3 || kw > 31 || kh > 31) return B200CV_NOT_IMPLEMENTED;
    if (border == B200CV_BORDER_WRAP) return B200CV_NOT_IMPLEMENTED;
    if (!tma_compatible(s) || s.rows >= 65536 * 4 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    static const int buckets[] = {3, 5, 7, 9, 11, 13, 15, 17, 21, 25, 27, 31};
    int kmax = kw > kh ? kw : kh, KB = 0;
    for (int b : buckets) if (kmax <= b) { KB = b; break; }
    if (!KB || s.cols < KB || s.rows < KB) return B200CV_NOT_IMPLEMENTED;
    for (int i = 0; i < kw; i++) if (fx[i] < 0 || fx[i] > 255) return B200CV_NOT_IMPLEMENTED;
    for (int i = 0; i < kh; i++) if (fy[i] < 0 || fy[i] > 255) return B200CV_NOT_IMPLEMENTED;
    int64_t sx = 0, sy = 0;
    for (int i = 0; i < kw; i++) sx += fx[i];
    for (int i = 0; i < kh; i++) sy += fy[i];
    if (sx > 256 || sy > 256) return B200CV_NOT_IMPLEMENTED;      // 16-bit row sums and an unsaturated result byte
    // GaussianBlur 3 x 3 / 5 x 5 with the binomial 8.8 taps (sigma = 0), one channel, 16-byte aligned rows of a multiple of 16 pixels: packed
    // 16-bit adds, no multiplier, rows through a lane-private cp.async ring (gauss_u8_binomial.cu).  The TMA tile kernel below keeps every other case
    // and is forced by B200CV_GAUSS_U8_PATH=tile (tests run both)
    if (sep_mode == 0 && !box) {
        const char* e = getenv("B200CV_GAUSS_U8_PATH");
        if (!(e && (!strcmp(e, "tile") || !strcmp(e, "stream")))) {
            const int brc = gauss_u8_binomial(s, d, cn, fx, kw, fy, kh, border, st);
            if (brc != B200CV_NOT_IMPLEMENTED) return brc;
        }
    }
    GU8Params p;
    memset(&p, 0, sizeof(p));
    unsigned char tx[36] = {0}, ty[36] = {0};
    for (int i = 0; i < kw; i++) tx[(KB - kw) / 2 + i] = (unsigned char)fx[i];
    for (int i = 0; i < kh; i++) ty[(KB - kh) / 2 + i] = (unsigned char)fy[i];
    for (int g = 0; g < 8; g++) p.kxw[g] = tx[4 * g] | (tx[4 * g + 1] << 8) | (tx[4 * g + 2] << 16) | ((uint32_t)tx[4 * g + 3] << 24);
    for (int o = 0; o < 4; o++)
        for (int g = 0; g < 9; g++) {
            uint32_t w = 0;
            for (int i = 0; i < 4; i++) { int j = 4 * g + i - o; if (j >= 0 && j < KB) w |= (uint32_t)ty[j] << (8 * i); }
            p.kyw[o][g] = w;
        }
    // single channel, K <= 9, Gaussian / 8.8 sepFilter2D epilogues: the warp-streaming register kernel (gauss_u8_march.cu) exists as a second
    // version; it executes fewer instructions per pixel but gives the memory system less in flight (per-warp chunks), so the tile kernel
    // below stays the default; B200CV_GAUSS_U8_PATH=stream selects it (tests run both)
    {
        const char* e = getenv("B200CV_GAUSS_U8_PATH");
        if (e && !strcmp(e, "stream") && cn == 1 && KB <= 9 && sep_mode <= 1) return gauss_u8_march(s, d, KB, tx, ty, border, st, sep_mode, even_limit);
    }
    p.W = s.cols * cn; p.H = s.rows; p.border = border; p.sep_mode = sep_mode; p.even_limit = even_limit;      // W in byte elements
    if (box) p.box = *box;
    p.TH = ((64 - (KB - 1)) / 4) * 4;
    CUtensorMap tm;
    int rc = make_tensor_map_3d(&tm, s.data, 1, s.cols * cn, s.rows, s.frames, s.step, s.fstep, GU_IW, p.TH + KB - 1);   // box start x0-RA: 16-byte aligned
    if (rc) return rc;
    switch (KB) {
    case 3: return launch_gu8<3>(tm, d, p, s.frames, cn, st);
    case 5: return launch_gu8<5>(tm, d, p, s.frames, cn, st);
    case 7: return launch_gu8<7>(tm, d, p, s.frames, cn, st);
    case 9: return launch_gu8<9>(tm, d, p, s.frames, cn, st);
    case 11: return launch_gu8<11>(tm, d, p, s.frames, cn, st);
    case 13: return launch_gu8<13>(tm, d, p, s.frames, cn, st);
    case 15: return launch_gu8<15>(tm, d, p, s.frames, cn, st);
    case 17: return launch_gu8<17>(tm, d, p, s.frames, cn, st);
    case 21: return launch_gu8<21>(tm, d, p, s.frames, cn, st);
    case 25: return launch_gu8<25>(tm, d, p, s.frames, cn, st);
    case 27: return launch_gu8<27>(tm, d, p, s.frames, cn, st);
    case 31: return launch_gu8<31>(tm, d, p, s.frames, cn, st);
    }
    return B200CV_NOT_IMPLEMENTED;
}

}  // namespace b200cv
