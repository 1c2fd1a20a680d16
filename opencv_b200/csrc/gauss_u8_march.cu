// gauss_u8_march.cu -- 8-bit single-channel GaussianBlur / 8.8 fixed-point sepFilter2D for kernels up to 9x9: every WARP streams down a
// 224-column strip of the image, TMA chunks double-buffered in shared memory, the whole separable filter in registers.  Second version of
// gauss_u8.cu's kernel for the sizes the north star names (that kernel stays for 3-/4-channel rows, box filters and 11 <= K <= 31).
//
// Same arithmetic as the reference's fixedSmoothInvoker<uint8_t, ufixedpoint16> (modules/imgproc/src/smooth.simd.hpp:1925-2197;
// evaluator modules/imgproc/test/test_smooth_bitexact.cpp:40-53):
//     dst = ((sum_j ky[j] * (sum_i kx[i] * src)) + 2^15) >> 16      8.8 taps, 16-bit row sums, bit for bit.
//
// History: v1 (gauss_u8.cu) = row pass -> shared memory -> barrier -> column pass on 4 x 4 items, instruction-issue bound.  v2 = one CTA
// per 224 x 128 tile, registers only: fewer instructions per pixel, but the warps waited in the CTA barrier behind the tile's TMA load, and
// each warp filtered K-1 rows twice.  v3 (this file):
//   * worker = one warp.  It owns (frame, 224-column strip, segment of rows) and walks DOWN it in chunks of CH rows: lane 0 issues one
//     3-D TMA box (256 x CH bytes) per chunk into one of the warp's two private buffers, one chunk ahead; completion on the warp's own
//     mbarrier.  No CTA-wide barrier anywhere, no launch per tile: the grid is one wave of 4-warp CTAs, each warp loops over its items.
//   * borders: TMA's zero fill is BORDER_CONSTANT.  For the other rules, chunks that reach above / below the image are loaded row by row
//     (256 x 1 boxes) from the mirrored source row, and strips that touch the left / right edge patch their apron columns in shared memory.
//   * a lane holds 8 adjacent columns (lanes 0, 1, 30, 31 only cover the 16-byte aprons the TMA box alignment needs) and per chunk row pair:
//       row pass    the 16 bytes around its columns are 4 aligned words (LDS.64 + 2 LDS.32); every row sum is 1-3 IDP4A against tap
//                   words pre-shifted on the host for the 4 byte phases -- no window extraction (PRMT) at all;
//       pairing     the sums of rows (2j, 2j+1) are packed into one word per column (1 PRMT per 2 pixels);
//       column pass a register window of K/2+1 such pairs per column that lives ACROSS chunks (every source row is filtered once);
//                   output rows (2m, 2m+1) are K/2+1 IDP2A each against tap words holding the even-row taps in bytes 0-1 and the odd-row
//                   taps in bytes 2-3; the window rotates by loop unrolling (CH/2 is a multiple of K/2+1);
//       epilogue    result byte = bits 16..23 (3 PRMT per 4 pixels), one 64-bit store per lane and row.
// IDP runs on the half-rate FMA-heavy pipe: 3.5 / 5 / 6.5 / 8 IDP per pixel at K = 3 / 5 / 7 / 9 bound K = 7 and 9 below the HBM
// roofline whatever else is done.
#include <string.h>
#include <algorithm>
#include "common.cuh"
#ifndef B200CV_HOST_EMULATION
#include "tma.cuh"
#endif

namespace b200cv {

constexpr int GM_IW = 256;      // staged tile width in bytes = TMA box width
constexpr int GM_OW = 224;      // output columns per tile (28 lanes x 8)
constexpr int GM_RA = 16;       // left / right apron staged (TMA: the box must start on a 16-byte boundary)

template <int KB> struct GMCfg {
    static constexpr int H = KB / 2, NP = H + 1;                                     // NP = pairs in the column window
    static constexpr int CH = KB == 3 ? 8 : KB == 5 ? 12 : KB == 7 ? 8 : 10;         // rows per chunk: CH/2 is a multiple of NP (small chunks: 4-5 KB per warp keep 32 warps per SM resident)
    static constexpr int BUFB = 256 * CH;                                            // bytes per chunk buffer
    static_assert((CH / 2) % NP == 0 && CH % 2 == 0 && CH / 2 >= H, "the window rotation needs CH/2 to be a multiple of K/2+1");
};
constexpr int GM_WARPS = 4;     // workers per CTA

struct GMParams {
    uint32_t tx[4][3];          // row taps: [start byte & 3][word]: byte b = kx[4*word + b - phase] or 0
    uint32_t ty[5];             // column taps for window pair i: bytes 0,1 = (ky[2i], ky[2i+1]) for even output rows, bytes 2,3 = (ky[2i-1], ky[2i]) for odd ones
    int W, H, border;
    int sep_mode, even_limit;   // sepFilter2D's 8.8 mode: columns < even_limit round half-to-even, the rest half-up (filter.simd.hpp:1011-1100)
    int tiles_x, nseg, seg_rows, nitems;   // work decomposition: item = (frame, strip, segment), item = (f * nseg + seg) * tiles_x + strip
    int* queue;                            // dynamic distribution: items beyond the first wave are drawn from this counter (zeroed per launch)
};

// 16-bit row sums of the lane's 8 columns for one staged row.  rp = the lane's own 8 bytes of that row.
template <int KB>
__device__ __forceinline__ void gm_row(const unsigned char* rp, int loff, int roff, const GMParams& p, uint32_t rs[8])
{
    constexpr int H = KB / 2;
    const uint2 own = *(const uint2*)rp;
    const uint32_t w[4] = {*(const uint32_t*)(rp + loff), own.x, own.y, *(const uint32_t*)(rp + roff)};
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const int a = 4 + c - H, ph = a & 3, w0 = a >> 2, nw = (ph + KB + 3) / 4;     // compile-time after unrolling
        uint32_t acc = 0;
#pragma unroll
        for (int q = 0; q < nw; q++) acc = __dp4a(w[w0 + q], p.tx[ph][q], acc);
        rs[c] = acc;
    }
}

// packed (row 2j, row 2j+1) sums for the lane's 8 columns; rp = the lane's own bytes of row 2j
template <int KB>
__device__ __forceinline__ void gm_pair(const unsigned char* rp, int loff, int roff, const GMParams& p, uint32_t out[8])
{
    uint32_t r0[8], r1[8];
    gm_row<KB>(rp, loff, roff, p, r0);
    gm_row<KB>(rp + GM_IW, loff, roff, p, r1);
#pragma unroll
    for (int c = 0; c < 8; c++) out[c] = __byte_perm(r0[c], r1[c], 0x5410);
}

__device__ __forceinline__ uint2 gm_pack8(const uint32_t a[8])      // byte 2 of every accumulator
{
    uint2 r;
    r.x = __byte_perm(__byte_perm(a[0], a[1], 0x0062), __byte_perm(a[2], a[3], 0x0062), 0x5410);
    r.y = __byte_perm(__byte_perm(a[4], a[5], 0x0062), __byte_perm(a[6], a[7], 0x0062), 0x5410);
    return r;
}

// checked stores of two output rows (chunks at the ends of a segment, partial strips, unaligned destinations): out of line, the hot
// loop stays small (the unrolled byte stores made the kernel 57 KB of code and the warps stalled on instruction fetch)
__device__ __noinline__ void gm_store_checked(unsigned char* d0, size_t dstep, uint2 pe, uint2 po, int ncols, bool row1, bool vec)
{
    if (vec) {
        *(uint2*)d0 = pe;
        if (row1) *(uint2*)(d0 + dstep) = po;
        return;
    }
#pragma unroll 1
    for (int c = 0; c < ncols; c++) {
        d0[c] = (unsigned char)((c < 4 ? pe.x : pe.y) >> (8 * (c & 3)));
        if (row1) d0[dstep + c] = (unsigned char)((c < 4 ? po.x : po.y) >> (8 * (c & 3)));
    }
}

// One chunk of CH rows for one lane.  rp = the lane's own 8 bytes in row 0 of the chunk buffer; win = the lane's window, which lives across
// chunks; m_first = output row pair produced by the chunk's first source pair (negative in a segment's first chunk: the window is filling);
// dp = destination of output row 2 * m_first at the lane's first column (never dereferenced for rows outside [0, nrows)).
// FAST: every output row of the chunk exists, all 8 columns exist, 64-bit stores are aligned -- no checks at all.
template <int KB, bool SEP, bool FAST>
__device__ __forceinline__ void gm_chunk(const unsigned char* rp, const GMParams& p, uint32_t (&win)[GMCfg<KB>::NP][8], unsigned char* dp, size_t dstep,
                                         int m_first, int nrows, int ncols, bool vec, bool half_even)
{
    constexpr int H = GMCfg<KB>::H, NP = GMCfg<KB>::NP, CH = GMCfg<KB>::CH;
#pragma unroll
    for (int jl = 0; jl < CH / 2; jl++) {
        gm_pair<KB>(rp + (2 * jl) * GM_IW, -4, 8, p, win[jl % NP]);          // global pair index = chunk * CH/2 + jl, CH/2 = 0 mod NP
        const int y = 2 * (m_first + jl);
        if (FAST || (y >= 0 && y < nrows)) {
            uint32_t e[8], o[8];
#pragma unroll
            for (int c = 0; c < 8; c++) { e[c] = SEP ? 32767u : 32768u; o[c] = e[c]; }
#pragma unroll
            for (int i = 0; i < NP; i++) {
                const uint32_t t = p.ty[i];
                const int slot = ((jl - H + i) % NP + NP) % NP;               // pair (m + i) of output pair m = (this pair) - H
#pragma unroll
                for (int c = 0; c < 8; c++) {
                    e[c] = __dp2a_lo(win[slot][c], t, e[c]);
                    o[c] = __dp2a_hi(win[slot][c], t, o[c]);
                }
            }
            if (SEP) {
#pragma unroll
                for (int c = 0; c < 8; c++) {
                    e[c] += half_even ? (((e[c] - 32767u) >> 16) & 1u) : 1u;
                    o[c] += half_even ? (((o[c] - 32767u) >> 16) & 1u) : 1u;
                }
            }
            const uint2 pe = gm_pack8(e), po = gm_pack8(o);
            unsigned char* d0 = dp + (size_t)(2 * jl) * dstep;
            if (FAST) {
                *(uint2*)d0 = pe;
                *(uint2*)(d0 + dstep) = po;
            } else {
                gm_store_checked(d0, dstep, pe, po, ncols, y + 1 < nrows, vec);
            }
        }
    }
}

// item -> geometry
struct GMItem { int f, x0, ys, rows, nchunks; };
template <int KB> __host__ __device__ __forceinline__ GMItem gm_item(const GMParams& p, int item)
{
    constexpr int H = GMCfg<KB>::H, CH = GMCfg<KB>::CH;
    GMItem g;
    const int strip = item % p.tiles_x, t = item / p.tiles_x, seg = t % p.nseg;
    g.f = t / p.nseg;
    g.x0 = strip * GM_OW;
    g.ys = seg * p.seg_rows;
    g.rows = min(p.seg_rows, p.H - g.ys);
    g.nchunks = (g.rows + 2 * H + CH - 1) / CH;          // source rows ys - H .. ys + rows - 1 + H
    return g;
}

// what one lane does with one staged chunk (the kernel after the wait + patch; tests/test_kernel_emulation.py on the host)
template <int KB, bool SEP>
__device__ __forceinline__ void gm_lane_chunk(const unsigned char* buf, int lane, const GMParams& p, const Img& dst, const GMItem& g, int chunk,
                                              uint32_t (&win)[GMCfg<KB>::NP][8])
{
    constexpr int H = GMCfg<KB>::H, CH = GMCfg<KB>::CH;
    const int gx = g.x0 + (lane - 2) * 8;
    int ncols = (lane < 2 || lane >= 30) ? 0 : min(8, p.W - gx);
    if (ncols <= 0) return;                                    // apron lanes and lanes right of the image
    const int m_first = chunk * (CH / 2) - H;
    const bool aligned = (((uintptr_t)dst.data | dst.step | dst.fstep) & 7) == 0;
    const bool vec = ncols == 8 && aligned;
    const bool half_even = SEP && gx < p.even_limit;           // uniform over the 8 columns: even_limit is a multiple of 16, gx of 8
    unsigned char* dp = dst.data + (size_t)g.f * dst.fstep + ((ptrdiff_t)g.ys + 2 * m_first) * (ptrdiff_t)dst.step + gx;
    // warp-uniform: the strip is fully inside the image, so every working lane has 8 columns
    const bool fast = aligned && g.x0 + GM_OW <= p.W && m_first >= 0 && 2 * (m_first + CH / 2) <= g.rows;
    const unsigned char* rp = buf + lane * 8;
    if (fast) gm_chunk<KB, SEP, true>(rp, p, win, dp, dst.step, m_first, g.rows, 8, true, half_even);
    else gm_chunk<KB, SEP, false>(rp, p, win, dp, dst.step, m_first, g.rows, ncols, vec, half_even);
}

#ifndef B200CV_HOST_EMULATION
template <int KB, bool SEP>
__global__ void __launch_bounds__(GM_WARPS * 32, KB <= 5 ? 8 : 6)
gauss_u8_stream_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_row, const Img dst, const __grid_constant__ GMParams p)
{
    constexpr int H = GMCfg<KB>::H, NP = GMCfg<KB>::NP, CH = GMCfg<KB>::CH, BUFB = GMCfg<KB>::BUFB;
    __shared__ __align__(128) unsigned char s_buf[GM_WARPS * 2 * BUFB];
    __shared__ __align__(8) uint64_t s_bar[GM_WARPS * 2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned char* buf = s_buf + warp * 2 * BUFB;
    uint64_t* bar = s_bar + warp * 2;
    const int nwk = gridDim.x * GM_WARPS;
    int item = blockIdx.x * GM_WARPS + warp;
    if (item >= p.nitems) return;
    if (lane == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); fence_barrier_init(); }
    __syncwarp();

    // lane 0: one chunk -> buffer b.  Chunks inside the image: one box; chunks reaching above / below it under a mirroring border rule:
    // row by row from the mirrored source row (rows TMA would zero-fill)
    auto issue = [&](const GMItem& g, int chunk, int b) {
        const int gy0 = g.ys - H + chunk * CH;
        mbar_arrive_expect_tx(&bar[b], (uint32_t)BUFB);
        if (p.border != B200CV_BORDER_CONSTANT && (gy0 < 0 || gy0 + CH > p.H)) {
            for (int r = 0; r < CH; r++)
                tma_load_3d(buf + b * BUFB + r * GM_IW, &tmap_row, g.x0 - GM_RA, border_interpolate(gy0 + r, p.H, p.border), g.f, &bar[b]);
        } else {
            tma_load_3d(buf + b * BUFB, &tmap, g.x0 - GM_RA, gy0, g.f, &bar[b]);
        }
    };

    GMItem g = gm_item<KB>(p, item);
    GMItem gn = g;                       // producer side: one chunk ahead of the consumer
    int n_item = item, n_chunk = 0;
    if (lane == 0) issue(g, 0, 0);
    uint32_t win[NP][8];
#pragma unroll
    for (int i = 0; i < NP; i++)
#pragma unroll
        for (int c = 0; c < 8; c++) win[i][c] = 0;
    int seq = 0;                         // chunks consumed so far: buffer = seq & 1, parity = (seq >> 1) & 1
    int chunk = 0;
    while (true) {
        // ---- prefetch the next chunk (this item's, or the first of the next item drawn from the queue) into the other buffer ----
        if (n_chunk + 1 < gn.nchunks) n_chunk++;
        else {
            int v = 0;
            if (lane == 0) v = nwk + atomicAdd(p.queue, 1);            // the first nwk items were dealt out statically
            n_item = __shfl_sync(0xffffffffu, v, 0);
            n_chunk = 0;
            if (n_item < p.nitems) gn = gm_item<KB>(p, n_item);
        }
        __syncwarp();                    // every lane is done reading the other buffer (chunk seq - 1)
        if (n_item < p.nitems && lane == 0) { fence_proxy_async(); issue(gn, n_chunk, (seq + 1) & 1); }
        // ---- wait for this chunk ----
        const int b = seq & 1;
        while (!mbar_try_wait(&bar[b], (uint32_t)((seq >> 1) & 1))) {}
        unsigned char* cb = buf + b * BUFB;
        // ---- strips on the left / right image edge: apron columns from the mirrored in-row bytes ----
        const int tx0 = g.x0 - GM_RA;
        if (p.border != B200CV_BORDER_CONSTANT && (tx0 < 0 || tx0 + GM_IW > p.W)) {
            const int c_first = p.W - tx0;                                      // first staged column right of the image
            const int nright = c_first < GM_IW ? min(GM_IW - c_first, H + 8) : 0;
            const int nleft = tx0 < 0 ? GM_RA : 0;
            const int ncol = nleft + nright;
            for (int idx = lane; idx < CH * ncol; idx += 32) {
                const int r = idx / ncol, k = idx - r * ncol;
                const int c = k < nleft ? k : c_first + (k - nleft);
                const int sc = border_interpolate(tx0 + c, p.W, p.border) - tx0;
                if ((unsigned)sc < (unsigned)GM_IW) cb[r * GM_IW + c] = cb[r * GM_IW + sc];
            }
            __syncwarp();
        }
        gm_lane_chunk<KB, SEP>(cb, lane, p, dst, g, chunk, win);
        // ---- advance: after an item's last chunk the producer already stands on the next item ----
        seq++;
        if (++chunk == g.nchunks) {
            item = n_item; chunk = 0;
            if (item >= p.nitems) break;
            g = gn;
        }
    }
}

template <int KB>
static int launch_gm(const CUtensorMap& tm, const CUtensorMap& tm_row, const Img& d, GMParams& p, int frames, cudaStream_t st)
{
    constexpr int CH = GMCfg<KB>::CH;
    auto k0 = gauss_u8_stream_kernel<KB, false>;
    auto k1 = gauss_u8_stream_kernel<KB, true>;
    int cps = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, p.sep_mode ? k1 : k0, GM_WARPS * 32, 0));
    if (cps < 1) cps = 1;
    const int capacity = num_sms() * cps * GM_WARPS;            // workers in one wave
    // decomposition: strips x frames x segments of ~64 rows.  One wave of CTAs; a warp that finishes its item draws the next from an atomic
    // counter.  (A static split into exactly one item per warp left the SMs idle for 30 % of the kernel: warps that share an SM with more
    // or slower neighbours finish late, and nothing can be moved to the SMs that are already done.)
    p.tiles_x = (int)div_up((unsigned)p.W, GM_OW);
    const long strips = (long)p.tiles_x * frames;
    p.seg_rows = (int)div_up(64u, CH) * CH;
    if (strips * div_up((unsigned)p.H, (unsigned)p.seg_rows) < 2L * capacity)         // small images: shorter segments, so that every warp gets work
        p.seg_rows = (int)std::max<long>(CH, (long)div_up((unsigned)std::max<long>(1, (long)p.H * strips / (2L * capacity)), CH) * CH);
    p.nseg = (int)div_up((unsigned)p.H, (unsigned)p.seg_rows);
    const long nitems = strips * p.nseg;
    if (nitems >= (1L << 30)) return B200CV_NOT_IMPLEMENTED;
    p.nitems = (int)nitems;
    const unsigned grid = (unsigned)((nitems < capacity ? nitems : capacity) + GM_WARPS - 1) / GM_WARPS;
    int* queue = nullptr;
    B200_CUDA(cudaMallocAsync(&queue, sizeof(int), st));
    B200_CUDA(cudaMemsetAsync(queue, 0, sizeof(int), st));
    p.queue = queue;
    if (p.sep_mode) k1<<<grid, GM_WARPS * 32, 0, st>>>(tm, tm_row, d, p);
    else k0<<<grid, GM_WARPS * 32, 0, st>>>(tm, tm_row, d, p);
    cudaError_t e = cudaGetLastError();
    cudaFreeAsync(queue, st);
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}
#endif

// taps already padded / centred to KB entries
void gm_fill_params(GMParams& p, int KB, const unsigned char* tx, const unsigned char* ty)
{
    memset(&p, 0, sizeof(p));
    for (int ph = 0; ph < 4; ph++)
        for (int q = 0; q < 3; q++) {
            uint32_t w = 0;
            for (int b = 0; b < 4; b++) { const int t = 4 * q + b - ph; if (t >= 0 && t < KB) w |= (uint32_t)tx[t] << (8 * b); }
            p.tx[ph][q] = w;
        }
    const int H = KB / 2;
    for (int i = 0; i <= H; i++) {
        const uint32_t e_lo = ty[2 * i], e_hi = 2 * i + 1 < KB ? ty[2 * i + 1] : 0, o_lo = i > 0 ? ty[2 * i - 1] : 0, o_hi = ty[2 * i];
        p.ty[i] = e_lo | (e_hi << 8) | (o_lo << 16) | (o_hi << 24);
    }
}

#ifndef B200CV_HOST_EMULATION
// single-channel, odd KB <= 9, taps 0..255 with sum <= 256 (checked by the caller): returns NOT_IMPLEMENTED otherwise
int gauss_u8_march(const Img& s, const Img& d, int KB, const unsigned char* tx, const unsigned char* ty, int border, cudaStream_t st, int sep_mode, int even_limit)
{
    if (KB != 3 && KB != 5 && KB != 7 && KB != 9) return B200CV_NOT_IMPLEMENTED;
    GMParams p;
    gm_fill_params(p, KB, tx, ty);
    p.W = s.cols; p.H = s.rows; p.border = border; p.sep_mode = sep_mode; p.even_limit = even_limit;
    const int CH = KB == 3 ? GMCfg<3>::CH : KB == 5 ? GMCfg<5>::CH : KB == 7 ? GMCfg<7>::CH : GMCfg<9>::CH;
    CUtensorMap tm, tm_row;
    int rc = make_tensor_map_3d(&tm, s.data, 1, s.cols, s.rows, s.frames, s.step, s.fstep, GM_IW, CH);
    if (rc) return rc;
    if ((rc = make_tensor_map_3d(&tm_row, s.data, 1, s.cols, s.rows, s.frames, s.step, s.fstep, GM_IW, 1))) return rc;
    switch (KB) {
    case 3: return launch_gm<3>(tm, tm_row, d, p, s.frames, st);
    case 5: return launch_gm<5>(tm, tm_row, d, p, s.frames, st);
    case 7: return launch_gm<7>(tm, tm_row, d, p, s.frames, st);
    default: return launch_gm<9>(tm, tm_row, d, p, s.frames, st);
    }
}
#endif

}  // namespace b200cv
