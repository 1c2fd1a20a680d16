// filter2d_tc_f32.cu -- float single-channel cv::filter2D with >= 130 taps on Hopper tensor cores (wgmma with BF16 operands and FP32
// accumulators in registers): exactly the sizes at which the reference leaves its direct sum for a float DFT
// (dft_filter_size, filter.dispatch.cpp:1288-1290; its own tolerance there is 1e-4 of the value range, test_filter.cpp:420-425).
// Smaller kernels stay on the FP32 kernel of filter2d_tma.cu, which reproduces the reference's direct sum bit for bit.
//
// Arithmetic: 3 x BF16.  Every float is split into hi = bf16(a) and lo = bf16(a - hi) (|a - hi - lo| <= 2^-16 |a|; hi saturates to the
// largest finite BF16 instead of overflowing, see ff_split); the product sum is
//   sum a k  ~=  sum a_hi k_hi + sum a_hi k_lo + sum a_lo k_hi        (the dropped a_lo k_lo term is another 2^-16)
// in FP32 accumulators.  Relative to sum |a| |k| the error is <= ~4e-5 worst case (all signs aligned), ~1e-6 typical -- inside the
// reference's bar for this regime and below what its float DFT itself loses on 31 x 31 kernels.  BF16 keeps float's exponent range, so
// no data-dependent scaling (and no reduction pass over the image) is needed.  A NaN or inf PIXEL is not contained: every padded pixel of
// a tile's strip meets the Toeplitz zero taps too (inf x 0 = NaN), so it spreads to up to 32 + kw - 1 columns of its output rows (the
// reference's DFT spreads it over more).
//
// Contraction = the Toeplitz form of filter2d_tc.cu / matchtemplate_tc.cu:
//   D[m][j] = sum_v sum_k A_v[m][k] * B_v[k][j],   A_v[m][k] = P(y0 + m + v, x0 + k),   B_v[k][j] = K(v, k - j)   (0 outside 0 <= k-j < kw)
// with P the border-extended image.  Tile = 256 rows x 32 columns, K = kw + 31 rounded up to 16.
//
// Every MMA reads its whole A operand from shared memory whatever N is, so the A reads are amortised over N: per K step and 64-row
// slab TWO MMAs instead of three,
//     D[:, 0:64)  += A_hi x [B_hi | B_lo]      (N = 64: the hi and lo Toeplitz planes side by side in N)
//     E[:, 0:32)  += A_lo x  B_hi              (N = 32: the same operand, first half)
// and the epilogue adds D[:, j] + E[:, j] + D[:, 32 + j].
// The Toeplitz operands do not fit shared memory for 31 rows (8 KB per kernel row): they stream through a ring from L2.
//
// Roles (320 threads, one persistent CTA per SM):
//   warp 8      A producer: per tile the hi and lo strips (K columns x 256 + kh - 1 rows) by TMA in the K-major no-swizzle core-matrix
//               layout (one 16-byte-wide box column per 8 K elements), ring of 2 stages
//   warp 9      B producer: one kernel row of Toeplitz operands (8 KB) per cp.async.bulk into a ring of FF_NB = 7, in the order the
//               consumers use them
//   warps 0-7   two consumer warpgroups of 128 tile rows each: kh x K/16 x 2 slabs x 2 wgmma per tile; a kernel row's A operand is the
//               same strip with the descriptor start address advanced by one 16-byte row; a B stage is released (by both warpgroups) as
//               soon as the next kernel row's MMAs are in flight
// Order.  The accumulators live in registers, so a warpgroup's epilogue cannot overlap its own next MMAs; the other warpgroup has to keep
// the tensor pipe busy meanwhile.  Both warpgroups share each A strip and each streamed B kernel row, so B is read from L2 once per
// 256-row strip (about 30 B per output pixel at 31 x 31).  Giving each warpgroup its own 128-row tile would double that; starting
// warpgroup 1 half a tile late would need half a tile of B rows (about 128 KB) resident.  Instead warpgroup 1 starts every tile
// FF_LAG = 3 kernel rows behind warpgroup 0: warpgroup 0 arrives on lag_bar once it has issued those rows, and warpgroup 1 waits on
// it before its first MMA.  (An mbarrier rather than a named barrier: the arrive sits between wgmma groups in flight, where only a
// predicated mbarrier arrive leaves the MMAs unserialised.)  So warpgroup 0 reaches its epilogue 3 kernel rows (about 1.3 k cycles of
// MMAs at K = 64) before warpgroup 1 does, and warpgroup 1 stores while warpgroup 0 starts the next tile: at most one warpgroup is
// in its epilogue as long as the epilogue is shorter than that.  The ring holds the lag plus the 4 stages of before.  Measured on an
// H100 80GB HBM3 at a 400 W power limit (bench.py c2, 8 4K frames): 15 x 15 taps 0.78 ms, 21 x 21 1.13 ms, 31 x 31 1.52 ms, against
// 0.86 / 1.23 / 1.60 ms with both warpgroups in step and storing from registers.
// Epilogue.  Per 64-row slab the warpgroup writes its sums into a staging area in shared memory and stores whole 128-byte tile rows
// with 16-byte stores (element stores only at the right edge or for an unaligned destination).
// mbarriers: a_full/a_empty[2], b_full/b_empty[7], lag_bar[2] (by tile parity).  Named barriers 1, 2: the staging area of warpgroup
// 0, 1.
// The border-extended BF16 planes are written once per call by pad_split_kernel (reads 4 B, writes 4 B per pixel).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <cuda_bf16.h>
#include "common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace b200cv {

constexpr int FF_N = 32;                      // output columns per tile; the MMAs are N = 64 (hi | lo Toeplitz planes) and N = 32 (hi)
constexpr int FF_WG = 2;                      // consumer warpgroups, 128 tile rows each
constexpr int FF_THREADS = 128 * FF_WG + 64;  // consumer warpgroups, A producer warp, B producer warp
constexpr int FF_SMEM_MAX = 227 * 1024 - 1024;
constexpr int FF_NA = 2;                      // A stages
constexpr int FF_LAG = 3;                     // kernel rows warpgroup 1 starts each tile behind warpgroup 0
constexpr int FF_NB = FF_LAG + 4;             // B stages (kernel rows in flight)
constexpr int FF_SST = FF_N * 4 + 16;         // epilogue staging row pitch (16 B of padding: fewer bank conflicts)
constexpr int FF_STAGE = 64 * FF_SST;         // staging bytes per warpgroup (one 64-row slab)
constexpr int FF_BAR_EPI = 1;                 // named barriers 1, 2: the staging area of warpgroup 0, 1

struct FFTaps { float k[33 * 33]; };

struct FFParams {
    int kh, kch;                              // kernel rows; 16-byte K chunks per plane (K = 8 * kch, even)
    int ra_alloc, box_h, nbox;
    int ow, oh, frames, tiles_x, tiles_y, ntiles;
    int vec;                                  // destination rows and frames 16-byte aligned: whole-row 16-byte stores
    float delta;
};

// hi = bf16(a), lo = bf16(a - hi).  A finite |a| >= 3.3962e38 rounds to a BF16 infinity, which would make lo the opposite infinity and
// the sums NaN: hi then takes the largest finite BF16 of a's sign, so lo stays finite and |a - hi - lo| <= 2^-16 |a| still holds.
__device__ __forceinline__ void ff_split(float a, __nv_bfloat16& hi, __nv_bfloat16& lo)
{
    hi = __float2bfloat16_rn(a);
    if (isinf(__bfloat162float(hi)) && !isinf(a)) hi = __ushort_as_bfloat16(a < 0.f ? 0xFF7Fu : 0x7F7Fu);
    lo = __float2bfloat16_rn(a - __bfloat162float(hi));
}

// B in global/shared memory: [kernel row v][chunk c][column n (64: 0..31 hi plane, 32..63 lo plane)][8 bf16]: element e of column j = n & 31
// = plane(K(v, 8c + e - j)): K-major core matrices of 8 columns x 16 bytes, 128 bytes apart in N, 1024 bytes apart in K
__global__ void ff_toeplitz_kernel(const __grid_constant__ FFTaps kp, int kw, int kch, __nv_bfloat16* out)
{
    const int v = blockIdx.x;
    const int per_row = kch * 2 * FF_N * 8;
    for (int idx = threadIdx.x; idx < per_row; idx += blockDim.x) {
        const int e = idx & 7, n = (idx >> 3) % (2 * FF_N), c = (idx >> 3) / (2 * FF_N);
        const int pl = n / FF_N, j = n % FF_N;
        const int u = 8 * c + e - j;
        const float t = (u >= 0 && u < kw) ? kp.k[v * kw + u] : 0.f;
        __nv_bfloat16 hi, lo;
        ff_split(t, hi, lo);
        out[(size_t)v * per_row + idx] = pl ? lo : hi;
    }
}

// border-extended source as two BF16 planes: out[pl][f][y][x] = split(src(border(y - ay), border(x - ax))).  One thread = 8 adjacent
// elements of a row (pw is a multiple of 8): two 16-byte stores; the border rule per element only in the strips that leave the image
// (the first version wrote one element and two 2-byte stores per thread).
__global__ void __launch_bounds__(128) ff_pad_split_kernel(Img src, __nv_bfloat16* out, int pw, int ph, int ax, int ay, int border, size_t plane_elems)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8, y = blockIdx.y, f = blockIdx.z;
    if (x0 >= pw) return;
    const int sy = border_interpolate(y - ay, src.rows, border);
    float a[8];
    const int sx0 = x0 - ax;
    if (sy >= 0 && sx0 >= 0 && sx0 + 8 <= src.cols) {
        const float* sp = src.row<float>(f, sy) + sx0;
#pragma unroll
        for (int i = 0; i < 8; i++) a[i] = __ldg(sp + i);
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int sx = border_interpolate(sx0 + i, src.cols, border);
            a[i] = (sy < 0 || sx < 0) ? 0.f : src.row<float>(f, sy)[sx];        // BORDER_CONSTANT: zeros
        }
    }
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        __nv_bfloat16 h0, h1, l0, l1;
        ff_split(a[2 * i], h0, l0);
        ff_split(a[2 * i + 1], h1, l1);
        hi[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        lo[i] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
    const size_t o = ((size_t)f * ph + y) * pw + x0;
    *(uint4*)(out + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *(uint4*)(out + plane_elems + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

template <int KS>      // K / 16: MMA steps per kernel row
__global__ void __launch_bounds__(FF_THREADS, 1) filter2d_tc_f32_kernel(const __grid_constant__ CUtensorMap tmap, const unsigned char* __restrict__ bglob,
                                                                        Img dst, const __grid_constant__ FFParams p)
{
    extern __shared__ __align__(128) unsigned char smem[];
    constexpr int KCH = 2 * KS;
    constexpr uint32_t brow = (uint32_t)KCH * 2 * FF_N * 16;                 // bytes of B per kernel row (hi | lo side by side in N)
    const uint32_t lbo_a = (uint32_t)p.ra_alloc * 16u;                       // one 16-byte-wide column of the strip
    const uint32_t aplane = (uint32_t)KCH * lbo_a;
    const uint32_t abytes = 2 * aplane;                                      // one A stage (hi + lo)
    unsigned char* sB = smem;                                                // FF_NB stages of one kernel row
    unsigned char* sA = smem + (size_t)FF_NB * brow;                         // FF_NA stages
    unsigned char* sE = sA + (size_t)FF_NA * abytes;                         // epilogue staging, one slab per warpgroup
    __shared__ __align__(8) uint64_t b_full[FF_NB], b_empty[FF_NB], a_full[FF_NA], a_empty[FF_NA], lag_bar[2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < FF_NB; s++) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 4 * FF_WG); }
        for (int s = 0; s < FF_NA; s++) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 4 * FF_WG); }
        for (int s = 0; s < 2; s++) mbar_init(&lag_bar[s], 4);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 4 * FF_WG) {
        if (lane == 0) {
            // ---- A producer: the hi + lo strips of every tile ----
            int i = 0;
            for (int t = blockIdx.x; t < p.ntiles; t += gridDim.x, i++) {
                const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, f = t / (p.tiles_x * p.tiles_y);
                const int buf = i % FF_NA;
                mbar_wait(&a_empty[buf], ((i / FF_NA) & 1) ^ 1);
                mbar_arrive_expect_tx(&a_full[buf], abytes);
                unsigned char* dstA = sA + (size_t)buf * abytes;
                for (int pl = 0; pl < 2; pl++)
                    for (int c = 0; c < KCH; c++)
                        for (int b = 0; b < p.nbox; b++)
                            tma_load_3d(dstA + (size_t)pl * aplane + (size_t)c * lbo_a + (size_t)b * p.box_h * 16, &tmap, tx * FF_N + 8 * c,
                                        ty * (128 * FF_WG) + b * p.box_h, f + pl * p.frames, &a_full[buf]);
            }
        }
        return;
    }
    if (warp == 4 * FF_WG + 1) {
        if (lane == 0) {
            // ---- B producer: kernel row after kernel row, tile after tile, in the consumers' order ----
            int g = 0;
            for (int t = blockIdx.x; t < p.ntiles; t += gridDim.x)
                for (int v = 0; v < p.kh; v++, g++) {
                    const int s = g % FF_NB;
                    mbar_wait(&b_empty[s], ((g / FF_NB) & 1) ^ 1);
                    mbar_arrive_expect_tx(&b_full[s], brow);
                    wg_bulk_load(sB + (size_t)s * brow, bglob + (size_t)v * brow, brow, &b_full[s]);
                }
        }
        return;
    }

    // ---- consumers: warpgroup wg owns tile rows 128 wg .. 128 wg + 127 as two 64-row slabs ----
    const int wg = warp >> 2, wl = warp & 3, tid = threadIdx.x & 127;
    const int lag = min(FF_LAG, p.kh);
    unsigned char* st = sE + wg * FF_STAGE;
    const uint32_t b_base = smem_u32(sB);
    int i = 0, g = 0;
    for (int t = blockIdx.x; t < p.ntiles; t += gridDim.x, i++) {
        const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, f = t / (p.tiles_x * p.tiles_y);
        const int buf = i % FF_NA;
        float acc[2][FF_N], alo[2][FF_N / 2];        // A_hi x [B_hi | B_lo] (64 columns) and A_lo x B_hi (32 columns)
#pragma unroll
        for (int m = 0; m < 2; m++) {
#pragma unroll
            for (int r = 0; r < FF_N; r++) acc[m][r] = 0.f;
#pragma unroll
            for (int r = 0; r < FF_N / 2; r++) alo[m][r] = 0.f;
        }
        mbar_wait(&a_full[buf], (i / FF_NA) & 1);
        if (wg == 1) mbar_wait(&lag_bar[i & 1], (i >> 1) & 1);     // warpgroup 0 has issued the first `lag` kernel rows of this tile
        wg_fence();
        const uint32_t a0 = smem_u32(sA + (size_t)buf * abytes) + (uint32_t)(wg * 128) * 16u;
        int prev = -1;
#pragma unroll 1
        for (int v = 0; v < p.kh; v++, g++) {
            const int s = g % FF_NB;
            mbar_wait(&b_full[s], (g / FF_NB) & 1);
#pragma unroll
            for (int ks = 0; ks < KS; ks++) {
                const uint64_t bd = wg_desc(b_base + (uint32_t)s * brow + (uint32_t)ks * (2 * 2 * FF_N * 16), 2 * FF_N * 16, 128);
#pragma unroll
                for (int m = 0; m < 2; m++) {       // kernel row v: the same strip, v rows further down
                    const uint32_t a = a0 + (uint32_t)ks * 2u * lbo_a + (uint32_t)(m * 64 + v) * 16u;
                    wgmma_bf16_n64(acc[m], wg_desc(a, lbo_a, 128), bd);
                    wgmma_bf16_n32(alo[m], wg_desc(a + aplane, lbo_a, 128), bd);
                }
            }
            wg_commit();
            wg_mbar_arrive_if(&lag_bar[i & 1], wg == 0 && lane == 0 && v == lag - 1);
            wg_wait<1>();                            // the previous kernel row's MMAs are done: its B stage may be refilled
            wg_mbar_arrive_if(&b_empty[prev < 0 ? 0 : prev], lane == 0 && prev >= 0);
            prev = s;
        }
        wg_wait<0>();
        wg_fence_operand(acc[0]);
        wg_fence_operand(acc[1]);
        wg_fence_operand(alo[0]);
        wg_fence_operand(alo[1]);
        wg_mbar_arrive_if(&b_empty[prev], lane == 0);
        wg_mbar_arrive_if(&a_empty[buf], lane == 0);
        // ---- epilogue: hi x hi + lo x hi + hi x lo + delta, per 64-row slab through the staging area, whole 128-byte rows out ----
#pragma unroll
        for (int m = 0; m < 2; m++) {
            wg_bar_sync(FF_BAR_EPI + wg, 128);                 // the staging area's previous contents are stored
#pragma unroll
            for (int ii = 0; ii < 2; ii++) {
                const int row = wl * 16 + (lane >> 2) + 8 * ii;
#pragma unroll
                for (int j = 0; j < FF_N / 8; j++) {
                    float o[2];
#pragma unroll
                    for (int c = 0; c < 2; c++) {
                        const int r = 4 * j + 2 * ii + c;
                        o[c] = __fadd_rn(__fadd_rn(__fadd_rn(acc[m][r], alo[m][r]), acc[m][r + FF_N / 2]), p.delta);
                    }
                    *(float2*)(st + row * FF_SST + (8 * j + 2 * (lane & 3)) * 4) = make_float2(o[0], o[1]);
                }
            }
            wg_bar_sync(FF_BAR_EPI + wg, 128);
            for (int idx = tid; idx < 64 * (FF_N / 4); idx += 128) {
                const int row = idx / (FF_N / 4), c = idx % (FF_N / 4);
                const int gy = ty * (128 * FF_WG) + wg * 128 + m * 64 + row, gx = tx * FF_N + 4 * c;
                if (gy >= p.oh) continue;
                float* gp = dst.row<float>(f, gy) + gx;
                const float* sp = (const float*)(st + row * FF_SST) + 4 * c;
                if (p.vec && gx + 4 <= p.ow) *(float4*)gp = *(const float4*)sp;
                else
                    for (int e = 0; e < 4 && gx + e < p.ow; e++) gp[e] = sp[e];
            }
        }
    }
}

// filter2D, float single-channel source and destination.
// returns B200CV_NOT_IMPLEMENTED when the tensor-core path does not apply (the caller uses the direct-sum kernels)
int filter2d_f32_tensor(const Img& s, const Img& d, const float* k, int kw, int kh, int ax, int ay, float delta, int border, cudaStream_t st)
{
    if (kw > 33 || kh > 33 || s.frames >= 32768) return B200CV_NOT_IMPLEMENTED;
    // the cost grows with the kernel ROWS whatever the width: below 14 rows the direct FP32 sum is faster.  Measured on an H100 80GB HBM3
    // (700 W) with tools/f2d_rows_switch.py, 8 4K frames: 13 x 11 taps 0.73 ms direct / 0.87 ms here, 15 x 9 taps 1.11 / 1.03 ms.
    if (kh < 14 && !getenv("B200CV_FILTER2D_TC_MIN_TAPS")) return B200CV_NOT_IMPLEMENTED;
    static thread_local FFTaps taps;
    for (int i = 0; i < kw * kh; i++) {
        if (!std::isfinite(k[i])) return B200CV_NOT_IMPLEMENTED;
        taps.k[i] = k[i];
    }
    FFParams p;
    memset(&p, 0, sizeof(p));
    p.kh = kh; p.ow = s.cols; p.oh = s.rows; p.frames = s.frames; p.delta = delta;
    p.kch = 2 * (int)div_up((unsigned)(kw + FF_N - 1), 16);                 // K = kw + 31 rounded up to a multiple of 16 elements
    p.tiles_x = (int)div_up((unsigned)p.ow, FF_N); p.tiles_y = (int)div_up((unsigned)p.oh, 128 * FF_WG);
    const long long nt = (long long)p.tiles_x * p.tiles_y * p.frames;
    if (nt > 0x7fffffff) return B200CV_NOT_IMPLEMENTED;
    p.ntiles = (int)nt;
    const int ra = 128 * FF_WG + kh - 1;
    p.nbox = (ra + 255) / 256;
    p.box_h = (((ra + p.nbox - 1) / p.nbox) + 7) & ~7;
    p.ra_alloc = p.nbox * p.box_h;
    const size_t brow = (size_t)p.kch * 2 * FF_N * 16, abytes = (size_t)2 * p.kch * p.ra_alloc * 16;
    const size_t smem = (size_t)FF_NB * brow + FF_NA * abytes + FF_WG * FF_STAGE;
    if (smem > (size_t)FF_SMEM_MAX) return B200CV_NOT_IMPLEMENTED;
    p.vec = (((uintptr_t)d.data | d.step | d.fstep) & 15) == 0;
    const int grid = (int)std::min<long long>(nt, num_sms());

    // border-extended source as BF16 hi / lo planes, rows padded to a multiple of 8 elements (16 bytes: TMA)
    const int pw = (s.cols + kw - 1 + 7) & ~7, ph = s.rows + kh - 1;
    const size_t plane_elems = (size_t)pw * ph * s.frames;
    __nv_bfloat16* pbuf = nullptr; unsigned char* bglob = nullptr;
    B200_CUDA(cudaMallocAsync(&pbuf, plane_elems * 2 * sizeof(__nv_bfloat16), st));
    B200_CUDA(cudaMallocAsync(&bglob, (size_t)kh * brow, st));
    ff_toeplitz_kernel<<<kh, 256, 0, st>>>(taps, kw, p.kch, (__nv_bfloat16*)bglob);
    count_launch();
    ff_pad_split_kernel<<<dim3(div_up((unsigned)pw / 8, 128), (unsigned)ph, (unsigned)s.frames), 128, 0, st>>>(s, pbuf, pw, ph, ax, ay, border, plane_elems);
    count_launch();
    CUtensorMap tm;
    int rc = make_tensor_map_3d(&tm, pbuf, 2, pw, ph, 2 * s.frames, (size_t)pw * 2, (size_t)pw * ph * 2, 8, p.box_h);
    if (!rc) {
        static PerDeviceFlag attr_pd; bool& attr = attr_pd.cur();
        if (!attr) {
            B200_CUDA(cudaFuncSetAttribute(filter2d_tc_f32_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, FF_SMEM_MAX));
            B200_CUDA(cudaFuncSetAttribute(filter2d_tc_f32_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, FF_SMEM_MAX));
            B200_CUDA(cudaFuncSetAttribute(filter2d_tc_f32_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, FF_SMEM_MAX));
            attr = true;
        }
        if (p.kch == 4) filter2d_tc_f32_kernel<2><<<grid, FF_THREADS, smem, st>>>(tm, bglob, d, p);          // kw = 1
        else if (p.kch == 6) filter2d_tc_f32_kernel<3><<<grid, FF_THREADS, smem, st>>>(tm, bglob, d, p);     // kw <= 17
        else filter2d_tc_f32_kernel<4><<<grid, FF_THREADS, smem, st>>>(tm, bglob, d, p);                     // kw <= 33
        cudaError_t e = cudaGetLastError();
        count_launch();
        if (e != cudaSuccess) rc = cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    }
    cudaFreeAsync(bglob, st);
    cudaFreeAsync(pbuf, st);
    return rc;
}

}  // namespace b200cv
