// filter2d_tc.cu -- 8-bit single-channel cv::filter2D with >= 11x11 taps on Hopper tensor cores: a persistent, warp-specialised
// wgmma kernel.  (These are the sizes at which the reference itself leaves the direct sum for a DFT,
// filter.dispatch.cpp:1288-1310; smaller kernels stay on the FP32 kernel of filter2d_tma.cu.)
//
// Arithmetic.  The float taps are quantised to 24-bit fixed point against max|k| (Kq = rint(k 2^sh), |Kq| < 2^22) and split into
// three balanced base-256 digits d0, d1, d2 in [-128, 127].  With the Toeplitz expansion of matchtemplate_tc.cu,
//   D_d[m][j] = sum_v sum_k A_v[m][k] * B_{v,d}[k][j],   A_v[m][k] = P(y0+m+v, x0+k),   B_{v,d}[k][j] = d(Kq(v, k-j)),
// one integer MMA (u8 x s8 -> s32, exact) carries the three digit planes of an NT-column output tile as N = 3 x NT; the epilogue
// recombines S0 + 256 S1 + 65536 S2 in 64-bit, converts once, scales by 2^-sh and adds delta.  The only error is the tap quantisation
// (<= 2^-23 max|k| per tap): the same order as a float accumulation, far inside the reference's own tolerance for this path (its
// DFT).  P is the border-extended image (pad_u8_kernel).
//
// Tile width.  A kernel row of K = NT + kw - 1 Toeplitz columns is consumed in K32 steps, and every wgmma reads both operands from
// shared memory (128 B/clk per SM), which bounds these MMAs.  kw <= 17 uses NT = 16: one K32 step of m64n48k32 (3.5 KB of operands)
// per 64 x 16 slab.  Wider kernels use NT = 32: two K32 steps of m64n96k32 (2 x 5 KB) per 64 x 32 slab, K = 64 covering kw <= 33.
// Per output pixel the narrow tile reads about 1.7x fewer operand bytes; the integer sums are the same.  Measured on an H100 80GB HBM3
// at a 400 W power limit (bench.py c2, 16 4K frames, kernel + pad + Toeplitz): 13 x 13 taps 0.65 ms, 15 x 15 0.68 ms, 21 x 21 0.92 ms,
// 31 x 31 1.17 ms, against 0.87 / 0.94 / 1.08 / 1.45 ms for 32-column 256-row tiles with both warpgroups storing at the same time.
//
// Data movement.  A kernel row's operand B_v is (K / 16) x 3 NT x 16 B (1.5 KB at NT = 16, 6 KB at NT = 32), so ALL of B stays
// RESIDENT in shared memory for the life of the CTA.  One CTA per SM walks destination tiles of 128 rows x NT columns:
//   warp 8     producer  -- all of B once, then per tile one TMA load of the (K bytes)-wide A strip (128 + kh - 1 rows) into a ring of
//                           2-4 buffers, in tile order
//   warps 0-7  consumers -- two warpgroups; the CTA's tiles alternate between them (local tile i goes to warpgroup i & 1), and each
//                           computes its own tile: kh x K/32 K-steps x 2 slabs of wgmma into registers, then the epilogue.
// Order ("ping-pong").  The accumulators live in registers, so a warpgroup cannot store one tile while its next tile's MMAs run.  The
// two warpgroups therefore take turns issuing: a warpgroup waits on named barrier 1 + (i & 1) for its turn, issues all MMAs of tile i,
// hands the turn to the other warpgroup (bar.arrive on 1 + ((i + 1) & 1)), and only then waits for its MMAs and runs its epilogue --
// while the other warpgroup's MMAs keep the tensor pipe busy.  At most one warpgroup is in its epilogue at a time as long as the
// epilogue is shorter than a tile's MMAs.  Giving each warpgroup its own 128-row tile (rather than two halves of a 256-row strip, one
// started half a tile late) keeps each A stage owned by one warpgroup, and wastes fewer rows at the bottom edge: 2160 rows are 17
// tiles of 128 (2176 rows computed) against 9 of 256 (2304).  The larger halo per strip (kh - 1 rows per 128 instead of per 256)
// costs only TMA traffic into shared memory, not MMAs.
// Epilogue.  Per 64-row slab the warpgroup writes its values into a staging area in shared memory, then stores whole rows to global
// memory with 16-byte stores (NT x element bytes per row), element stores only at the right edge or for an unaligned destination.
// mbarriers: b_full, a_full/a_empty[4] (a stage is released by the four warps of the warpgroup that read it).  Named barriers: 1, 2
// the MMA turn; 3, 4 the staging area of warpgroup 0, 1.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <type_traits>
#include "common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace b200cv {

void launch_pad_u8(const Img& src, const Img& dst, int ax, int ay, int border, cudaStream_t st);     // matchtemplate_tc.cu

constexpr int FC_WG = 2;                      // consumer warpgroups, one 128-row tile each
constexpr int FC_TH = 128;                    // tile rows
constexpr int FC_THREADS = 128 * FC_WG + 32;  // consumer warpgroups + one producer warp
constexpr int FC_SMEM_MAX = 227 * 1024 - 512;   // opt-in limit per CTA (232448 B) minus this kernel's static shared memory (barriers)
constexpr int FC_BAR_MMA = 1, FC_BAR_EPI = 3; // named barriers (see the header)

// geometry of one tile width: NT output columns, MMA N = 3 NT (three digit planes), K = 32 (NT = 16) or 64 (NT = 32) per kernel row
template <int NT> struct FCTile {
    static constexpr int N = 3 * NT;
    static constexpr int K = NT == 16 ? 32 : 64;
    static constexpr int BROW = (K / 16) * N * 16;         // bytes of B per kernel row: 1536 / 6144
    static constexpr int SST = NT * 4 + 16;                // staging row pitch, sized for float output (16 B of padding: fewer bank conflicts)
    static constexpr int STAGE = 64 * SST;                 // staging bytes per warpgroup (one 64-row slab)
};

struct FCKq { int q[33 * 33]; };

struct FCParams {
    int kh, ra_alloc, box_h, nbox;
    int ow, oh, frames, tiles_x, tiles_y, ntiles;
    int na;                                   // A strip buffers (2..4): as many as fit next to the resident B
    int vec;                                  // destination rows and frames 16-byte aligned: whole-row 16-byte stores
    float scale, delta;
};

// B in global/shared memory: [kernel row v][k-chunk c (K / 16)][column j (3 NT) = digit d * NT + jj][16 bytes]:
// byte b = digit_d(Kq(v, 16c + b - jj))
template <int NT>
__global__ void fc_toeplitz_kernel(const __grid_constant__ FCKq kp, int w, signed char* out)
{
    using T = FCTile<NT>;
    const int v = blockIdx.x;
    for (int idx = threadIdx.x; idx < T::BROW; idx += blockDim.x) {
        const int b = idx & 15, j = (idx >> 4) % T::N, c = (idx >> 4) / T::N;
        const int d = j / NT, jj = j - d * NT;
        const int u = 16 * c + b - jj;
        int q = (u >= 0 && u < w) ? kp.q[v * w + u] : 0;
        const int d0 = ((q + 128) & 255) - 128; q = (q - d0) >> 8;      // balanced base-256 digits
        const int d1 = ((q + 128) & 255) - 128; q = (q - d1) >> 8;
        out[(size_t)v * T::BROW + idx] = (signed char)(d == 0 ? d0 : d == 1 ? d1 : q);
    }
}

enum { FC_U8 = 0, FC_F32 = 1, FC_S16 = 2 };

template <int NT>
__device__ __forceinline__ void fc_mma(uint32_t (&d)[3 * NT / 2], uint64_t adesc, uint64_t bdesc)
{
    if constexpr (NT == 16) wgmma_u8s8_n48(d, adesc, bdesc);
    else wgmma_u8s8_n96(d, adesc, bdesc);
}

template <int EPI, int NT>
__global__ void __launch_bounds__(FC_THREADS, 1) filter2d_tc_kernel(const __grid_constant__ CUtensorMap tmap, const unsigned char* __restrict__ bglob,
                                                                    Img dst, const __grid_constant__ FCParams p)
{
    using T = FCTile<NT>;
    using OutT = typename std::conditional<EPI == FC_U8, uchar, typename std::conditional<EPI == FC_S16, short, float>::type>::type;
    constexpr int ES = (int)sizeof(OutT);
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t abytes = (uint32_t)(T::K / 16) * p.ra_alloc * 16;        // one A buffer
    unsigned char* sB = smem;                                               // kh x BROW, resident
    unsigned char* sE = smem + (size_t)p.kh * T::BROW;                      // staging, one slab per warpgroup
    unsigned char* sA = sE + FC_WG * T::STAGE;                              // p.na buffers
    __shared__ __align__(8) uint64_t b_full, a_full[4], a_empty[4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t lbo_a = (uint32_t)p.ra_alloc * 16u;

    if (threadIdx.x == 0) {
        mbar_init(&b_full, 1);
        for (int s = 0; s < 4; s++) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 4); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 4 * FC_WG) {
        if (lane == 0) {
            // ---- producer: all of B once, then one A strip per tile, in tile order ----
            mbar_arrive_expect_tx(&b_full, (uint32_t)p.kh * T::BROW);
            for (int v = 0; v < p.kh; v++) wg_bulk_load(sB + (size_t)v * T::BROW, bglob + (size_t)v * T::BROW, T::BROW, &b_full);
            int i = 0;
            for (int t = blockIdx.x; t < p.ntiles; t += gridDim.x, i++) {
                const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, f = t / (p.tiles_x * p.tiles_y);
                const int buf = i % p.na;
                mbar_wait(&a_empty[buf], ((i / p.na) & 1) ^ 1);
                mbar_arrive_expect_tx(&a_full[buf], abytes);
                unsigned char* dstA = sA + (size_t)buf * abytes;
                for (int c = 0; c < T::K / 16; c++)
                    for (int b = 0; b < p.nbox; b++)
                        tma_load_3d(dstA + (size_t)c * lbo_a + (size_t)b * p.box_h * 16, &tmap, tx * NT + 16 * c, ty * FC_TH + b * p.box_h, f, &a_full[buf]);
            }
        }
        return;
    }

    // ---- consumers: warpgroup wg computes the CTA's local tiles wg, wg + 2, ...: rows ty * 128 .. + 127 as two 64-row slabs ----
    const int wg = warp >> 2, wl = warp & 3, tid = threadIdx.x & 127;
    unsigned char* st = sE + wg * T::STAGE;
    mbar_wait(&b_full, 0);
    const uint32_t b0 = smem_u32(sB);
    int i = wg;
    for (int t = blockIdx.x + wg * gridDim.x; t < p.ntiles; t += FC_WG * gridDim.x, i += FC_WG) {
        const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, f = t / (p.tiles_x * p.tiles_y);
        const int buf = i % p.na;
        uint32_t acc[2][T::N / 2];
#pragma unroll
        for (int m = 0; m < 2; m++)
#pragma unroll
            for (int r = 0; r < T::N / 2; r++) acc[m][r] = 0;
        mbar_wait(&a_full[buf], (i / p.na) & 1);
        wg_bar_sync_if(FC_BAR_MMA + (i & 1), 256, i > 0);             // our turn: the other warpgroup has issued tile i - 1
        wg_fence();
        const uint32_t a0 = smem_u32(sA + (size_t)buf * abytes);
#pragma unroll 1
        for (int v = 0; v < p.kh; v++) {
#pragma unroll
            for (int ks = 0; ks < T::K / 32; ks++) {
                const uint64_t bd = wg_desc(b0 + (uint32_t)v * T::BROW + (uint32_t)ks * (2 * T::N * 16), T::N * 16, 128);
#pragma unroll
                for (int m = 0; m < 2; m++)    // kernel row v: the same strip, v rows further down
                    fc_mma<NT>(acc[m], wg_desc(a0 + (uint32_t)ks * 2u * lbo_a + (uint32_t)(m * 64 + v) * 16u, lbo_a, 128), bd);
            }
        }
        wg_commit();
        wg_bar_arrive(FC_BAR_MMA + ((i + 1) & 1), 256);     // the other warpgroup's turn (tile i + 1; after the last tile see below)
        wg_wait<0>();
        wg_fence_operand(acc[0]);
        wg_fence_operand(acc[1]);
        wg_mbar_arrive_if(&a_empty[buf], lane == 0);          // 4 arrivals (one per warp of this warpgroup) free the strip
        // ---- epilogue: column jj of the tile has its digit sums at N = jj, NT + jj, 2 NT + jj ----
#pragma unroll
        for (int m = 0; m < 2; m++) {
            wg_bar_sync(FC_BAR_EPI + wg, 128);                 // the staging area's previous contents are stored
#pragma unroll
            for (int ii = 0; ii < 2; ii++) {
                const int row = wl * 16 + (lane >> 2) + 8 * ii;
#pragma unroll
                for (int j = 0; j < NT / 8; j++) {
                    OutT o[2];
#pragma unroll
                    for (int c = 0; c < 2; c++) {
                        const int r = 4 * j + 2 * ii + c;
                        const long long sum = (long long)(int)acc[m][r] + ((long long)(int)acc[m][r + NT / 2] << 8) +
                                              ((long long)(int)acc[m][r + NT] << 16);
                        const float v = __fadd_rn(__fmul_rn(__ll2float_rn(sum), p.scale), p.delta);
                        if constexpr (EPI == FC_U8) o[c] = sat_u8(v);
                        else if constexpr (EPI == FC_S16) o[c] = sat_s16(v);
                        else o[c] = v;
                    }
                    unsigned char* sp = st + row * T::SST + (8 * j + 2 * (lane & 3)) * ES;      // the pair as one 2-, 4- or 8-byte store
                    if constexpr (ES == 1) *(unsigned short*)sp = (unsigned short)(o[0] | (o[1] << 8));
                    else if constexpr (ES == 2) *(uint32_t*)sp = (uint32_t)(unsigned short)o[0] | ((uint32_t)(unsigned short)o[1] << 16);
                    else *(float2*)sp = make_float2(o[0], o[1]);
                }
            }
            wg_bar_sync(FC_BAR_EPI + wg, 128);
            constexpr int CH = NT * ES / 16;                   // 16-byte chunks per tile row
            for (int idx = tid; idx < 64 * CH; idx += 128) {
                const int row = idx / CH, c = idx % CH;
                const int gy = ty * FC_TH + m * 64 + row, gx = tx * NT + c * (16 / ES);
                if (gy >= p.oh) continue;
                OutT* gp = dst.row<OutT>(f, gy) + gx;
                const unsigned char* sp = st + row * T::SST + c * 16;
                if (p.vec && gx + 16 / ES <= p.ow) {
                    *(uint4*)gp = *(const uint4*)sp;
                } else {
                    for (int e = 0; e < 16 / ES && gx + e < p.ow; e++) gp[e] = ((const OutT*)sp)[e];
                }
            }
        }
    }
    // The hand-over after the CTA's last tile n - 1 is unconditional (a predicated bar.arrive between wgmma groups in flight makes
    // ptxas serialise the MMAs), so the warpgroup that would own tile n takes it here: no barrier is left half-arrived at exit.
    if (i > 0 && blockIdx.x + (i - 1) * gridDim.x < p.ntiles) wg_bar_sync(FC_BAR_MMA + (i & 1), 256);
}

template <int EPI, int NT>
static int launch_fc(const CUtensorMap& tm, const unsigned char* bglob, const Img& d, const FCParams& p, size_t smem, int grid, cudaStream_t st)
{
    auto kern = filter2d_tc_kernel<EPI, NT>;
    static PerDeviceFlag attr_pd; bool& attr = attr_pd.cur();
    if (!attr) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FC_SMEM_MAX)); attr = true; }
    kern<<<grid, FC_THREADS, smem, st>>>(tm, bglob, d, p);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

template <int NT>
static int filter2d_u8_tensor_nt(const Img& s, const Img& d, int dd, const FCKq& kq, int kw, int kh, int ax, int ay, int border, FCParams p,
                                 cudaStream_t st)
{
    using T = FCTile<NT>;
    p.tiles_x = (int)div_up((unsigned)p.ow, NT); p.tiles_y = (int)div_up((unsigned)p.oh, FC_TH);
    const long long nt = (long long)p.tiles_x * p.tiles_y * p.frames;
    if (nt > 0x7fffffff) return B200CV_NOT_IMPLEMENTED;
    p.ntiles = (int)nt;
    const int ra = FC_TH + kh - 1;
    p.nbox = (ra + 255) / 256;
    p.box_h = (((ra + p.nbox - 1) / p.nbox) + 7) & ~7;
    p.ra_alloc = p.nbox * p.box_h;
    const size_t abytes = (size_t)(T::K / 16) * p.ra_alloc * 16;
    const size_t fixed = (size_t)kh * T::BROW + FC_WG * T::STAGE;
    if (fixed + 2 * abytes > (size_t)FC_SMEM_MAX) return B200CV_NOT_IMPLEMENTED;
    p.na = (int)std::min<size_t>(4, ((size_t)FC_SMEM_MAX - fixed) / abytes);
    const size_t smem = fixed + p.na * abytes;
    const int grid = (int)std::min<long long>(nt, num_sms());
    p.vec = (((uintptr_t)d.data | d.step | d.fstep) & 15) == 0;

    // border-extended source, rows padded to a multiple of 16 bytes (TMA)
    Img pad = s;
    pad.cols = (s.cols + kw - 1 + 15) & ~15;
    pad.rows = s.rows + kh - 1;
    pad.step = (size_t)pad.cols;
    pad.fstep = pad.step * pad.rows;
    unsigned char* pbuf = nullptr; unsigned char* bglob = nullptr;
    B200_CUDA(cudaMallocAsync(&pbuf, pad.fstep * (size_t)s.frames, st));
    B200_CUDA(cudaMallocAsync(&bglob, (size_t)kh * T::BROW, st));
    pad.data = pbuf;
    fc_toeplitz_kernel<NT><<<kh, 256, 0, st>>>(kq, kw, (signed char*)bglob);
    count_launch();
    launch_pad_u8(s, pad, ax, ay, border, st);
    CUtensorMap tm;
    int rc = make_tensor_map_3d(&tm, pad.data, 1, pad.cols, pad.rows, pad.frames, pad.step, pad.fstep, 16, p.box_h);
    if (!rc) {
        rc = dd == B200CV_8U ? launch_fc<FC_U8, NT>(tm, bglob, d, p, smem, grid, st)
           : dd == B200CV_16S ? launch_fc<FC_S16, NT>(tm, bglob, d, p, smem, grid, st)
                              : launch_fc<FC_F32, NT>(tm, bglob, d, p, smem, grid, st);
    }
    cudaFreeAsync(bglob, st);
    cudaFreeAsync(pbuf, st);
    return rc;
}

// filter2D, 8-bit single-channel source.  dd = destination depth.
// returns B200CV_NOT_IMPLEMENTED when the tensor-core path does not apply (caller uses the direct-sum kernel)
int filter2d_u8_tensor(const Img& s, const Img& d, int dd, const float* k, int kw, int kh, int ax, int ay, float delta, int border, cudaStream_t st)
{
    // kh <= 31: the largest kernel whose resident B leaves room for two A strips at NT = 32 (and the bound for either width, so that
    // which calls take this path does not depend on the tile width)
    if (kw > 33 || kh > 31 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    if (dd != B200CV_8U && dd != B200CV_32F && dd != B200CV_16S) return B200CV_NOT_IMPLEMENTED;
    float mx = 0.f;
    for (int i = 0; i < kw * kh; i++) {
        if (!std::isfinite(k[i])) return B200CV_NOT_IMPLEMENTED;
        mx = std::max(mx, std::fabs(k[i]));
    }
    if (!(mx > 0.f) || mx > 1e30f || mx < 1e-30f) return B200CV_NOT_IMPLEMENTED;
    int e;
    std::frexp((double)mx, &e);                       // mx = m * 2^e, m in [0.5, 1)
    const int sh = 22 - e;                            // |k| * 2^sh < 2^22: the three balanced digits stay inside [-128, 127]
    static thread_local FCKq kq;
    for (int i = 0; i < kw * kh; i++) kq.q[i] = (int)std::lrint(std::ldexp((double)k[i], sh));

    FCParams p;
    memset(&p, 0, sizeof(p));
    p.kh = kh; p.ow = s.cols; p.oh = s.rows; p.frames = s.frames; p.scale = (float)std::ldexp(1.0, -sh); p.delta = delta;
    return kw <= 17 ? filter2d_u8_tensor_nt<16>(s, d, dd, kq, kw, kh, ax, ay, border, p, st)
                    : filter2d_u8_tensor_nt<32>(s, d, dd, kq, kw, kh, ax, ay, border, p, st);
}

}  // namespace b200cv
