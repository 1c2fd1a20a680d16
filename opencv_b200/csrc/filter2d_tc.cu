// filter2d_tc.cu -- 8-bit single-channel cv::filter2D with >= 11x11 taps on Hopper tensor cores: a persistent, warp-specialised
// wgmma kernel.  (These are the sizes at which the reference itself leaves the direct sum for a DFT,
// filter.dispatch.cpp:1288-1310; smaller kernels stay on the FP32 kernel of filter2d_tma.cu.)
//
// Arithmetic.  The float taps are quantised to 24-bit fixed point against max|k| (Kq = rint(k 2^sh), |Kq| < 2^22) and split into
// three balanced base-256 digits d0, d1, d2 in [-128, 127].  With the Toeplitz expansion of matchtemplate_tc.cu,
//   D_d[m][j] = sum_v sum_k A_v[m][k] * B_{v,d}[k][j],   A_v[m][k] = P(y0+m+v, x0+k),   B_{v,d}[k][j] = d(Kq(v, k-j)),
// one integer MMA (u8 x s8 -> s32, exact) of shape M64 x N96 x K32 carries the three digit planes of a 32-column output tile
// as N = 3 x 32; the epilogue recombines S0 + 256 S1 + 65536 S2 in 64-bit, converts once, scales by 2^-sh and adds delta.  The only
// error is the tap quantisation (<= 2^-23 max|k| per tap): the same order as a float accumulation, far inside the reference's own
// tolerance for this path (its DFT).  P is the border-extended image (pad_u8_kernel).
//
// Data movement.  K = 64 per kernel row covers kw <= 33 (kw + 31 <= 64): a kernel row's operand B_v is 4 x 96 x 16 B = 6 KB, so
// ALL of B (31 rows = 186 KB) stays RESIDENT in shared memory for the life of the CTA.  One CTA per SM walks destination tiles of
// 256 rows x 32 columns:
//   warp 8     producer  -- all of B once, then per tile one TMA load of the 64-byte-wide A strip (256 + kh - 1 rows, 18 KB) into a
//                           ring of 2-4 buffers
//   warps 0-7  consumers -- two warpgroups of 128 tile rows each: kh x 2 K-steps x 2 slabs of wgmma m64n96k32 per tile into
//                           registers, then recombination and stores from the registers; the strip is released before the epilogue,
//                           so the producer refills it while the warpgroups store
// mbarriers: b_full, a_full/a_empty[4].
#include <algorithm>
#include <cmath>
#include <cstring>
#include "common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace b200cv {

void launch_pad_u8(const Img& src, const Img& dst, int ax, int ay, int border, cudaStream_t st);     // matchtemplate_tc.cu

constexpr int FC_NT = 32;                     // output columns per tile
constexpr int FC_N = 3 * FC_NT;               // MMA N (three digit planes)
constexpr int FC_K = 64;                      // K per kernel row
constexpr int FC_WG = 2;                      // consumer warpgroups, 128 tile rows each
constexpr int FC_BROW = (FC_K / 16) * FC_N * 16;   // bytes of B per kernel row = 6144
constexpr int FC_THREADS = 128 * FC_WG + 32;  // consumer warpgroups + one producer warp
constexpr int FC_SMEM_MAX = 227 * 1024 - 512;   // opt-in limit per CTA (232448 B) minus this kernel's static shared memory (barriers)

struct FCKq { int q[33 * 33]; };

struct FCParams {
    int kh, ra_alloc, box_h, nbox;
    int ow, oh, frames, tiles_x, tiles_y, ntiles;
    int na;                                   // A strip buffers (2..4): as many as fit next to the resident B
    float scale, delta;
};

// B in global/shared memory: [kernel row v][k-chunk c (4)][column j (96) = digit d * 32 + jj][16 bytes]: byte b = digit_d(Kq(v, 16c + b - jj))
__global__ void fc_toeplitz_kernel(const __grid_constant__ FCKq kp, int w, signed char* out)
{
    const int v = blockIdx.x;
    for (int idx = threadIdx.x; idx < FC_BROW; idx += blockDim.x) {
        const int b = idx & 15, j = (idx >> 4) % FC_N, c = (idx >> 4) / FC_N;
        const int d = j / FC_NT, jj = j - d * FC_NT;
        const int u = 16 * c + b - jj;
        int q = (u >= 0 && u < w) ? kp.q[v * w + u] : 0;
        const int d0 = ((q + 128) & 255) - 128; q = (q - d0) >> 8;      // balanced base-256 digits
        const int d1 = ((q + 128) & 255) - 128; q = (q - d1) >> 8;
        out[(size_t)v * FC_BROW + idx] = (signed char)(d == 0 ? d0 : d == 1 ? d1 : q);
    }
}

enum { FC_U8 = 0, FC_F32 = 1, FC_S16 = 2 };

template <int EPI>
__global__ void __launch_bounds__(FC_THREADS, 1) filter2d_tc_kernel(const __grid_constant__ CUtensorMap tmap, const unsigned char* __restrict__ bglob,
                                                                    Img dst, const __grid_constant__ FCParams p)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t abytes = (uint32_t)(FC_K / 16) * p.ra_alloc * 16;        // one A buffer
    unsigned char* sB = smem;                                               // kh x 6 KB, resident
    unsigned char* sA = smem + (size_t)p.kh * FC_BROW;                      // p.na buffers
    __shared__ __align__(8) uint64_t b_full, a_full[4], a_empty[4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t lbo_a = (uint32_t)p.ra_alloc * 16u;

    if (threadIdx.x == 0) {
        mbar_init(&b_full, 1);
        for (int s = 0; s < 4; s++) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 4 * FC_WG); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 4 * FC_WG) {
        if (lane == 0) {
            // ---- producer: all of B once, then one A strip per tile ----
            mbar_arrive_expect_tx(&b_full, (uint32_t)p.kh * FC_BROW);
            for (int v = 0; v < p.kh; v++) wg_bulk_load(sB + (size_t)v * FC_BROW, bglob + (size_t)v * FC_BROW, FC_BROW, &b_full);
            int i = 0;
            for (int t = blockIdx.x; t < p.ntiles; t += gridDim.x, i++) {
                const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, f = t / (p.tiles_x * p.tiles_y);
                const int buf = i % p.na;
                mbar_wait(&a_empty[buf], ((i / p.na) & 1) ^ 1);
                mbar_arrive_expect_tx(&a_full[buf], abytes);
                unsigned char* dstA = sA + (size_t)buf * abytes;
                for (int c = 0; c < FC_K / 16; c++)
                    for (int b = 0; b < p.nbox; b++)
                        tma_load_3d(dstA + (size_t)c * lbo_a + (size_t)b * p.box_h * 16, &tmap, tx * FC_NT + 16 * c, ty * (128 * FC_WG) + b * p.box_h, f, &a_full[buf]);
            }
        }
        return;
    }

    // ---- consumers: warpgroup wg owns tile rows 128 wg .. 128 wg + 127 as two 64-row slabs; per tile kh x 2 K-steps x 2 slabs of
    //      wgmma m64n96k32, then the epilogue from the registers while the other warpgroup / the next strip keep the pipe busy ----
    const int wg = warp >> 2, wl = warp & 3;
    mbar_wait(&b_full, 0);
    const uint32_t b0 = smem_u32(sB);
    int i = 0;
    for (int t = blockIdx.x; t < p.ntiles; t += gridDim.x, i++) {
        const int tx = t % p.tiles_x, ty = (t / p.tiles_x) % p.tiles_y, f = t / (p.tiles_x * p.tiles_y);
        const int buf = i % p.na;
        uint32_t acc[2][FC_N / 2];
#pragma unroll
        for (int m = 0; m < 2; m++)
#pragma unroll
            for (int r = 0; r < FC_N / 2; r++) acc[m][r] = 0;
        mbar_wait(&a_full[buf], (i / p.na) & 1);
        wg_fence();
        const uint32_t a0 = smem_u32(sA + (size_t)buf * abytes) + (uint32_t)(wg * 128) * 16u;
#pragma unroll 1
        for (int v = 0; v < p.kh; v++) {
#pragma unroll
            for (int ks = 0; ks < FC_K / 32; ks++) {
                const uint64_t bd = wg_desc(b0 + (uint32_t)v * FC_BROW + (uint32_t)ks * (2 * FC_N * 16), FC_N * 16, 128);
#pragma unroll
                for (int m = 0; m < 2; m++)    // kernel row v: the same strip, v rows further down
                    wgmma_u8s8_n96(acc[m], wg_desc(a0 + (uint32_t)ks * 2u * lbo_a + (uint32_t)(m * 64 + v) * 16u, lbo_a, 128), bd);
            }
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_operand(acc[0]);
        wg_fence_operand(acc[1]);
        wg_mbar_arrive_if(&a_empty[buf], lane == 0);          // 8 arrivals (one per consumer warp) free the strip
        // ---- epilogue: column jj of the tile has its digit sums at N = jj, 32 + jj, 64 + jj ----
#pragma unroll
        for (int m = 0; m < 2; m++)
#pragma unroll
            for (int ii = 0; ii < 2; ii++) {
                const int gy = ty * (128 * FC_WG) + wg * 128 + m * 64 + wl * 16 + (lane >> 2) + 8 * ii;
                if (gy >= p.oh) continue;
#pragma unroll
                for (int j = 0; j < FC_NT / 8; j++) {
                    const int gx = tx * FC_NT + 8 * j + 2 * (lane & 3);
                    float v[2];
#pragma unroll
                    for (int c = 0; c < 2; c++) {
                        const int r = 4 * j + 2 * ii + c;
                        const long long sum = (long long)(int)acc[m][r] + ((long long)(int)acc[m][r + FC_NT / 2] << 8) +
                                              ((long long)(int)acc[m][r + FC_NT] << 16);
                        v[c] = __fadd_rn(__fmul_rn(__ll2float_rn(sum), p.scale), p.delta);
                    }
#pragma unroll
                    for (int c = 0; c < 2; c++) {
                        if (gx + c >= p.ow) continue;
                        if constexpr (EPI == FC_U8) dst.row<uchar>(f, gy)[gx + c] = sat_u8(v[c]);
                        else if constexpr (EPI == FC_S16) dst.row<short>(f, gy)[gx + c] = sat_s16(v[c]);
                        else dst.row<float>(f, gy)[gx + c] = v[c];
                    }
                }
            }
    }
}

template <int EPI>
static int launch_fc(const CUtensorMap& tm, const unsigned char* bglob, const Img& d, const FCParams& p, size_t smem, int grid, cudaStream_t st)
{
    auto kern = filter2d_tc_kernel<EPI>;
    static PerDeviceFlag attr_pd; bool& attr = attr_pd.cur();
    if (!attr) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FC_SMEM_MAX)); attr = true; }
    kern<<<grid, FC_THREADS, smem, st>>>(tm, bglob, d, p);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

// filter2D, 8-bit single-channel source.  dd = destination depth.
// returns B200CV_NOT_IMPLEMENTED when the tensor-core path does not apply (caller uses the direct-sum kernel)
int filter2d_u8_tensor(const Img& s, const Img& d, int dd, const float* k, int kw, int kh, int ax, int ay, float delta, int border, cudaStream_t st)
{
    if (kw + FC_NT - 1 > FC_K || kh > 33 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
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
    p.tiles_x = (int)div_up((unsigned)p.ow, FC_NT); p.tiles_y = (int)div_up((unsigned)p.oh, 128 * FC_WG);
    const long long nt = (long long)p.tiles_x * p.tiles_y * p.frames;
    if (nt > 0x7fffffff) return B200CV_NOT_IMPLEMENTED;
    p.ntiles = (int)nt;
    const int ra = 128 * FC_WG + kh - 1;
    p.nbox = (ra + 255) / 256;
    p.box_h = (((ra + p.nbox - 1) / p.nbox) + 7) & ~7;
    p.ra_alloc = p.nbox * p.box_h;
    const size_t abytes = (size_t)(FC_K / 16) * p.ra_alloc * 16;
    if ((size_t)kh * FC_BROW + 2 * abytes > (size_t)FC_SMEM_MAX) return B200CV_NOT_IMPLEMENTED;
    p.na = (int)std::min<size_t>(4, ((size_t)FC_SMEM_MAX - (size_t)kh * FC_BROW) / abytes);
    const size_t smem = (size_t)kh * FC_BROW + p.na * abytes;
    const int n_sm = num_sms();
    const int grid = (int)std::min<long long>(nt, n_sm);

    // border-extended source, rows padded to a multiple of 16 bytes (TMA)
    Img pad = s;
    pad.cols = (s.cols + kw - 1 + 15) & ~15;
    pad.rows = s.rows + kh - 1;
    pad.step = (size_t)pad.cols;
    pad.fstep = pad.step * pad.rows;
    unsigned char* pbuf = nullptr; unsigned char* bglob = nullptr;
    B200_CUDA(cudaMallocAsync(&pbuf, pad.fstep * (size_t)s.frames, st));
    B200_CUDA(cudaMallocAsync(&bglob, (size_t)kh * FC_BROW, st));
    pad.data = pbuf;
    fc_toeplitz_kernel<<<kh, 256, 0, st>>>(kq, kw, (signed char*)bglob);
    count_launch();
    launch_pad_u8(s, pad, ax, ay, border, st);
    CUtensorMap tm;
    int rc = make_tensor_map_3d(&tm, pad.data, 1, pad.cols, pad.rows, pad.frames, pad.step, pad.fstep, 16, p.box_h);
    if (!rc) {
        rc = dd == B200CV_8U ? launch_fc<FC_U8>(tm, bglob, d, p, smem, grid, st)
           : dd == B200CV_16S ? launch_fc<FC_S16>(tm, bglob, d, p, smem, grid, st)
                              : launch_fc<FC_F32>(tm, bglob, d, p, smem, grid, st);
    }
    cudaFreeAsync(bglob, st);
    cudaFreeAsync(pbuf, st);
    return rc;
}

}  // namespace b200cv
