// matchtemplate_tc.cu -- the matchTemplate correlation numerator on Hopper tensor cores (wgmma, u8 x u8 -> s32).
//
//   R(y, x) = sum_{v<h} sum_{u<w} T(v,u) * I(y+v, x+u)          8-bit image and template, exact 32-bit integer result
//
// is a dense contraction with N = 1 per window.  To give the MMA a useful N the template row is expanded into a banded
// (Toeplitz) operand: for an x-tile of 64 outputs and one template row v
//   D[m][j] += sum_{k<128} A_v[m][k] * B_v[k][j],   A_v[m][k] = I(y0+m+v, x0+k),   B_v[k][j] = T(v, k-j) (0 outside [0,w))
// A_v is a plain 128-byte-wide box of image rows -- NO im2col is materialised: the CTA stages rows y0 .. y0+M+h-2 once
// (TMA, 16-byte-column boxes = the canonical K-major no-swizzle core-matrix layout) and the A descriptor of step v simply
// starts v rows (v*16 bytes) further down.  B_v (8 KB) is pre-expanded once per call into global memory in the same layout
// and streamed through a 4-stage cp.async.bulk ring by a producer warp.  Two consumer warpgroups each own 128 output rows
// (two wgmma m64n64k32 slabs sharing every B_v, accumulators in registers) and store float(R) from their registers.  Half of B
// is zeros (2.1x redundant MACs), the price of a well-shaped MMA; the result is exact because products <= 65025
// and sums < 2^31.
//
//
// (8-bit filter2D with >= 11x11 taps uses the same Toeplitz formulation in a persistent kernel: filter2d_tc.cu.)
//
// Reference: crossCorr, modules/imgproc/src/templmatch.cpp:566-760 (block DFT in float on one thread).
#include "common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"
#include <cmath>
#include <vector>

namespace b200cv {

constexpr int TC_N = 64;          // outputs per x-tile (MMA N)
constexpr int TC_K = 128;         // K per template row: w + N - 1 <= 128
constexpr int TC_WG = 2;          // consumer warpgroups per CTA, 128 output rows each
constexpr int TC_THREADS = 128 * TC_WG + 32;   // + one producer warp
constexpr int TC_NS = 4;          // B ring stages
constexpr int TC_BBYTES = TC_N * TC_K;   // 8192


// B_v in smem/global: [k-chunk c (8)][column j (64)][16 bytes]: byte b = T(v, 16c + b - j)
__global__ void toeplitz_kernel(Img templ, int w, int h, unsigned char* out)
{
    const int v = blockIdx.x;
    for (int idx = threadIdx.x; idx < TC_BBYTES; idx += blockDim.x) {
        int c = idx >> 10, j = (idx >> 4) & 63, b = idx & 15;
        int u = 16 * c + b - j;
        out[(size_t)v * TC_BBYTES + idx] = (u >= 0 && u < w) ? templ.row<uchar>(0, v)[u] : (uchar)0;
    }
}

// border-extended copy of an 8-bit single-channel image: P(y, x) = src(y - ay, x - ax) under `border`.
// 16 output bytes per thread; away from the borders the (generally unaligned) source run is read as 5 aligned words and realigned
// with funnel shifts.
__global__ void __launch_bounds__(128) pad_u8_kernel(Img src, Img dst, int ax, int ay, int border, int words_ok)
{
    const int f = blockIdx.z, y = blockIdx.y;
    const int x16 = (blockIdx.x * blockDim.x + threadIdx.x) * 16;
    if (x16 >= dst.cols) return;
    const int sy = border_interpolate(y - ay, src.rows, border);
    uint32_t o[4] = {0, 0, 0, 0};
    if (sy >= 0) {
        const uchar* sp = src.row<uchar>(f, sy);
        const int sx0 = x16 - ax;
        if (words_ok && sx0 >= 0 && sx0 + 20 <= src.cols) {
            const int a = sx0 & 3;
            const uint32_t* wp = (const uint32_t*)(sp + (sx0 - a));
            uint32_t w[5];
#pragma unroll
            for (int i = 0; i < 5; i++) w[i] = wp[i];
#pragma unroll
            for (int i = 0; i < 4; i++) o[i] = __funnelshift_r(w[i], w[i + 1], 8 * a);
        } else {
#pragma unroll
            for (int i = 0; i < 16; i++) {
                int sx = border_interpolate(sx0 + i, src.cols, border);
                o[i >> 2] |= (uint32_t)(sx >= 0 ? sp[sx] : (uchar)0) << (8 * (i & 3));
            }
        }
    }
    *(uint4*)(dst.row<uchar>(f, y) + x16) = make_uint4(o[0], o[1], o[2], o[3]);
}

struct TCParams {
    int h, ra_alloc, box_h, nbox;       // template rows; staged image rows (allocated), rows per TMA box, boxes per column chunk
    int ow, oh;
    int kch;                            // K per template row = 32 * kch (w + N - 1 <= 32 * kch)
};

__global__ void __launch_bounds__(TC_THREADS) ccorr_u8_tc_kernel(const __grid_constant__ CUtensorMap tmap, const unsigned char* __restrict__ bglob, Img res, TCParams p)
{
    constexpr int NN = TC_N;                                           // MMA N
    extern __shared__ __align__(128) unsigned char smem[];
    const int nchunk = 2 * p.kch;                                      // 16-byte K chunks per row
    const uint32_t bbytes = (uint32_t)nchunk * NN * 16;                // one B slab
    unsigned char* sA = smem;                                          // nchunk x ra_alloc rows x 16 B
    unsigned char* sB = smem + (size_t)nchunk * p.ra_alloc * 16;       // TC_NS slabs
    __shared__ __align__(8) uint64_t full[TC_NS], empty[TC_NS], a_full;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.z, x0 = blockIdx.x * TC_N, y0 = blockIdx.y * (128 * TC_WG);
    const uint32_t lbo_a = (uint32_t)p.ra_alloc * 16u;

    if (threadIdx.x == 0) {
        for (int s = 0; s < TC_NS; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4 * TC_WG); }
        mbar_init(&a_full, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 4 * TC_WG) {
        // ---- producer: image rows once, then the Toeplitz operand of every template row through the ring ----
        if (lane == 0) {
            mbar_arrive_expect_tx(&a_full, (uint32_t)p.ra_alloc * 16u * nchunk);
            for (int c = 0; c < nchunk; c++)
                for (int b = 0; b < p.nbox; b++)
                    tma_load_3d(sA + (size_t)c * lbo_a + (size_t)b * p.box_h * 16, &tmap, x0 + 16 * c, y0 + b * p.box_h, f, &a_full);
            for (int v = 0; v < p.h; v++) {
                const int s = v % TC_NS;
                mbar_wait(&empty[s], ((v / TC_NS) & 1) ^ 1);
                mbar_arrive_expect_tx(&full[s], bbytes);
                wg_bulk_load(sB + (size_t)s * bbytes, bglob + (size_t)v * bbytes, bbytes, &full[s]);
            }
        }
        return;
    }

    // ---- consumers: warpgroup wg owns accumulator rows 128 wg .. 128 wg + 127 as two 64-row slabs ----
    const int wg = warp >> 2, wl = warp & 3;
    uint32_t acc[2][NN / 2];
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
        for (int r = 0; r < NN / 2; r++) acc[m][r] = 0;
    mbar_wait(&a_full, 0);
    wg_fence();
    const uint32_t a0 = smem_u32(sA) + (uint32_t)(wg * 128) * 16u, b0 = smem_u32(sB);
    int prev = -1;
    for (int v = 0; v < p.h; v++) {
        const int s = v % TC_NS;
        mbar_wait(&full[s], (v / TC_NS) & 1);
#pragma unroll
        for (int ks = 0; ks < TC_K / 32; ks++) {
            const uint64_t bd = wg_desc(b0 + (uint32_t)s * bbytes + (uint32_t)ks * (2 * NN * 16), NN * 16, 128);
#pragma unroll
            for (int m = 0; m < 2; m++)    // the A operand of template row v starts v image rows (v x 16 bytes) further down
                wgmma_u8u8_n64(acc[m], wg_desc(a0 + (uint32_t)ks * 2u * lbo_a + (uint32_t)(m * 64 + v) * 16u, lbo_a, 128), bd);
        }
        wg_commit();
        wg_wait<1>();                      // the previous row's MMAs are done: its ring slot may be refilled
        wg_mbar_arrive_if(&empty[prev < 0 ? 0 : prev], lane == 0 && prev >= 0);
        prev = s;
    }
    wg_wait<0>();
    wg_fence_operand(acc[0]);
    wg_fence_operand(acc[1]);
    // ---- epilogue straight from the accumulator registers ----
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int gy = y0 + wg * 128 + m * 64 + wl * 16 + (lane >> 2) + 8 * i;
            if (gy >= p.oh) continue;
            float* rp = res.row<float>(f, gy);
#pragma unroll
            for (int j = 0; j < NN / 8; j++)
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    const int gx = x0 + 8 * j + 2 * (lane & 3) + c;
                    if (gx < p.ow) rp[gx] = (float)(int)acc[m][4 * j + 2 * i + c];
                }
        }
}

// returns B200CV_NOT_IMPLEMENTED when the tensor-core path does not apply (caller uses the IDP4A kernel)
int ccorr_u8_tensor(const Img& im, const Img& tp, const Img& rs, int w, int h, cudaStream_t st)
{
    if (w > TC_K - TC_N + 1 || h > 512 || !tma_compatible(im) || im.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    const int ow = im.cols - w + 1, oh = im.rows - h + 1;
    TCParams p;
    p.h = h; p.ow = ow; p.oh = oh; p.kch = TC_K / 32;
    int ra = 128 * TC_WG + h - 1;
    p.nbox = (ra + 255) / 256;
    p.box_h = (((ra + p.nbox - 1) / p.nbox) + 7) & ~7;
    p.ra_alloc = p.nbox * p.box_h;
    size_t smem = (size_t)8 * p.ra_alloc * 16 + (size_t)TC_NS * TC_BBYTES;
    if (smem > 200 * 1024) return B200CV_NOT_IMPLEMENTED;
    static PerDeviceFlag attr_pd; bool& attr = attr_pd.cur();
    if (!attr) { B200_CUDA(cudaFuncSetAttribute(ccorr_u8_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
    unsigned char* bglob = nullptr;
    B200_CUDA(cudaMallocAsync(&bglob, (size_t)h * TC_BBYTES, st));
    toeplitz_kernel<<<h, 256, 0, st>>>(tp, w, h, bglob);
    count_launch();
    CUtensorMap tm;
    int rc = make_tensor_map_3d(&tm, im.data, 1, im.cols, im.rows, im.frames, im.step, im.fstep, 16, p.box_h);
    if (rc) { cudaFreeAsync(bglob, st); return rc; }
    dim3 grid(div_up((unsigned)ow, TC_N), div_up((unsigned)oh, 128 * TC_WG), (unsigned)im.frames);
    ccorr_u8_tc_kernel<<<grid, TC_THREADS, smem, st>>>(tm, bglob, rs, p);
    cudaError_t e = cudaGetLastError();
    cudaFreeAsync(bglob, st);
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

void launch_pad_u8(const Img& src, const Img& dst, int ax, int ay, int border, cudaStream_t st)
{
    pad_u8_kernel<<<dim3(div_up((unsigned)dst.cols / 16, 128), (unsigned)dst.rows, (unsigned)src.frames), 128, 0, st>>>(
        src, dst, ax, ay, border, (((uintptr_t)src.data | src.step | src.fstep) & 3) == 0);
    count_launch();
}

}  // namespace b200cv
