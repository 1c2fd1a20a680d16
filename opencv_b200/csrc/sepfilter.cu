// sepfilter.cu -- separable linear filters: cv::GaussianBlur, cv::sepFilter2D, cv::Sobel.
//
// One fused kernel per call: a CTA stages an input tile + apron in shared memory (128-bit loads of whole
// 16-byte segments; border pixels resolved per cv::borderInterpolate), runs the row pass into a shared
// float buffer and the column pass straight to global memory -- the intermediate never touches HBM
// (the CPU reference does the same through a ksize-row ring, smooth.simd.hpp:2013-2130 / filter.simd.hpp:198-297).
//
// Arithmetic
//  * u8 GaussianBlur (bit-exact): taps are the reference's 8.8 fixed-point values; the reference computes
//      dst = sat_u8((sum_j ky[j] * (sum_i kx[i]*src) + 2^15) >> 16)        (smooth.simd.hpp:1925-2197,
//      model: modules/imgproc/test/test_smooth_bitexact.cpp:40-53).  Every partial sum is an integer
//      < 2^24 (sum k = 256, src <= 255), hence exactly representable in fp32: the kernel accumulates with
//      FFMA and is still bit-exact.  Same for sepFilter2D's int32 "bit-exact mode" (filter.dispatch.cpp:334-362).
//  * float paths (f32 images, u8->f32/s16/u8 with non-exact taps): row pass s=0; s=fma(src,kx[i],s) in tap order
//      (RowVec_32f, filter.simd.hpp:1634-1648); column pass starts from delta and adds taps in order
//      (ColumnFilter, filter.simd.hpp:2580-2650); output through saturate_cast (round-half-even).
//
// Two kernels:
//  * sep_fast_kernel<ST,DT,MODE,KB>  single-channel images, odd centred kernels up to 31 taps; tap count is a
//      template bucket so the taps are constant-bank operands and all window indexing is resolved at compile time; for a
//      float source the zero taps the reference never evaluates (the padding to the bucket, the centre of antisymmetric columns and
//      3/5-tap rows) are skipped (SKIP0, here and in the generic kernel), so a non-finite pixel reaches only the real footprint;
//  * sep_generic_kernel<ST,DT,MODE>  any channel count / anchor / tap count <= 33, run-time loops.
#include <cmath>
#include <vector>
#include "common.cuh"
#include "host_tables.h"

namespace b200cv {

int sep_u8_float_fast(const Img& s, const Img& d, const float* kx, int nx, const float* ky, int ny, float delta, int border, cudaStream_t st);
int sep_f32_fast(const Img& s, const Img& d, const float* kx, int nx, const float* ky, int ny, float delta, int border, const Img* dog, cudaStream_t st);


enum { M_FLOAT = 0, M_FIXED16 = 1, M_INT = 2 };

struct SepParams {
    SepTaps t;        // kx/ky (for the fast kernel: zero padded + centred to KB taps)
    float delta;      // M_FLOAT: added in the column pass
    int delta_i;      // M_FIXED16 / M_INT: integer delta added after the exact accumulation
    int border;
    int cn;
    Img dog;          // optional second output (f32 only): dog = dst - src, the SIFT difference-of-Gaussians level
    int has_dog;
    int even_limit;   // M_FIXED16: row elements < even_limit round half-to-even (sepFilter2D's vector body), the rest half-up
    int row_small;    // M_FLOAT, float source, 3/5 (anti)symmetric taps: 1|2 = centre-out order of SymmRowSmallVec_32f, 0 = tap order
    int col_mode;     // M_FLOAT: 1|2 = (anti)symmetric column kernel, mirrored rows added first; 0 = scalar ColumnFilter order (no FMA)
    int px, py;       // M_FLOAT fast kernel: zero taps padding kx / ky to the bucket on each side, not evaluated under SKIP0 (fma(inf, 0, s) = NaN)
};

template <typename T> __device__ __forceinline__ float to_f(T v) { return (float)v; }

template <typename DT, int MODE> __device__ __forceinline__ DT finish(float acc, int delta_i, int xe = 0, int even_limit = 0)
{
    if constexpr (MODE == M_FIXED16) {
        int t = (int)acc + delta_i;
        if (xe < even_limit) {   // reference: SymmColumnVec_32s8u rounds the exact value half-to-even (filter.simd.hpp:1011-1100)
            int q = t >> 16, r = t & 0xffff;
            return (DT)sat_u8(q + ((r > 32768) || (r == 32768 && (q & 1))));
        }
        return (DT)sat_u8((t + 32768) >> 16);
    } else if constexpr (MODE == M_INT) {
        if constexpr (sizeof(DT) == 2) return (DT)sat_s16((int)acc + delta_i);
        else return (DT)sat_u8((int)acc + delta_i);
    } else {
        return OutCast<DT>::from(acc);
    }
}

// ================================================================================================================
// generic kernel: any cn, any anchor, run-time tap loops
// ================================================================================================================
constexpr int G_TPX = 64;   // tile width in pixels
constexpr int G_TH = 16;    // tile height

template <typename ST, typename DT, int MODE>
__global__ void __launch_bounds__(256) sep_generic_kernel(Img src, Img dst, SepParams p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int cn = p.cn, nx = p.t.nx, ny = p.t.ny, ax = p.t.ax, ay = p.t.ay;
    const int tile_px = G_TPX + nx - 1;            // input tile width in pixels
    const int tile_rows = G_TH + ny - 1;
    const int in_w = tile_px * cn;                 // elements per input row
    const int mid_w = G_TPX * cn;
    float* s_in = (float*)smem_raw;                // tile_rows x in_w
    float* s_mid = s_in + tile_rows * in_w;        // tile_rows x mid_w
    const int f = blockIdx.z;
    const int x0 = blockIdx.x * G_TPX, y0 = blockIdx.y * G_TH;

    // ---- load (with border) ----
    for (int idx = threadIdx.x; idx < tile_rows * tile_px; idx += blockDim.x) {
        int r = idx / tile_px, c = idx - r * tile_px;
        int sy = border_interpolate(y0 - ay + r, src.rows, p.border);
        int sx = border_interpolate(x0 - ax + c, src.cols, p.border);
        float* d = s_in + r * in_w + c * cn;
        if (sy < 0 || sx < 0) {
            for (int ch = 0; ch < cn; ch++) d[ch] = 0.f;
        } else {
            const ST* sp = src.row<ST>(f, sy) + (size_t)sx * cn;
            for (int ch = 0; ch < cn; ch++) d[ch] = to_f(sp[ch]);
        }
    }
    __syncthreads();
    // ---- row pass ----
    for (int idx = threadIdx.x; idx < tile_rows * mid_w; idx += blockDim.x) {
        int r = idx / mid_w, e = idx - r * mid_w;
        const float* s = s_in + r * in_w + e;
        float acc = 0.f;
        if (MODE == M_FLOAT && p.row_small) {             // filter.simd.hpp:1768-1844 (see sep_f32.cu)
            const int m = nx / 2;
            const float sg = p.row_small == 2 ? -1.f : 1.f;
            acc = __fmul_rn(__fadd_rn(s[(m + 1) * cn], sg * s[(m - 1) * cn]), p.t.kx[m + 1]);
            if (p.row_small != 2) acc = fmaf(s[m * cn], p.t.kx[m], acc);      // antisymmetric: no centre term
            if (nx == 5) acc = fmaf(__fadd_rn(s[(m + 2) * cn], sg * s[(m - 2) * cn]), p.t.kx[m + 2], acc);
        } else {
            for (int i = 0; i < nx; i++) acc = fmaf(s[i * cn], p.t.kx[i], acc);
        }
        s_mid[idx] = acc;
    }
    __syncthreads();
    // ---- column pass ----
    for (int idx = threadIdx.x; idx < G_TH * mid_w; idx += blockDim.x) {
        int r = idx / mid_w, e = idx - r * mid_w;
        int y = y0 + r, xe = x0 * cn + e;
        if (y >= dst.rows || xe >= dst.cols * cn) continue;
        const float* s = s_mid + r * mid_w + e;
        float acc = 0.f;
        if constexpr (MODE == M_FLOAT) {
            if (p.col_mode) {                             // SymmColumnVec_32f / _32f8u: filter.simd.hpp:1878-1949, :1158-1202
                const int c = ny / 2;
                const float sg = p.col_mode == 2 ? -1.f : 1.f;
                acc = p.col_mode == 2 ? p.delta : fmaf(p.t.ky[c], s[c * mid_w], p.delta);      // antisymmetric: no centre row
                for (int k = 1; k <= c; k++) acc = fmaf(p.t.ky[c + k], __fadd_rn(s[(c + k) * mid_w], sg * s[(c - k) * mid_w]), acc);
            } else {                                      // scalar ColumnFilter: products rounded before they are added, :2590-2640
                acc = fmaf(s[0], p.t.ky[0], p.delta);      // only the delta term is contracted in the reference object
                for (int j = 1; j < ny; j++) acc = __fadd_rn(acc, __fmul_rn(s[j * mid_w], p.t.ky[j]));
            }
        } else {
            for (int j = 0; j < ny; j++) acc = fmaf(s[j * mid_w], p.t.ky[j], acc);
        }
        DT outv = finish<DT, MODE>(acc, p.delta_i, xe, p.even_limit);
        dst.row<DT>(f, y)[xe] = outv;
        if constexpr (MODE == M_FLOAT && sizeof(ST) == 4 && sizeof(DT) == 4)
            if (p.has_dog) p.dog.row<float>(f, y)[xe] = __fsub_rn((float)outv, s_in[(r + ay) * in_w + e + ax * cn]);
    }
}

// ================================================================================================================
// fast kernel: single channel, centred odd kernels, compile-time tap bucket KB
// ================================================================================================================
constexpr int F_TW = 256;   // tile width (pixels == elements)
constexpr int F_R = 8;      // outputs per row-pass work item

template <typename ST> struct Apron {   // horizontal apron rounded so that tile rows start on 16-byte boundaries
    static constexpr int of(int rb) { return sizeof(ST) == 1 ? ((rb + 15) / 16) * 16 : ((rb + 3) / 4) * 4; }
};

__device__ __forceinline__ float byte_to_float(uint32_t w, int j)
{
    // place byte j of w into the mantissa of 2^23 and subtract 2^23: exact u8 -> f32 without I2F
    return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540u | (unsigned)j)) - 8388608.0f;
}

template <typename ST, typename DT, int MODE, int KB, bool SKIP0>
__global__ void __launch_bounds__(256) sep_fast_kernel(Img src, Img dst, const __grid_constant__ SepParams p, int TH)
{
    constexpr int RB = KB / 2;
    constexpr int RP = Apron<ST>::of(RB);
    constexpr int SW = F_TW + 2 * RP;                     // input tile row stride in elements
    constexpr int EPV = 16 / (int)sizeof(ST);             // elements per 16-byte vector
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int in_rows = TH + 2 * RB;
    ST* s_in = (ST*)smem_raw;
    float* s_mid = (float*)(smem_raw + (((size_t)in_rows * SW * sizeof(ST) + 15) & ~(size_t)15));   // in_rows x F_TW

    const int f = blockIdx.z;
    const int x0 = blockIdx.x * F_TW, y0 = blockIdx.y * TH;
    const bool aligned = (((uintptr_t)src.data | src.step | src.fstep) & 15) == 0;

    // ---- load tile + apron: one 16-byte vector per work item --------------------------------------------------
    {
        constexpr int VPR = SW / EPV;                     // vectors per tile row
        for (int idx = threadIdx.x; idx < in_rows * VPR; idx += 256) {
            int r = idx / VPR, v = idx - r * VPR;
            int gx = x0 - RP + v * EPV;                   // first source column of this vector
            int sy = border_interpolate(y0 - RB + r, src.rows, p.border);
            ST* d = s_in + r * SW + v * EPV;
            if (sy < 0) {
                *(uint4*)d = make_uint4(0, 0, 0, 0);
            } else if (aligned && gx >= 0 && gx + EPV <= src.cols) {
                *(uint4*)d = __ldg((const uint4*)(src.row<ST>(f, sy) + gx));
            } else {
                const ST* sp = src.row<ST>(f, sy);
#pragma unroll
                for (int e = 0; e < EPV; e++) {
                    int sx = border_interpolate(gx + e, src.cols, p.border);
                    d[e] = sx < 0 ? (ST)0 : sp[sx];
                }
            }
        }
    }
    __syncthreads();

    // ---- row pass: work item = F_R consecutive outputs of one tile row -------------------------------------------
    {
        constexpr int GPR = F_TW / F_R;                   // items per row
        constexpr int LO = RP - RB;                       // first needed column offset inside the item's window
        constexpr int NEED = F_R + KB - 1;                // window elements
        for (int idx = threadIdx.x; idx < in_rows * GPR; idx += 256) {
            int r = idx / GPR, g = idx - r * GPR;
            const ST* base = s_in + r * SW + g * F_R;     // aligned: g*F_R multiple of 8 elements
            float acc[F_R];
#pragma unroll
            for (int o = 0; o < F_R; o++) acc[o] = 0.f;
            if constexpr (sizeof(ST) == 1) {
                constexpr int W0 = LO / 4, W1 = (LO + NEED - 1) / 4;
                const uint32_t* wp = (const uint32_t*)base;
#pragma unroll
                for (int w = W0; w <= W1; w++) {
                    uint32_t word = wp[w];
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        const int e = w * 4 + b - LO;     // window element index (compile-time after unrolling)
                        if (e >= 0 && e < NEED) {
                            float v = byte_to_float(word, b);
#pragma unroll
                            for (int o = 0; o < F_R; o++) {
                                const int i = e - o;
                                if (i >= 0 && i < KB) acc[o] = fmaf(v, p.t.kx[i], acc[o]);
                            }
                        }
                    }
                }
            } else if (MODE == M_FLOAT && KB <= 5 && p.row_small) {
                const float sg = p.row_small == 2 ? -1.f : 1.f;
                const ST* x = base + LO + RB;              // centre tap of output 0
#pragma unroll
                for (int o = 0; o < F_R; o++) {
                    float t = __fmul_rn(__fadd_rn((float)x[o + 1], sg * (float)x[o - 1]), p.t.kx[RB + 1]);
                    if (!SKIP0 || p.row_small != 2) t = fmaf((float)x[o], p.t.kx[RB], t);
                    if (KB == 5 && (!SKIP0 || !p.px)) t = fmaf(__fadd_rn((float)x[o + 2], sg * (float)x[o - 2]), p.t.kx[RB + 2], t);
                    acc[o] = t;
                }
            } else {
                constexpr int V0 = LO / 4, V1 = (LO + NEED - 1) / 4;
                const float4* vp = (const float4*)base;
#pragma unroll
                for (int w = V0; w <= V1; w++) {
                    float4 q = vp[w];
                    float vals[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        const int e = w * 4 + b - LO;
                        if (e >= 0 && e < NEED) {
#pragma unroll
                            for (int o = 0; o < F_R; o++) {
                                const int i = e - o;
                                if (i >= 0 && i < KB && (!SKIP0 || (i >= p.px && i < KB - p.px))) acc[o] = fmaf(vals[b], p.t.kx[i], acc[o]);
                            }
                        }
                    }
                }
            }
            float4* mp = (float4*)(s_mid + r * F_TW + g * F_R);
            mp[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
            mp[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
        }
    }
    __syncthreads();

    // ---- column pass: work item = 4 columns x 8 rows, streaming over the mid rows ----------------------------------
    {
        constexpr int RV = 8;
        const int qn = TH / RV;
        const bool dst_vec = (((uintptr_t)dst.data | dst.step | dst.fstep) & (4 * sizeof(DT) - 1)) == 0;
        for (int idx = threadIdx.x; idx < (F_TW / 4) * qn; idx += 256) {
            int q = idx / (F_TW / 4), c4 = idx - q * (F_TW / 4);
            const float* mbase = s_mid + (q * RV) * F_TW + c4 * 4;
            float acc[RV][4];
#pragma unroll
            for (int o = 0; o < RV; o++)
#pragma unroll
                for (int c = 0; c < 4; c++) acc[o][c] = 0.f;
            if constexpr (MODE == M_FLOAT) {
                // (anti)symmetric column kernel, mirrored rows added first (the only float kernels routed here)
                const float sg = p.col_mode == 2 ? -1.f : 1.f;
#pragma unroll 1
                for (int o = 0; o < RV; o++) {
                    const float* ctr = mbase + (o + RB) * F_TW;
                    const float4 v0 = *(const float4*)ctr;
                    const float t0 = p.t.ky[RB];
                    float a0 = p.delta, a1 = p.delta, a2 = p.delta, a3 = p.delta;
                    if (!SKIP0 || p.col_mode != 2) {                // antisymmetric: no centre row
                        a0 = fmaf(t0, v0.x, p.delta); a1 = fmaf(t0, v0.y, p.delta); a2 = fmaf(t0, v0.z, p.delta); a3 = fmaf(t0, v0.w, p.delta);
                    }
#pragma unroll
                    for (int k = 1; k <= RB; k++) {
                        if (SKIP0 && k > RB - p.py) break;          // zero taps padding ky to the bucket
                        const float4 va = *(const float4*)(ctr + k * F_TW), vb = *(const float4*)(ctr - k * F_TW);
                        const float t = p.t.ky[RB + k];
                        a0 = fmaf(t, __fadd_rn(va.x, sg * vb.x), a0); a1 = fmaf(t, __fadd_rn(va.y, sg * vb.y), a1);
                        a2 = fmaf(t, __fadd_rn(va.z, sg * vb.z), a2); a3 = fmaf(t, __fadd_rn(va.w, sg * vb.w), a3);
                    }
                    acc[o][0] = a0; acc[o][1] = a1; acc[o][2] = a2; acc[o][3] = a3;
                }
            } else
#pragma unroll
            for (int m = 0; m < RV + KB - 1; m++) {
                float4 v = *(const float4*)(mbase + m * F_TW);
#pragma unroll
                for (int o = 0; o < RV; o++) {
                    const int j = m - o;
                    if (j >= 0 && j < KB) {
                        float t = p.t.ky[j];
                        acc[o][0] = fmaf(v.x, t, acc[o][0]);
                        acc[o][1] = fmaf(v.y, t, acc[o][1]);
                        acc[o][2] = fmaf(v.z, t, acc[o][2]);
                        acc[o][3] = fmaf(v.w, t, acc[o][3]);
                    }
                }
            }
            const int gx = x0 + c4 * 4;
            if (gx >= dst.cols) continue;
#pragma unroll
            for (int o = 0; o < RV; o++) {
                int gy = y0 + q * RV + o;
                if (gy >= dst.rows) break;
                DT* dp = dst.row<DT>(f, gy) + gx;
                DT out[4];
#pragma unroll
                for (int c = 0; c < 4; c++) out[c] = finish<DT, MODE>(acc[o][c], p.delta_i, gx + c, p.even_limit);
                if (dst_vec && gx + 4 <= dst.cols) {
                    if constexpr (sizeof(DT) == 1) *(uchar4*)dp = make_uchar4(out[0], out[1], out[2], out[3]);
                    else if constexpr (sizeof(DT) == 2) *(short4*)dp = make_short4(out[0], out[1], out[2], out[3]);
                    else *(float4*)dp = make_float4(out[0], out[1], out[2], out[3]);
                } else {
#pragma unroll
                    for (int c = 0; c < 4; c++) if (gx + c < dst.cols) dp[c] = out[c];
                }
                if constexpr (MODE == M_FLOAT && sizeof(ST) == 4 && sizeof(DT) == 4) {
                    if (p.has_dog) {       // DoG level fused into the blur that produces its minuend (sift.dispatch.cpp:292)
                        const ST* ctr = s_in + (q * RV + o + RB) * SW + RP + c4 * 4;
                        float* gp = p.dog.row<float>(f, gy) + gx;
#pragma unroll
                        for (int c = 0; c < 4; c++) if (gx + c < dst.cols) gp[c] = __fsub_rn((float)out[c], (float)ctr[c]);
                    }
                }
            }
        }
    }
}

// ================================================================================================================
// host dispatch
// ================================================================================================================
template <typename ST, typename DT, int MODE, int KB, bool SKIP0>
static int launch_fast(const Img& s, const Img& d, const SepParams& p, cudaStream_t st)
{
    constexpr int RB = KB / 2;
    constexpr int RP = Apron<ST>::of(RB);
    constexpr int SW = F_TW + 2 * RP;
    auto smem_for = [&](int TH) { return (((size_t)(TH + 2 * RB) * SW * sizeof(ST) + 15) & ~(size_t)15) + (size_t)(TH + 2 * RB) * F_TW * sizeof(float); };
    int TH = 32;
    if (smem_for(TH) > 110 * 1024) TH = 16;     // keep two CTAs per SM resident
    if (s.rows <= 16) TH = 16;
    if (s.rows <= 8) TH = 8;
    size_t smem = smem_for(TH);
    auto kern = sep_fast_kernel<ST, DT, MODE, KB, SKIP0>;
    static PerDeviceFlag attr_done_pd; bool& attr_done = attr_done_pd.cur();
    if (!attr_done) {
        B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_done = true;
    }
    dim3 grid(div_up((unsigned)s.cols, F_TW), div_up((unsigned)s.rows, (unsigned)TH), (unsigned)s.frames);
    kern<<<grid, 256, smem, st>>>(s, d, p, TH);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

template <typename ST, typename DT, int MODE, bool SKIP0>
static int launch_fast_kb(int kb, const Img& s, const Img& d, const SepParams& p, cudaStream_t st)
{
    switch (kb) {
    case 3: return launch_fast<ST, DT, MODE, 3, SKIP0>(s, d, p, st);
    case 5: return launch_fast<ST, DT, MODE, 5, SKIP0>(s, d, p, st);
    case 7: return launch_fast<ST, DT, MODE, 7, SKIP0>(s, d, p, st);
    case 9: return launch_fast<ST, DT, MODE, 9, SKIP0>(s, d, p, st);
    case 11: return launch_fast<ST, DT, MODE, 11, SKIP0>(s, d, p, st);
    case 13: return launch_fast<ST, DT, MODE, 13, SKIP0>(s, d, p, st);
    case 15: return launch_fast<ST, DT, MODE, 15, SKIP0>(s, d, p, st);
    case 17: return launch_fast<ST, DT, MODE, 17, SKIP0>(s, d, p, st);
    case 21: return launch_fast<ST, DT, MODE, 21, SKIP0>(s, d, p, st);
    case 25: return launch_fast<ST, DT, MODE, 25, SKIP0>(s, d, p, st);
    case 27: return launch_fast<ST, DT, MODE, 27, SKIP0>(s, d, p, st);
    case 31: return launch_fast<ST, DT, MODE, 31, SKIP0>(s, d, p, st);
    }
    set_error("internal: no fast bucket for %d taps", kb);
    return B200CV_ERR_BAD_ARG;
}

// float sources with zero taps the reference never evaluates (padding to the bucket, antisymmetric centres): the instantiation that skips
// them (8-bit rows and integer modes are finite)
template <typename ST, typename DT, int MODE>
static int launch_fast_k(int kb, const Img& s, const Img& d, const SepParams& p, cudaStream_t st)
{
    if (MODE == M_FLOAT && sizeof(ST) == 4 && (p.px || p.py || p.row_small == 2 || p.col_mode == 2)) return launch_fast_kb<ST, DT, MODE, true>(kb, s, d, p, st);
    return launch_fast_kb<ST, DT, MODE, false>(kb, s, d, p, st);
}

static int fast_bucket(int k)
{
    static const int buckets[] = {3, 5, 7, 9, 11, 13, 15, 17, 21, 25, 27, 31};
    for (int b : buckets) if (k <= b) return b;
    return 0;
}

template <typename ST, typename DT, int MODE>
static int launch_generic(const Img& s, const Img& d, const SepParams& p, cudaStream_t st)
{
    int tile_px = G_TPX + p.t.nx - 1, tile_rows = G_TH + p.t.ny - 1;
    size_t smem = ((size_t)tile_rows * tile_px * p.cn + (size_t)tile_rows * G_TPX * p.cn) * sizeof(float);
    if (smem > 200 * 1024) return B200CV_NOT_IMPLEMENTED;
    auto kern = sep_generic_kernel<ST, DT, MODE>;
    static PerDeviceFlag attr_done_pd; bool& attr_done = attr_done_pd.cur();
    if (!attr_done) {
        B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_done = true;
    }
    dim3 grid(div_up((unsigned)s.cols, G_TPX), div_up((unsigned)s.rows, G_TH), (unsigned)s.frames);
    kern<<<grid, 256, smem, st>>>(s, d, p);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

// common entry: taps are float arrays; mode picks the epilogue
template <typename ST, typename DT, int MODE>
static int sep_dispatch(const Img& s, const Img& d, int cn, const float* kx, int nx, const float* ky, int ny, int ax, int ay,
                        float delta, int delta_i, int border, cudaStream_t st, int even_limit = 0, const Img* dog = nullptr)
{
    SepParams p;
    memset(&p, 0, sizeof(p));
    bool fast_ok = true;
    if (MODE == M_FLOAT) {
        auto symmetry = [](const float* k, int n) {
            bool sy = true, as = true;
            for (int i = 0; i < n; i++) { if (k[i] != k[n - 1 - i]) sy = false; if (k[i] != -k[n - 1 - i]) as = false; }
            return sy ? 1 : as ? 2 : 0;
        };
        if ((ny & 1) && ay == ny / 2) p.col_mode = symmetry(ky, ny);
        if (sizeof(ST) == 4 && (nx == 3 || nx == 5) && ax == nx / 2) p.row_small = symmetry(kx, nx);
        // the fast kernel implements the (anti)symmetric column order only, and the small-row order only in the 3/5 buckets
        fast_ok = p.col_mode != 0 && (!p.row_small || (nx <= 5 && ny <= 5));
    }
    if (dog) { p.dog = *dog; p.has_dog = 1; }
    p.delta = delta; p.delta_i = delta_i; p.border = border; p.cn = cn; p.even_limit = even_limit;
    bool centred = (nx & 1) && (ny & 1) && ax == nx / 2 && ay == ny / 2;
    int kb = centred ? fast_bucket(nx > ny ? nx : ny) : 0;
    if (cn == 1 && kb && fast_ok) {
        int ox = (kb - nx) / 2, oy = (kb - ny) / 2;
        for (int i = 0; i < nx; i++) p.t.kx[ox + i] = kx[i];
        for (int i = 0; i < ny; i++) p.t.ky[oy + i] = ky[i];
        p.t.nx = p.t.ny = kb; p.t.ax = p.t.ay = kb / 2;
        p.px = ox; p.py = oy;
        return launch_fast_k<ST, DT, MODE>(kb, s, d, p, st);
    }
    if (nx > 33 || ny > 33) return B200CV_NOT_IMPLEMENTED;
    for (int i = 0; i < nx; i++) p.t.kx[i] = kx[i];
    for (int i = 0; i < ny; i++) p.t.ky[i] = ky[i];
    p.t.nx = nx; p.t.ny = ny; p.t.ax = ax; p.t.ay = ay;
    return launch_generic<ST, DT, MODE>(s, d, p, st);
}

// kernel classification (reference: getKernelType, filter.dispatch.cpp:225-259)
enum { K_SYMM = 1, K_ASYMM = 2, K_SMOOTH = 4, K_INTEGER = 8 };
static int kernel_type(const float* k, int n, int anchor)
{
    int type = K_SMOOTH | K_INTEGER;
    if (anchor * 2 + 1 == n) type |= K_SYMM | K_ASYMM;
    double sum = 0;
    for (int i = 0; i < n; i++) {
        double a = k[i], b = k[n - 1 - i];
        if (a != b) type &= ~K_SYMM;
        if (a != -b) type &= ~K_ASYMM;
        if (a < 0) type &= ~K_SMOOTH;
        if (a != (double)(int)lrint(a)) type &= ~K_INTEGER;
        sum += a;
    }
    if (fabs(sum - 1) > 1.1920928955078125e-07 * (fabs(sum) + 1)) type &= ~K_SMOOTH;
    return type;
}

// createBitExactKernel_32S (filter.dispatch.cpp:288-303)
static bool bit_exact_kernel(const float* k, int n, int bits, std::vector<float>& out)
{
    out.resize(n);
    const double eps = 10 * 1.1920928955078125e-07 * (1 << bits);
    for (int i = 0; i < n; i++) {
        double a = (double)k[i] * (1 << bits);
        int v = (int)lrint(a);
        if (fabs(a - v) > eps) return false;
        out[i] = (float)v;
    }
    return true;
}

int sep_filter_impl(const b200cvMat* src, const b200cvMat* dst, const float* kx, int nx, const float* ky, int ny,
                    int ax, int ay, double delta, int border, void* stream, const b200cvMat* dog)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->cols == dst->cols && src->rows == dst->rows, "src/dst size mismatch");
    B200_REQUIRE(B200CV_CN(src->type) == B200CV_CN(dst->type), "src/dst channel mismatch");
    B200_REQUIRE(kx && ky && nx > 0 && ny > 0, "bad kernels");
    B200_REQUIRE(src->data != dst->data, "in-place filtering is not supported: pass distinct buffers");
    border &= ~B200CV_BORDER_ISOLATED;
    if (border < 0 || border > B200CV_BORDER_REFLECT_101) return B200CV_NOT_IMPLEMENTED;
    if (ax < 0) ax = nx / 2;
    if (ay < 0) ay = ny / 2;
    B200_REQUIRE(ax < nx && ay < ny, "anchor outside kernel");
    const int sdepth = B200CV_DEPTH(src->type), ddepth = B200CV_DEPTH(dst->type), cn = B200CV_CN(src->type);
    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    cudaStream_t st = as_stream(stream);

    if (sdepth == B200CV_8U && (ddepth == B200CV_8U || ddepth == B200CV_16S)) {
        int rtype = kernel_type(kx, nx, ax), ctype = kernel_type(ky, ny, ay);
        bool smooth8 = ddepth == B200CV_8U && rtype == (K_SMOOTH | K_SYMM) && ctype == (K_SMOOTH | K_SYMM);
        bool int16 = ddepth == B200CV_16S && (rtype & (K_SYMM | K_ASYMM)) && (ctype & (K_SYMM | K_ASYMM)) && (rtype & ctype & K_INTEGER);
        if (smooth8 || int16) {
            int bits = ddepth == B200CV_8U ? 8 : 0;
            std::vector<float> ikx, iky;
            if (bit_exact_kernel(kx, nx, bits, ikx) && bit_exact_kernel(ky, ny, bits, iky)) {
                double sx = 0, sy = 0;
                for (float v : ikx) sx += fabs(v);
                for (float v : iky) sy += fabs(v);
                if (sx * sy * 255.0 < 16777216.0) {     // every partial sum exact in fp32
                    long long di = llrint(delta * (double)(1 << (2 * bits)));
                    if (di > INT32_MAX) di = INT32_MAX;
                    if (di < INT32_MIN) di = INT32_MIN;
                    const int even_limit = ny > 1 ? ((s.cols * cn) / 16) * 16 : 0;
                    if (ddepth == B200CV_8U && di == 0 && ax == nx / 2 && ay == ny / 2 && ny > 1) {   // TMA + IDP fast path (gauss_u8.cu)
                        int64_t qx[32], qy[32];
                        if (nx <= 31 && ny <= 31) {
                            for (int i = 0; i < nx; i++) qx[i] = (int64_t)ikx[i];
                            for (int i = 0; i < ny; i++) qy[i] = (int64_t)iky[i];
                            int frc = gauss_u8_fast(s, d, cn, qx, nx, qy, ny, border, st, 1, even_limit);
                            if (frc != B200CV_NOT_IMPLEMENTED) return frc;
                        }
                    }
                    if (ddepth == B200CV_8U)
                        return sep_dispatch<uchar, uchar, M_FIXED16>(s, d, cn, ikx.data(), nx, iky.data(), ny, ax, ay, 0.f, (int)di, border, st,
                                                                     even_limit);
                    return sep_dispatch<uchar, short, M_INT>(s, d, cn, ikx.data(), nx, iky.data(), ny, ax, ay, 0.f, (int)di, border, st);
                }
            }
        }
    }
    float fd = (float)delta;
    if (sdepth == B200CV_8U && ddepth == B200CV_8U && cn == 1 && ax == nx / 2 && ay == ny / 2) {     // TMA fast path (sep_f32.cu); declines what it cannot do
        int frc = sep_u8_float_fast(s, d, kx, nx, ky, ny, fd, border, st);
        if (frc != B200CV_NOT_IMPLEMENTED) return frc;
    }
    if (sdepth == B200CV_8U && ddepth == B200CV_8U) return sep_dispatch<uchar, uchar, M_FLOAT>(s, d, cn, kx, nx, ky, ny, ax, ay, fd, 0, border, st);
    if (sdepth == B200CV_8U && ddepth == B200CV_16S) return sep_dispatch<uchar, short, M_FLOAT>(s, d, cn, kx, nx, ky, ny, ax, ay, fd, 0, border, st);
    if (sdepth == B200CV_8U && ddepth == B200CV_32F) return sep_dispatch<uchar, float, M_FLOAT>(s, d, cn, kx, nx, ky, ny, ax, ay, fd, 0, border, st);
    if (sdepth == B200CV_32F && ddepth == B200CV_32F) {
        Img g;
        if (dog) { g = make_img(dog); B200_REQUIRE(g.frames == s.frames && dog->cols == src->cols && dog->rows == src->rows, "dog shape mismatch"); }
        if (cn == 1 && ax == nx / 2 && ay == ny / 2) {     // TMA fast path (sep_f32.cu); declines what it cannot do
            int frc = sep_f32_fast(s, d, kx, nx, ky, ny, fd, border, dog ? &g : nullptr, st);
            if (frc != B200CV_NOT_IMPLEMENTED) return frc;
        }
        return sep_dispatch<float, float, M_FLOAT>(s, d, cn, kx, nx, ky, ny, ax, ay, fd, 0, border, st, 0, dog ? &g : nullptr);
    }
    if (dog) return B200CV_NOT_IMPLEMENTED;
    return B200CV_NOT_IMPLEMENTED;
}

int copy_impl(const b200cvMat* src, const b200cvMat* dst, void* stream)
{
    size_t wb = (size_t)src->cols * elem_size(src->type);
    int frames = src->frames > 1 ? src->frames : 1;
    for (int f = 0; f < frames; f++)
        B200_CUDA(cudaMemcpy2DAsync((char*)dst->data + (size_t)f * dst->frame_step, dst->step,
                                    (const char*)src->data + (size_t)f * src->frame_step, src->step, wb, src->rows,
                                    cudaMemcpyDeviceToDevice, as_stream(stream)));
    return B200CV_OK;
}

// Sobel taps (reference behaviour: getSobelKernels, modules/imgproc/src/deriv.cpp:96-160): the order-d derivative
// kernel of size n is the binomial smoother (1+z)^(n-d-1) times the difference operator (z-1)^d, as polynomial
// coefficients in z; built here by repeated 2-tap polynomial multiplication.
void sobel_kernel_1d(int ksize, int order, std::vector<float>& out)
{
    std::vector<long long> poly(1, 1);
    auto mul2 = [&](long long c0, long long c1) {     // poly *= (c0 + c1*z)
        std::vector<long long> r(poly.size() + 1, 0);
        for (size_t i = 0; i < poly.size(); i++) { r[i] += poly[i] * c0; r[i + 1] += poly[i] * c1; }
        poly.swap(r);
    };
    if (ksize > 1) {
        for (int i = 0; i < ksize - order - 1; i++) mul2(1, 1);
        for (int i = 0; i < order; i++) mul2(-1, 1);
    }
    out.resize(poly.size());
    for (size_t i = 0; i < poly.size(); i++) out[i] = (float)poly[i];
}

int sobel_taps(int dx, int dy, int ksize, double scale, std::vector<float>& kx, std::vector<float>& ky)
{
    // cv::Sobel: ksize 1 with a derivative uses 3 taps in that direction (deriv.cpp:116-121)
    if (ksize == -1) {   // Scharr
        if (dx + dy != 1) return B200CV_ERR_BAD_ARG;
        static const float d[] = {-1, 0, 1}, sm[] = {3, 10, 3};
        kx.assign(dx ? d : sm, (dx ? d : sm) + 3);
        ky.assign(dy ? d : sm, (dy ? d : sm) + 3);
    } else {
        if (ksize != 1 && ksize != 3 && ksize != 5 && ksize != 7) return B200CV_NOT_IMPLEMENTED;
        int ksx = ksize, ksy = ksize;
        if (ksx == 1 && dx > 0) ksx = 3;
        if (ksy == 1 && dy > 0) ksy = 3;
        if (dx >= ksx && ksx > 1) return B200CV_ERR_BAD_ARG;
        if (dy >= ksy && ksy > 1) return B200CV_ERR_BAD_ARG;
        sobel_kernel_1d(ksx, dx, kx);
        sobel_kernel_1d(ksy, dy, ky);
    }
    if (scale != 1) {
        // the scale goes into the smoothing kernel, converted to float (deriv.cpp:431-439)
        // (Mat *= double on a CV_32F kernel multiplies in float)
        std::vector<float>& k = dx == 0 ? kx : ky;
        const float fs = (float)scale;
        for (float& v : k) v = v * fs;
    }
    return B200CV_OK;
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_sep_filter2d(const b200cvMat* src, const b200cvMat* dst, const float* kx, int kx_len, const float* ky,
                                   int ky_len, int anchor_x, int anchor_y, double delta, int border, void* stream)
{
    return sep_filter_impl(src, dst, kx, kx_len, ky, ky_len, anchor_x, anchor_y, delta, border, stream, nullptr);
}

extern "C" int b200cv_sobel(const b200cvMat* src, const b200cvMat* dst, int dx, int dy, int ksize, double scale, double delta,
                            int border, void* stream)
{
    std::vector<float> kx, ky;
    int rc = sobel_taps(dx, dy, ksize, scale, kx, ky);
    if (rc) return rc;
    return sep_filter_impl(src, dst, kx.data(), (int)kx.size(), ky.data(), (int)ky.size(), -1, -1, delta, border, stream, nullptr);
}

extern "C" int b200cv_get_gaussian_kernel(int n, double sigma, double* out)
{
    B200_REQUIRE(n > 0 && out, "bad arguments");
    std::vector<double> k;
    gaussian_kernel_bitexact(n, sigma, k);
    for (int i = 0; i < n; i++) out[i] = k[i];
    return B200CV_OK;
}

extern "C" int b200cv_get_gaussian_kernel_fixed8(int n, double sigma, uint16_t* out)
{
    B200_REQUIRE(n > 0 && (n & 1) && out, "bad arguments");
    std::vector<int64_t> k;
    gaussian_kernel_fixed(n, sigma, 8, k);
    for (int i = 0; i < n; i++) out[i] = (uint16_t)k[i];
    return B200CV_OK;
}

extern "C" int b200cv_get_gaussian_kernel_fixed(int n, double sigma, int bits, uint32_t* out)
{
    B200_REQUIRE(n > 0 && (n & 1) && out && (bits == 8 || bits == 16), "bad arguments");
    std::vector<int64_t> k;
    gaussian_kernel_fixed(n, sigma, bits, k);
    for (int i = 0; i < n; i++) out[i] = (uint32_t)k[i];
    return B200CV_OK;
}

// cv::GaussianBlur (smooth.dispatch.cpp:609-826)
namespace b200cv {
int gaussian_blur_impl(const b200cvMat* src, const b200cvMat* dst, int kw, int kh, double sigma1, double sigma2, int border, void* stream,
                       const b200cvMat* dog);
}

extern "C" int b200cv_gaussian_blur(const b200cvMat* src, const b200cvMat* dst, int kw, int kh, double sigma1, double sigma2,
                                    int border, void* stream)
{
    return gaussian_blur_impl(src, dst, kw, kh, sigma1, sigma2, border, stream, nullptr);
}

int b200cv::gaussian_blur_impl(const b200cvMat* src, const b200cvMat* dst, int kw, int kh, double sigma1, double sigma2, int border,
                               void* stream, const b200cvMat* dog)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->type == dst->type, "GaussianBlur: dst type must equal src type");
    const int depth = B200CV_DEPTH(src->type);
    if (depth != B200CV_8U && depth != B200CV_32F && depth != B200CV_16U) return B200CV_NOT_IMPLEMENTED;
    int b = border & ~B200CV_BORDER_ISOLATED;
    if (b != B200CV_BORDER_CONSTANT) {           // :624-631
        if (src->rows == 1) kh = 1;
        if (src->cols == 1) kw = 1;
    }
    if (kw == 1 && kh == 1) { if (dog) return B200CV_NOT_IMPLEMENTED; return copy_impl(src, dst, stream); }
    if (sigma2 <= 0) sigma2 = sigma1;
    // createGaussianKernels (:280-304)
    if (kw <= 0 && sigma1 > 0) kw = gaussian_auto_ksize(sigma1, depth == B200CV_8U);
    if (kh <= 0 && sigma2 > 0) kh = gaussian_auto_ksize(sigma2, depth == B200CV_8U);
    B200_REQUIRE(kw > 0 && (kw & 1) && kh > 0 && (kh & 1), "GaussianBlur: ksize must be positive and odd");
    sigma1 = sigma1 > 0 ? sigma1 : 0;
    sigma2 = sigma2 > 0 ? sigma2 : 0;
    std::vector<float> kx(kw), ky(kh);
    if (depth == B200CV_16U) {       // 16.16 fixed point, bit-exact (gauss_u16.cu)
        if (dog) return B200CV_NOT_IMPLEMENTED;
        std::vector<int64_t> fx, fy;
        gaussian_kernel_fixed(kw, sigma1, 16, fx);
        gaussian_kernel_fixed(kh, sigma2, 16, fy);
        Img s = make_img(src), d = make_img(dst);
        B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
        B200_REQUIRE(src->data != dst->data, "in-place filtering is not supported: pass distinct buffers");
        B200_REQUIRE(src->cols == dst->cols && src->rows == dst->rows, "src/dst size mismatch");
        if (b < 0 || b > B200CV_BORDER_REFLECT_101) return B200CV_NOT_IMPLEMENTED;
        std::vector<long long> lx(fx.begin(), fx.end()), ly(fy.begin(), fy.end());
        return gauss_u16_impl(s, d, B200CV_CN(src->type), lx.data(), kw, ly.data(), kh, b, as_stream(stream));
    }
    if (depth == B200CV_8U) {
        if (dog) return B200CV_NOT_IMPLEMENTED;
        std::vector<int64_t> fx, fy;
        gaussian_kernel_fixed(kw, sigma1, 8, fx);
        if (kh == kw && fabs(sigma1 - sigma2) < 2.220446049250313e-16) fy = fx;
        else gaussian_kernel_fixed(kh, sigma2, 8, fy);
        for (int i = 0; i < kw; i++) kx[i] = (float)fx[i];
        for (int i = 0; i < kh; i++) ky[i] = (float)fy[i];
        Img s = make_img(src), d = make_img(dst);
        B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
        B200_REQUIRE(src->data != dst->data, "in-place filtering is not supported: pass distinct buffers");
        B200_REQUIRE(src->cols == dst->cols && src->rows == dst->rows, "src/dst size mismatch");
        if (b < 0 || b > B200CV_BORDER_REFLECT_101) return B200CV_NOT_IMPLEMENTED;
        {      // TMA + IDP fast path (gauss_u8.cu); declines what it cannot do
            int frc = gauss_u8_fast(s, d, B200CV_CN(src->type), fx.data(), kw, fy.data(), kh, b, as_stream(stream));
            if (frc != B200CV_NOT_IMPLEMENTED) return frc;
        }
        return sep_dispatch<uchar, uchar, M_FIXED16>(s, d, B200CV_CN(src->type), kx.data(), kw, ky.data(), kh, kw / 2, kh / 2,
                                                     0.f, 0, b, as_stream(stream));
    }
    std::vector<double> dx, dy;
    gaussian_kernel_bitexact(kw, sigma1, dx);
    if (kh == kw && fabs(sigma1 - sigma2) < 2.220446049250313e-16) dy = dx;
    else gaussian_kernel_bitexact(kh, sigma2, dy);
    for (int i = 0; i < kw; i++) kx[i] = (float)dx[i];
    for (int i = 0; i < kh; i++) ky[i] = (float)dy[i];
    return sep_filter_impl(src, dst, kx.data(), kw, ky.data(), kh, kw / 2, kh / 2, 0.0, b, stream, dog);
}
