// filter2d.cu -- cv::filter2D: correlation with an arbitrary kh x kw float kernel.
//
// Reference arithmetic (Filter2D<ST,CastOp,VecOp>, modules/imgproc/src/filter.simd.hpp:3103-3175): per output
//   s = (float)delta; for every non-zero tap in row-major order: s = fma(k, src, s); dst = saturate_cast<DT>(s)
//   (8-bit source with a float destination: the scalar FilterNoVec object, s += round(k * src), no FMA).
// (The CPU switches to a DFT for >= 130 taps, filter.dispatch.cpp:1288; the GPU evaluates the direct sum for every
//  size, which is the more accurate of the two -- parity tolerance per modules/imgproc/test/test_filter.cpp:420-425.)
//
// A CTA stages a (TH+kh-1) x (TW+kw-1) float tile (+apron, borders per cv::borderInterpolate) in shared memory.
// Fast kernel (1 channel, centred odd kw <= 31): each thread produces 8 adjacent outputs; per kernel row it reads its
// window with 128-bit shared loads and issues 8*KB FFMAs with the taps as uniform constant-bank operands.
// Generic kernel: any channel count / anchor / kernel up to 33x33, run-time loops.
#include <cstring>
#include "common.cuh"

namespace b200cv {

int filter2d_tma(const Img& s, const Img& d, int sd, int dd, int cn, const float* k, int kw, int kh, int ax, int ay, float delta, int border, cudaStream_t st);
int filter2d_u8_tensor(const Img& s, const Img& d, int dd, const float* k, int kw, int kh, int ax, int ay, float delta, int border, cudaStream_t st);
int filter2d_f32_tensor(const Img& s, const Img& d, const float* k, int kw, int kh, int ax, int ay, float delta, int border, cudaStream_t st);   // filter2d_tc_f32.cu

struct F2DParams {
    float k[33 * 33];    // row-major, row stride = kstride
    int kw, kh, ax, ay, kstride;
    float delta;
    int border, cn;
};

constexpr int F2_TW = 128, F2_TH = 16, F2_R = 8;

template <typename ST, typename DT, int KB>
__global__ void __launch_bounds__(256) filter2d_fast_kernel(Img src, Img dst, const __grid_constant__ F2DParams p)
{
    constexpr int RB = KB / 2;
    constexpr int RP = ((RB + 3) / 4) * 4;
    constexpr int SW = F2_TW + 2 * RP;
    extern __shared__ __align__(16) float s_in[];       // (F2_TH + kh - 1) x SW
    const int in_rows = F2_TH + p.kh - 1;
    const int f = blockIdx.z, x0 = blockIdx.x * F2_TW, y0 = blockIdx.y * F2_TH;

    for (int idx = threadIdx.x; idx < in_rows * SW; idx += 256) {
        int r = idx / SW, c = idx - r * SW;
        int sy = border_interpolate(y0 - p.ay + r, src.rows, p.border);
        int sx = border_interpolate(x0 - RP + c, src.cols, p.border);
        s_in[idx] = (sy < 0 || sx < 0) ? 0.f : (float)src.row<ST>(f, sy)[sx];
    }
    __syncthreads();

    const int ty = threadIdx.x / (F2_TW / F2_R), tg = threadIdx.x % (F2_TW / F2_R);
    constexpr int LO = RP - RB, NEED = F2_R + KB - 1;
    constexpr int V0 = LO / 4, V1 = (LO + NEED - 1) / 4;
    float acc[F2_R];
#pragma unroll
    for (int o = 0; o < F2_R; o++) acc[o] = p.delta;
    for (int ky = 0; ky < p.kh; ky++) {
        const float4* vp = (const float4*)(s_in + (ty + ky) * SW + tg * F2_R);
        const float* kr = p.k + ky * KB;
#pragma unroll
        for (int w = V0; w <= V1; w++) {
            float4 q = vp[w];
            float vals[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const int e = w * 4 + b - LO;
                if (e >= 0 && e < NEED) {
#pragma unroll
                    for (int o = 0; o < F2_R; o++) {
                        const int i = e - o;
                        if (i >= 0 && i < KB) {
                            if constexpr (sizeof(ST) == 1 && sizeof(DT) == 4) acc[o] = __fadd_rn(acc[o], __fmul_rn(kr[i], vals[b]));   // scalar FilterNoVec: no FMA
                            else acc[o] = fmaf(kr[i], vals[b], acc[o]);
                        }
                    }
                }
            }
        }
    }
    const int gy = y0 + ty, gx = x0 + tg * F2_R;
    if (gy >= dst.rows) return;
    DT* dp = dst.row<DT>(f, gy) + gx;
#pragma unroll
    for (int o = 0; o < F2_R; o++)
        if (gx + o < dst.cols) dp[o] = OutCast<DT>::from(acc[o]);
}

constexpr int G2_TPX = 32, G2_TH = 8;

template <typename ST, typename DT>
__global__ void __launch_bounds__(256) filter2d_generic_kernel(Img src, Img dst, const __grid_constant__ F2DParams p)
{
    extern __shared__ __align__(16) float s_in[];
    const int cn = p.cn;
    const int tile_px = G2_TPX + p.kw - 1, in_rows = G2_TH + p.kh - 1, in_w = tile_px * cn;
    const int f = blockIdx.z, x0 = blockIdx.x * G2_TPX, y0 = blockIdx.y * G2_TH;
    for (int idx = threadIdx.x; idx < in_rows * tile_px; idx += blockDim.x) {
        int r = idx / tile_px, c = idx - r * tile_px;
        int sy = border_interpolate(y0 - p.ay + r, src.rows, p.border);
        int sx = border_interpolate(x0 - p.ax + c, src.cols, p.border);
        float* d = s_in + r * in_w + c * cn;
        if (sy < 0 || sx < 0) for (int ch = 0; ch < cn; ch++) d[ch] = 0.f;
        else {
            const ST* sp = src.row<ST>(f, sy) + (size_t)sx * cn;
            for (int ch = 0; ch < cn; ch++) d[ch] = (float)sp[ch];
        }
    }
    __syncthreads();
    const int out_w = G2_TPX * cn;
    for (int idx = threadIdx.x; idx < G2_TH * out_w; idx += blockDim.x) {
        int r = idx / out_w, e = idx - r * out_w;
        int gy = y0 + r, xe = x0 * cn + e;
        if (gy >= dst.rows || xe >= dst.cols * cn) continue;
        float acc = p.delta;
        for (int ky = 0; ky < p.kh; ky++) {
            const float* s = s_in + (r + ky) * in_w + e;
            const float* kr = p.k + ky * p.kstride;
            for (int kx = 0; kx < p.kw; kx++) {
                if constexpr (sizeof(ST) == 1 && sizeof(DT) == 4) acc = __fadd_rn(acc, __fmul_rn(kr[kx], s[kx * cn]));   // scalar FilterNoVec: no FMA
                else acc = fmaf(kr[kx], s[kx * cn], acc);
            }
        }
        dst.row<DT>(f, gy)[xe] = OutCast<DT>::from(acc);
    }
}

template <typename ST, typename DT, int KB>
static int launch_f2d_fast(const Img& s, const Img& d, const F2DParams& p, cudaStream_t st)
{
    constexpr int RP = ((KB / 2 + 3) / 4) * 4;
    size_t smem = (size_t)(F2_TH + p.kh - 1) * (F2_TW + 2 * RP) * sizeof(float);
    auto kern = filter2d_fast_kernel<ST, DT, KB>;
    static PerDeviceFlag attr_done_pd; bool& attr_done = attr_done_pd.cur();
    if (!attr_done) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024)); attr_done = true; }
    dim3 grid(div_up((unsigned)s.cols, F2_TW), div_up((unsigned)s.rows, F2_TH), (unsigned)s.frames);
    kern<<<grid, 256, smem, st>>>(s, d, p);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

template <typename ST, typename DT>
static int f2d_dispatch(const Img& s, const Img& d, int cn, const float* k, int kw, int kh, int ax, int ay, float delta, int border, cudaStream_t st)
{
    static thread_local F2DParams tp;   // ~4.4 KB: keep it off the stack
    memset(&tp, 0, sizeof(tp));
    tp.kw = kw; tp.kh = kh; tp.ax = ax; tp.ay = ay; tp.delta = delta; tp.border = border; tp.cn = cn;
    bool centred = (kw & 1) && ax == kw / 2;
    int kb = 0;
    if (cn == 1 && centred && kh <= 33) {
        static const int buckets[] = {3, 5, 7, 9, 11, 13, 15, 21, 31};
        for (int b : buckets) if (kw <= b) { kb = b; break; }
    }
    if (kb) {
        int ox = (kb - kw) / 2;
        tp.kstride = kb;
        for (int y = 0; y < kh; y++) for (int x = 0; x < kw; x++) tp.k[y * kb + ox + x] = k[y * kw + x];
        switch (kb) {
        case 3: return launch_f2d_fast<ST, DT, 3>(s, d, tp, st);
        case 5: return launch_f2d_fast<ST, DT, 5>(s, d, tp, st);
        case 7: return launch_f2d_fast<ST, DT, 7>(s, d, tp, st);
        case 9: return launch_f2d_fast<ST, DT, 9>(s, d, tp, st);
        case 11: return launch_f2d_fast<ST, DT, 11>(s, d, tp, st);
        case 13: return launch_f2d_fast<ST, DT, 13>(s, d, tp, st);
        case 15: return launch_f2d_fast<ST, DT, 15>(s, d, tp, st);
        case 21: return launch_f2d_fast<ST, DT, 21>(s, d, tp, st);
        case 31: return launch_f2d_fast<ST, DT, 31>(s, d, tp, st);
        }
    }
    if (kw > 33 || kh > 33) return B200CV_NOT_IMPLEMENTED;
    tp.kstride = kw;
    for (int i = 0; i < kw * kh; i++) tp.k[i] = k[i];
    size_t smem = (size_t)(G2_TH + kh - 1) * (G2_TPX + kw - 1) * cn * sizeof(float);
    if (smem > 100 * 1024) return B200CV_NOT_IMPLEMENTED;
    auto kern = filter2d_generic_kernel<ST, DT>;
    static PerDeviceFlag attr_done_pd; bool& attr_done = attr_done_pd.cur();
    if (!attr_done) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024)); attr_done = true; }
    dim3 grid(div_up((unsigned)s.cols, G2_TPX), div_up((unsigned)s.rows, G2_TH), (unsigned)s.frames);
    kern<<<grid, 256, smem, st>>>(s, d, tp);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_filter2d(const b200cvMat* src, const b200cvMat* dst, const float* kernel, int kw, int kh, int ax, int ay,
                               double delta, int border, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->cols == dst->cols && src->rows == dst->rows, "src/dst size mismatch");
    B200_REQUIRE(B200CV_CN(src->type) == B200CV_CN(dst->type), "src/dst channel mismatch");
    B200_REQUIRE(kernel && kw > 0 && kh > 0, "bad kernel");
    B200_REQUIRE(src->data != dst->data, "in-place filtering is not supported: pass distinct buffers");
    border &= ~B200CV_BORDER_ISOLATED;
    if (border < 0 || border > B200CV_BORDER_REFLECT_101 || border == B200CV_BORDER_WRAP) return B200CV_NOT_IMPLEMENTED;
    if (ax < 0) ax = kw / 2;
    if (ay < 0) ay = kh / 2;
    B200_REQUIRE(ax < kw && ay < kh, "anchor outside kernel");
    const int sd = B200CV_DEPTH(src->type), dd = B200CV_DEPTH(dst->type), cn = B200CV_CN(src->type);
    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    cudaStream_t st = as_stream(stream);
    float fd = (float)delta;
    const char* tc_env = getenv("B200CV_FILTER2D_TC_MIN_TAPS");          // test hook: lower / raise the tensor-core threshold
    const int tc_min_taps = tc_env ? atoi(tc_env) : 0;
    // Exactly the sizes at which the reference leaves the direct sum for a DFT (dft_filter_size, filter.dispatch.cpp:1288-1290): below
    // them the FP32 kernels reproduce the reference bit for bit (tools/f2d_exactness.py: 0 of 2 M pixels differ), from there on the
    // reference is a float DFT and the fixed-point tensor-core correlation is the more accurate of the two.
    if (sd == B200CV_8U && cn == 1 && kw * kh >= (tc_min_taps ? tc_min_taps : dd == B200CV_32F ? 50 : 130)) {
        const char* path = getenv("B200CV_FILTER2D_PATH");
        if (!(path && !strcmp(path, "direct"))) {
            rc = filter2d_u8_tensor(s, d, dd, kernel, kw, kh, ax, ay, fd, border, st);
            if (rc != B200CV_NOT_IMPLEMENTED) return rc;
        }
    }
    // float images: same switch point (the reference's DFT regime), 3 x BF16 on the tensor cores (wgmma) with FP32 accumulation (filter2d_tc_f32.cu)
    if (sd == B200CV_32F && dd == B200CV_32F && cn == 1 && kw * kh >= (tc_min_taps ? tc_min_taps : 130)) {
        const char* path = getenv("B200CV_FILTER2D_PATH");
        if (!(path && !strcmp(path, "direct"))) {
            rc = filter2d_f32_tensor(s, d, kernel, kw, kh, ax, ay, fd, border, st);
            if (rc != B200CV_NOT_IMPLEMENTED) return rc;
        }
    }
    {
        const char* path = getenv("B200CV_FILTER2D_PATH");
        if (!(path && !strcmp(path, "v1"))) {
            rc = filter2d_tma(s, d, sd, dd, cn, kernel, kw, kh, ax, ay, fd, border, st);
            if (rc != B200CV_NOT_IMPLEMENTED) return rc;
        }
    }
    if (sd == B200CV_8U && dd == B200CV_8U) return f2d_dispatch<uchar, uchar>(s, d, cn, kernel, kw, kh, ax, ay, fd, border, st);
    if (sd == B200CV_8U && dd == B200CV_16S) return f2d_dispatch<uchar, short>(s, d, cn, kernel, kw, kh, ax, ay, fd, border, st);
    if (sd == B200CV_8U && dd == B200CV_32F) return f2d_dispatch<uchar, float>(s, d, cn, kernel, kw, kh, ax, ay, fd, border, st);
    if (sd == B200CV_32F && dd == B200CV_32F) return f2d_dispatch<float, float>(s, d, cn, kernel, kw, kh, ax, ay, fd, border, st);
    return B200CV_NOT_IMPLEMENTED;
}
