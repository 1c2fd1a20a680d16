// laplacian.cu -- cv::Laplacian (reference: modules/imgproc/src/deriv.cpp:787-876).
//
// ksize 1 / 3: the reference runs filter2D with a 3x3 float kernel whose taps are multiplied by (float)scale, and so does this file:
//   it builds that kernel and calls the filter2D dispatch (filter2d.cu).
// ksize 5..31 (odd): with kd, ks = getSobelKernels(2, 0, ksize) the reference computes
//   d2x = sepFilter(row kd, column ks), d2y = sepFilter(row ks, column kd)   into the working depth W (createSeparableLinearFilter)
//   d2x += d2y                                                              in W, saturating for 16S
//   dst = d2x.convertTo(ddepth, scale, delta)
// with W = 16S for an 8-bit source at ksize 5 (the integer bit-exact mode: taps and sums are integers, exact here in fp32 because every
// partial sum stays below 2^24) and W = 32F otherwise.  laplacian_kernel fuses all of it: one launch per call or batch, no intermediate
// plane in HBM.  A CTA stages a TW x TH tile plus its (ksize-1)/2 apron in shared memory (borders resolved by border_interpolate, as in
// the separable kernels), runs both row passes from it into two shared planes, then both column passes, the add and the conversion.
//
// Float operation order (the reference's AVX2 objects; oracle/port/port_laplacian.c restates the same order):
//   rows     8-bit source, or a float source at ksize >= 7: s = fma(x[i], k[i], s) from 0 in tap order, zero taps included (RowVec_*)
//            float source at ksize 5: kd = [1 0 -2 0 1] is SymmRowSmallVec_32f's special case fma(x0, -2, x-2 + x2), which never reads
//            the zero taps; ks = [1 4 6 4 1] runs the centre-out order fma(x+-2 sum, 1, fma(x0, 6, (x-1 + x1) * 4)); the last
//            (cols*cn mod 8) elements of a row come from SymmRowSmallFilter's scalar remainder (filter.simd.hpp:2508-2532, compiled
//            with contraction): pairs of kd as fma(-2, x0, x-2) + x2, an odd last element of both as k0*x0 then fma(k[j], x[j] + x[-j], s)
//   columns  both kernels are symmetric: s = fma(k[c], S[c], 0); s = fma(k[c+j], S[c+j] + S[c-j], s) (SymmColumnVec_32f)
//   convert  scale == 1 && delta == 0: saturate_cast; otherwise saturate_cast(fma(v, (float)scale, (float)delta)) (cvt_32f's v_fma)
//   saturate_cast to 8U / 16S rounds half to even and, as the reference's cvtss2si does, turns NaN and anything outside the int32
//   range into INT_MIN (an 8-bit source reaches 2^31 at large apertures)
#include <cmath>
#include <cstring>
#include <vector>
#include "common.cuh"

namespace b200cv {

void sobel_kernel_1d(int ksize, int order, std::vector<float>& out);     // sepfilter.cu: getSobelKernels' taps

struct LapParams {
    float kd[32], ks[32];
    int k, cn, border;
    int we;             // elements per row (cols * cn): where the reference's 8-lane row body ends
    int plain;          // scale == 1 && delta == 0: no multiply-add before the cast
    float a, b;         // (float)scale, (float)delta
    int TH;             // tile rows
};

constexpr int L_TW = 32;        // tile width in pixels
constexpr int L_TX = 32, L_TY = 8, L_THREADS = L_TX * L_TY;

__device__ __forceinline__ int x86_round(float v)
{
    return (v >= -2147483648.f && v < 2147483648.f) ? __float2int_rn(v) : INT_MIN;
}

template <typename DT> __device__ __forceinline__ DT lap_cast(float v);
template <> __device__ __forceinline__ uchar lap_cast<uchar>(float v) { return sat_u8(x86_round(v)); }
template <> __device__ __forceinline__ short lap_cast<short>(float v) { return sat_s16(x86_round(v)); }
template <> __device__ __forceinline__ float lap_cast<float>(float v) { return v; }

// W16: the 16S working depth (8-bit source, ksize 5).  CN: channels.  A CTA is L_TX x L_TY threads: a warp per tile row at a time.
template <typename ST, typename DT, bool W16, int CN>
__global__ void __launch_bounds__(L_THREADS, 2) laplacian_kernel(Img src, Img dst, const __grid_constant__ LapParams p)
{
    extern __shared__ __align__(16) float smem[];
    const int k = p.k, R = k / 2, TH = p.TH;
    const int rows = TH + 2 * R;
    const int in_w = (L_TW + 2 * R) * CN;
    constexpr int mid_w = L_TW * CN;
    float* s_in = smem;                         // rows x in_w
    float* s_rd = s_in + rows * in_w;           // rows x mid_w: row pass with kd
    float* s_rs = s_rd + rows * mid_w;          // rows x mid_w: row pass with ks
    const int f = blockIdx.z;
    const int x0 = blockIdx.x * L_TW, y0 = blockIdx.y * TH;
    const int tx = threadIdx.x, ty = threadIdx.y;

    for (int r = ty; r < rows; r += L_TY) {
        const int sy = border_interpolate(y0 - R + r, src.rows, p.border);
        const ST* srow = sy < 0 ? nullptr : src.row<ST>(f, sy);
        float* d = s_in + r * in_w;
        for (int e = tx; e < in_w; e += L_TX) {
            const int px = e / CN, c = e - px * CN;
            const int sx = border_interpolate(x0 - R + px, src.cols, p.border);
            d[e] = (srow == nullptr || sx < 0) ? 0.f : (float)srow[(size_t)sx * CN + c];
        }
    }
    __syncthreads();

    const int tail = p.we - (p.we & 7);
    for (int r = ty; r < rows; r += L_TY) {
        for (int e = tx; e < mid_w; e += L_TX) {
            const float* x = s_in + r * in_w + e;   // x[i * CN]: tap i of output element e
            float d, s;
            if (sizeof(ST) == 4 && k == 5) {
                const float* c0 = x + 2 * CN;
                const float s1 = __fadd_rn(c0[-CN], c0[CN]), s2 = __fadd_rn(c0[-2 * CN], c0[2 * CN]);
                const int xe = x0 * CN + e;
                if (xe >= tail + ((p.we - tail) & ~1)) {          // the last element of an odd remainder: the generic loop
                    d = fmaf(p.kd[4], s2, fmaf(p.kd[3], s1, __fmul_rn(p.kd[2], c0[0])));
                    s = fmaf(p.ks[4], s2, fmaf(p.ks[3], s1, __fmul_rn(p.ks[2], c0[0])));
                } else {
                    d = xe >= tail ? __fadd_rn(fmaf(-2.f, c0[0], c0[-2 * CN]), c0[2 * CN])     // the remainder's pairs
                                   : fmaf(c0[0], -2.f, s2);
                    s = fmaf(s2, p.ks[4], fmaf(c0[0], p.ks[2], __fmul_rn(s1, p.ks[3])));
                }
            } else {
                d = 0.f; s = 0.f;
#pragma unroll 4
                for (int i = 0; i < k; i++) {
                    const float v = x[i * CN];
                    d = fmaf(v, p.kd[i], d);
                    s = fmaf(v, p.ks[i], s);
                }
            }
            s_rd[r * mid_w + e] = d;
            s_rs[r * mid_w + e] = s;
        }
    }
    __syncthreads();

    for (int r = ty; r < TH; r += L_TY) {
        const int y = y0 + r;
        if (y >= dst.rows) break;
        DT* drow = dst.row<DT>(f, y);
        for (int e = tx; e < mid_w; e += L_TX) {
            const int xe = x0 * CN + e;
            if (xe >= dst.cols * CN) break;
            const float* cd = s_rd + (r + R) * mid_w + e;   // centre row of the kd plane
            const float* cs = s_rs + (r + R) * mid_w + e;
            float dx = fmaf(p.ks[R], cd[0], 0.f);          // d2x: column ks over the kd rows
            float dy = fmaf(p.kd[R], cs[0], 0.f);          // d2y: column kd over the ks rows
#pragma unroll 4
            for (int j = 1; j <= R; j++) {
                dx = fmaf(p.ks[R + j], __fadd_rn(cd[j * mid_w], cd[-j * mid_w]), dx);
                dy = fmaf(p.kd[R + j], __fadd_rn(cs[j * mid_w], cs[-j * mid_w]), dy);
            }
            float v;
            if constexpr (W16) v = (float)sat_s16(sat_s16((int)dx) + sat_s16((int)dy));
            else v = __fadd_rn(dx, dy);
            if (!p.plain) v = fmaf(v, p.a, p.b);
            drow[xe] = lap_cast<DT>(v);
        }
    }
}

static size_t lap_smem(int k, int cn, int TH)
{
    const int R = k / 2;
    return (size_t)(TH + 2 * R) * ((L_TW + 2 * R) * cn + 2 * L_TW * cn) * sizeof(float);
}

template <typename ST, typename DT, bool W16, int CN>
static int launch_cn(const Img& s, const Img& d, const LapParams& p, size_t smem, cudaStream_t st)
{
    auto kern = laplacian_kernel<ST, DT, W16, CN>;
    static PerDeviceFlag attr_done_pd; bool& attr_done = attr_done_pd.cur();
    if (!attr_done) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024)); attr_done = true; }
    dim3 grid(div_up((unsigned)s.cols, L_TW), div_up((unsigned)s.rows, (unsigned)p.TH), (unsigned)s.frames);
    kern<<<grid, dim3(L_TX, L_TY), smem, st>>>(s, d, p);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

template <typename ST, typename DT, bool W16>
static int launch_laplacian(const Img& s, const Img& d, LapParams& p, cudaStream_t st)
{
    p.TH = 32;
    while (p.TH > 8 && lap_smem(p.k, p.cn, p.TH) > 110 * 1024) p.TH /= 2;     // two CTAs per SM at ksize 31, 4 channels
    const size_t smem = lap_smem(p.k, p.cn, p.TH);
    switch (p.cn) {
    case 1: return launch_cn<ST, DT, W16, 1>(s, d, p, smem, st);
    case 2: return launch_cn<ST, DT, W16, 2>(s, d, p, smem, st);
    case 3: return launch_cn<ST, DT, W16, 3>(s, d, p, smem, st);
    default: return launch_cn<ST, DT, W16, 4>(s, d, p, smem, st);
    }
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_laplacian(const b200cvMat* src, const b200cvMat* dst, int ksize, double scale, double delta, int border, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(ksize >= 1 && ksize <= 31 && (ksize & 1), "Laplacian: ksize must be odd and in 1..31");
    B200_REQUIRE(src->cols == dst->cols && src->rows == dst->rows, "src/dst size mismatch");
    B200_REQUIRE(B200CV_CN(src->type) == B200CV_CN(dst->type), "src/dst channel mismatch");
    B200_REQUIRE(src->data != dst->data, "in-place filtering is not supported: pass distinct buffers");
    const int sd = B200CV_DEPTH(src->type), dd = B200CV_DEPTH(dst->type), cn = B200CV_CN(src->type);
    if (!((sd == B200CV_8U && (dd == B200CV_8U || dd == B200CV_16S || dd == B200CV_32F)) || (sd == B200CV_32F && dd == B200CV_32F)))
        return B200CV_NOT_IMPLEMENTED;
    if (cn > 4) return B200CV_NOT_IMPLEMENTED;
    border &= ~B200CV_BORDER_ISOLATED;      // a device view has no parent image to read past its edges
    if (border < 0 || border > B200CV_BORDER_REFLECT_101 || border == B200CV_BORDER_WRAP) return B200CV_NOT_IMPLEMENTED;

    if (ksize <= 3) {
        static const float K[2][9] = {{0, 1, 0, 1, -4, 1, 0, 1, 0}, {2, 0, 2, 0, -8, 0, 2, 0, 2}};
        float kern[9];
        for (int i = 0; i < 9; i++) kern[i] = scale != 1 ? K[ksize == 3][i] * (float)scale : K[ksize == 3][i];
        return b200cv_filter2d(src, dst, kern, 3, 3, -1, -1, delta, border, stream);
    }

    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    B200_REQUIRE(s.frames <= 65535, "Laplacian: at most 65535 frames per call");
    LapParams p;
    memset(&p, 0, sizeof(p));
    std::vector<float> kd, ks;
    sobel_kernel_1d(ksize, 2, kd);
    sobel_kernel_1d(ksize, 0, ks);
    for (int i = 0; i < ksize; i++) { p.kd[i] = kd[i]; p.ks[i] = ks[i]; }
    p.k = ksize; p.cn = cn; p.border = border; p.we = src->cols * cn;
    p.plain = scale == 1 && delta == 0;
    p.a = (float)scale; p.b = (float)delta;
    cudaStream_t st = as_stream(stream);
    if (sd == B200CV_8U && ksize == 5) {
        if (dd == B200CV_8U) return launch_laplacian<uchar, uchar, true>(s, d, p, st);
        if (dd == B200CV_16S) return launch_laplacian<uchar, short, true>(s, d, p, st);
        return launch_laplacian<uchar, float, true>(s, d, p, st);
    }
    if (sd == B200CV_8U) {
        if (dd == B200CV_8U) return launch_laplacian<uchar, uchar, false>(s, d, p, st);
        if (dd == B200CV_16S) return launch_laplacian<uchar, short, false>(s, d, p, st);
        return launch_laplacian<uchar, float, false>(s, d, p, st);
    }
    return launch_laplacian<float, float, false>(s, d, p, st);
}
