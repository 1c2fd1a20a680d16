// boxfilter.cu -- cv::boxFilter / cv::blur (the unweighted member of the separable-filter family).
//
// Reference arithmetic (box_filter.simd.hpp), reproduced per destination element:
//   8U -> 8U, kw*kh <= 256 ... 16-bit sums, integer divide of ColumnSum<ushort,uchar> (:430-600):
//                              d = cvRound(1/scale); (s + divDelta) * divScale >> 23                                   bit-exact
//   8U -> 8U, larger ......... int sums; SIMD body cvRound(float(s) * float(scale)), scalar remainder (last w*cn mod 8
//                              elements) cvRound(double(s) * scale)   (ColumnSum<int,uchar> :275-428)                bit-exact
//   8U -> 32F ................ int sums; body float(s) * float(scale), remainder (w*cn mod 4) float(double(s) * scale)  bit-exact
//   32F -> 32F ............... double sums, float(s * scale).  The reference slides its sums along the row and down the whole
//                              image; here every window is summed on its own.  Both are exact (and equal) unless a double
//                              addition rounds, i.e. the window spans > 2^29 in magnitude.
// 8U -> 8U with odd sizes <= 31 around the centre runs on the TMA + IDP4A/IDP2A kernel of GaussianBlur (gauss_u8.cu) with all taps 1
// and the epilogues above; everything else on the kernel of this file:
// one CTA = 128 destination elements x 32 rows: horizontal sums of the 32 + kh - 1 source rows of the tile go to shared memory
// (taps through a per-CTA border table), then each thread slides one column down 16 rows.
#include <stdlib.h>
#include <string.h>
#include "common.cuh"

namespace b200cv {

namespace {

enum { BX_TW = 128, BX_TH = 32, BX_THREADS = 256 };
enum { BX_U16 = 0, BX_INT_U8 = 1, BX_INT_F32 = 2, BX_F64_F32 = 3 };

struct BoxParams {
    int kw, kh, ax, ay, border, cn;
    int have_scale, div_scale, div_delta, tail_from, pack4;
    float scale_f;
    double scale;
};

template <int MODE, typename WT, typename DT>
__device__ __forceinline__ DT box_out(WT s, int e, const BoxParams& p)
{
    if constexpr (MODE == BX_U16) {
        return p.have_scale ? (uchar)(((unsigned)(s + p.div_delta) * (unsigned)p.div_scale) >> 23) : (uchar)min(s, 255);
    } else if constexpr (MODE == BX_INT_U8) {
        if (!p.have_scale) return (uchar)min(s, 255);
        const int r = e < p.tail_from ? __float2int_rn(__fmul_rn(__int2float_rn(s), p.scale_f)) : __double2int_rn(__dmul_rn((double)s, p.scale));
        return (uchar)min(max(r, 0), 255);
    } else if constexpr (MODE == BX_INT_F32) {
        if (!p.have_scale) return __int2float_rn(s);
        return e < p.tail_from ? __fmul_rn(__int2float_rn(s), p.scale_f) : __double2float_rn(__dmul_rn((double)s, p.scale));
    } else {
        return p.have_scale ? __double2float_rn(__dmul_rn(s, p.scale)) : __double2float_rn(s);
    }
}

template <typename ST, typename WT, typename DT, int MODE>
__global__ void __launch_bounds__(BX_THREADS) box_filter_kernel(Img src, Img dst, BoxParams p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WT* hs = (WT*)smem_raw;                                              // [(BX_TH + kh - 1)][BX_TW] horizontal sums
    int* xtab = (int*)(hs + (size_t)(BX_TH + p.kh - 1) * BX_TW);          // source element of tap position j, -1 = constant border
    const int t = threadIdx.x, f = blockIdx.z;
    const int e0 = blockIdx.x * BX_TW, y0 = blockIdx.y * BX_TH;
    const int cn = p.cn, wn = src.cols * cn;
    const int ntab = BX_TW + (p.kw - 1) * cn;
    for (int j = t; j < ntab; j += BX_THREADS) {
        const int g = e0 - p.ax * cn + j;
        const int px = g >= 0 ? g / cn : -((-g + cn - 1) / cn);
        const int sx = border_interpolate(px, src.cols, p.border);
        xtab[j] = sx < 0 ? -1 : sx * cn + (g - px * cn);
    }
    __syncthreads();
    const int nrows = BX_TH + p.kh - 1;
    for (int idx = t; idx < nrows * BX_TW; idx += BX_THREADS) {
        const int r = idx / BX_TW, i = idx - r * BX_TW;
        const int sy = border_interpolate(y0 - p.ay + r, src.rows, p.border);
        WT s = 0;
        if (sy >= 0 && e0 + i < wn) {
            const ST* row = src.row<ST>(f, sy);
            for (int k = 0; k < p.kw; k++) {
                const int sx = xtab[i + k * cn];
                if (sx >= 0) s += (WT)__ldg(row + sx);
            }
        }
        hs[idx] = s;
    }
    __syncthreads();
    const int i = t & (BX_TW - 1), seg = t / BX_TW;
    const int e = e0 + i;
    const int r0 = seg * (BX_TH / 2);
    WT sum = 0;
    for (int k = 0; k < p.kh - 1; k++) sum += hs[(r0 + k) * BX_TW + i];
#pragma unroll 4
    for (int r = r0; r < r0 + BX_TH / 2; r++) {
        const WT s0 = sum + hs[(r + p.kh - 1) * BX_TW + i];
        sum = s0 - hs[r * BX_TW + i];
        const int y = y0 + r;
        const DT v = box_out<MODE, WT, DT>(s0, e, p);
        if constexpr (sizeof(DT) == 1) {
            if (p.pack4) {                                                // whole warp takes the same branch (pack4, y are uniform)
                unsigned w = v;
                w |= __shfl_down_sync(0xffffffffu, w, 1) << 8;
                w |= __shfl_down_sync(0xffffffffu, w, 2) << 16;
                if (y < dst.rows && (i & 3) == 0) {
                    if (e + 3 < wn) *(unsigned*)(dst.row<uchar>(f, y) + e) = w;
                    else for (int q = 0; q < 4 && e + q < wn; q++) dst.row<uchar>(f, y)[e + q] = (uchar)(w >> (8 * q));
                }
                continue;
            }
        }
        if (y < dst.rows && e < wn) dst.row<DT>(f, y)[e] = v;
    }
}

template <typename ST, typename WT, typename DT, int MODE>
int box_launch(const Img& s, const Img& d, const BoxParams& p, cudaStream_t st)
{
    const size_t smem = (size_t)(BX_TH + p.kh - 1) * BX_TW * sizeof(WT) + (size_t)(BX_TW + (p.kw - 1) * p.cn) * sizeof(int);
    if (smem > 200 * 1024) return B200CV_NOT_IMPLEMENTED;
    auto kern = box_filter_kernel<ST, WT, DT, MODE>;
    if (smem > 48 * 1024) B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(div_up((unsigned)(s.cols * p.cn), BX_TW), div_up((unsigned)s.rows, BX_TH), (unsigned)s.frames);
    if (grid.y >= 65536 || grid.z >= 65536) return B200CV_NOT_IMPLEMENTED;
    kern<<<grid, BX_THREADS, smem, st>>>(s, d, p);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_box_filter(const b200cvMat* src, const b200cvMat* dst, int ksize_w, int ksize_h, int anchor_x, int anchor_y,
                                 int normalize, int border, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->cols == dst->cols && src->rows == dst->rows, "boxFilter: dst size must equal src size");
    B200_REQUIRE(B200CV_CN(src->type) == B200CV_CN(dst->type), "boxFilter: channel count mismatch");
    B200_REQUIRE(src->data != dst->data, "boxFilter: in-place is not supported");
    B200_REQUIRE(ksize_w > 0 && ksize_h > 0, "boxFilter: ksize must be positive");
    if (anchor_x < 0) anchor_x = ksize_w / 2;
    if (anchor_y < 0) anchor_y = ksize_h / 2;
    B200_REQUIRE(anchor_x < ksize_w && anchor_y < ksize_h, "boxFilter: anchor outside the kernel");
    const int sdepth = B200CV_DEPTH(src->type), ddepth = B200CV_DEPTH(dst->type), cn = B200CV_CN(src->type);
    border &= ~B200CV_BORDER_ISOLATED;
    if (border < 0 || border > B200CV_BORDER_REFLECT_101 || border == B200CV_BORDER_WRAP) return B200CV_NOT_IMPLEMENTED;
    if (cn < 1 || cn > 4 || ksize_w > 128 || ksize_h > 128) return B200CV_NOT_IMPLEMENTED;
    const bool u8u8 = sdepth == B200CV_8U && ddepth == B200CV_8U, u8f = sdepth == B200CV_8U && ddepth == B200CV_32F;
    const bool ff = sdepth == B200CV_32F && ddepth == B200CV_32F;
    if (!u8u8 && !u8f && !ff) return B200CV_NOT_IMPLEMENTED;
    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    BoxParams p;
    p.kw = ksize_w; p.kh = ksize_h; p.ax = anchor_x; p.ay = anchor_y; p.border = border; p.cn = cn;
    p.scale = normalize ? 1. / ((double)ksize_w * ksize_h) : 1.;
    p.scale_f = (float)p.scale;
    p.have_scale = p.scale != 1;
    p.div_scale = 1; p.div_delta = 0;
    const int wn = src->cols * cn;
    p.tail_from = wn - wn % (u8u8 ? 8 : 4);
    p.pack4 = ddepth == B200CV_8U && ((size_t)dst->data % 4 == 0) && dst->step % 4 == 0 && (d.frames == 1 || dst->frame_step % 4 == 0);
    cudaStream_t st = as_stream(stream);
    const bool u16sums = u8u8 && ksize_w * ksize_h <= 256;
    if (u16sums && p.have_scale) {            // ColumnSum<ushort,uchar> constructor, box_filter.simd.hpp:435-455
        const int dv = (int)nearbyint(1. / p.scale);
        double sf = (double)(1 << 23) / dv;
        p.div_scale = (int)floor(sf);
        sf -= p.div_scale;
        p.div_delta = dv / 2;
        if (sf < 0.5) p.div_delta++; else p.div_scale++;
    }
    // 8U -> 8U, odd sizes up to 31 around the centre: the TMA + IDP4A/IDP2A kernel of GaussianBlur with all taps 1 and a box epilogue
    const char* path = getenv("B200CV_BOX_PATH");                       // test hook: "generic" keeps every call on the kernel of this file
    if (u8u8 && (ksize_w & 1) && (ksize_h & 1) && anchor_x == ksize_w / 2 && anchor_y == ksize_h / 2 && !(path && !strcmp(path, "generic"))) {
        int64_t ones[32];
        for (int i = 0; i < 32; i++) ones[i] = 1;
        GU8Box b;
        b.have_scale = p.have_scale; b.tail_from = p.tail_from; b.div_scale = (unsigned)p.div_scale; b.div_delta = (unsigned)p.div_delta;
        b.scale_f = p.scale_f; b.scale = p.scale;
        rc = gauss_u8_fast(s, d, cn, ones, ksize_w, ones, ksize_h, border, st, u16sums ? 2 : 3, 0, &b);
        if (rc != B200CV_NOT_IMPLEMENTED) return rc;
    }
    if (u16sums) return box_launch<uchar, int, uchar, BX_U16>(s, d, p, st);
    if (u8u8) return box_launch<uchar, int, uchar, BX_INT_U8>(s, d, p, st);
    if (u8f) return box_launch<uchar, int, float, BX_INT_F32>(s, d, p, st);
    return box_launch<float, double, float, BX_F64_F32>(s, d, p, st);
}
