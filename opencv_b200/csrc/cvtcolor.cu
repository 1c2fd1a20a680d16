// cvtcolor.cu -- cv::cvtColor for the BGR/RGB(A) <-> GRAY / YUV / YCrCb / HSV(_FULL) / BGR(A) families, 8-bit.
//
// Pure streaming op: HBM-bound (4 B/px GRAY, 6 B/px YUV/HSV).  Each thread converts 16 consecutive pixels:
// SCN 128-bit streaming loads in flight per thread, DCN 128-bit stores; rows whose base/pitch is not
// 16-byte aligned, and the last (width % 16) pixels of a row, take a byte-granular path in the same kernel.
//
// Arithmetic restated from the reference's scalar forms (bit-exact, integer):
//   RGB2Gray<uchar>     modules/imgproc/src/color_rgb.simd.hpp:660-750   (RY15/GY15/BY15, shift 15, color.simd_helpers.hpp:14-25)
//   Gray2RGB<uchar>     modules/imgproc/src/color_rgb.simd.hpp:387-470
//   RGB2YCrCb_i<uchar>  modules/imgproc/src/color_yuv.simd.hpp:397-572   (coefficients :66-92)
//   YCrCb2RGB_i<uchar>  modules/imgproc/src/color_yuv.simd.hpp:738-888
//   RGB2HSV_b           modules/imgproc/src/color_hsv.simd.hpp:47-268    (12-bit reciprocal tables :64-79)
//   HSV2RGB_b           modules/imgproc/src/color_hsv.simd.hpp:518-672   (float; SIMD body truncates, scalar tail rounds)
//   RGB2RGB<uchar>      modules/imgproc/src/color_rgb.simd.hpp:120-200
// Dispatch of `code` -> (scn, dcn, blueIdx, flags) follows modules/imgproc/src/color.cpp:208-390.
#include "common.cuh"

namespace b200cv {

#define DESCALE(x, n) (((x) + (1 << ((n)-1))) >> (n))

// ---- per-pixel functors ---------------------------------------------------------------------------------------
struct OpBGR2Gray {   // scn 3|4 -> 1
    int cb, cg, cr;
    __device__ __forceinline__ void px(const uchar* s, uchar* d) const
    {
        d[0] = (uchar)DESCALE(s[0] * cb + s[1] * cg + s[2] * cr, 15);
    }
};

struct OpGray2BGR {   // 1 -> 3|4
    __device__ __forceinline__ void px(const uchar* s, uchar* d) const
    {
        d[0] = d[1] = d[2] = s[0];
        d[3] = 255;   // only stored when DCN == 4
    }
};

// NOTE: every channel index below is a compile-time constant (template parameters): run-time indices into the
// per-pixel register arrays would demote them to local memory.
template <int SWAP, int SRC_ALPHA>
struct OpBGR2BGR {    // 3|4 -> 3|4, optional R<->B swap (cvtBGRtoBGR)
    __device__ __forceinline__ void px(const uchar* s, uchar* d) const
    {
        d[0] = s[SWAP ? 2 : 0];
        d[1] = s[1];
        d[2] = s[SWAP ? 0 : 2];
        d[3] = SRC_ALPHA ? s[3] : (uchar)255;
    }
};

template <int bidx, int yuvOrder>
struct OpBGR2YCrCb {  // 3|4 -> 3
    int c0, c1, c2, c3, c4;
    __device__ __forceinline__ void px(const uchar* s, uchar* d) const
    {
        const int delta = 128 * (1 << 14);
        int Y = DESCALE(s[0] * c0 + s[1] * c1 + s[2] * c2, 14);
        int Cr = DESCALE((s[bidx ^ 2] - Y) * c3 + delta, 14);
        int Cb = DESCALE((s[bidx] - Y) * c4 + delta, 14);
        d[0] = sat_u8(Y);
        d[1 + yuvOrder] = sat_u8(Cr);
        d[2 - yuvOrder] = sat_u8(Cb);
    }
};

template <int bidx, int yuvOrder>
struct OpYCrCb2BGR {  // 3 -> 3|4
    int c0, c1, c2, c3;
    __device__ __forceinline__ void px(const uchar* s, uchar* d) const
    {
        int Y = s[0], Cr = s[1 + yuvOrder], Cb = s[2 - yuvOrder];
        int b = Y + DESCALE((Cb - 128) * c3, 14);
        int g = Y + DESCALE((Cb - 128) * c2 + (Cr - 128) * c1, 14);
        int r = Y + DESCALE((Cr - 128) * c0, 14);
        d[bidx] = sat_u8(b);
        d[1] = sat_u8(g);
        d[bidx ^ 2] = sat_u8(r);
        d[3] = 255;
    }
};

// 12-bit reciprocal tables, computed exactly on the host once (hsv tables: color_hsv.simd.hpp:64-79)
__device__ int g_sdiv_table[256];
__device__ int g_hdiv_table180[256];
__device__ int g_hdiv_table256[256];

template <int bidx>
struct OpBGR2HSV {    // 3|4 -> 3
    int hrange;
    const int* sdiv;   // shared-memory copies
    const int* hdiv;
    __device__ __forceinline__ void px(const uchar* s, uchar* d) const
    {
        int b = s[bidx], g = s[1], r = s[bidx ^ 2];
        int v = max(b, max(g, r));
        int vmin = min(b, min(g, r));
        int diff = v - vmin;
        int vr = v == r ? -1 : 0;
        int vg = v == g ? -1 : 0;
        int sat = (diff * sdiv[v] + (1 << 11)) >> 12;
        int h = (vr & (g - b)) + (~vr & ((vg & (b - r + 2 * diff)) + ((~vg) & (r - g + 4 * diff))));
        h = (h * hdiv[diff] + (1 << 11)) >> 12;
        h += h < 0 ? hrange : 0;
        d[0] = sat_u8(h);
        d[1] = (uchar)sat;
        d[2] = (uchar)v;
    }
};

constexpr int PPT = 16;  // pixels per thread

template <int bidx>
struct OpHSV2BGR {    // 3 -> 3|4 ; float arithmetic mirroring the reference's vector body
    float hscale;
    int trunc_cols;     // pixels x < trunc_cols are truncated after scaling (vector body), the rest rounded (scalar tail)
    // Conversions are the scarce resource here (I2F/F2I/FRND issue at a quarter of the FP32 rate): bytes become floats by
    // OR-ing them into the mantissa of 2^23, floats become bytes by adding 2^23 (round-to-nearest-even = cvRound, or
    // round-toward-zero = the vector body's truncation) and taking the low mantissa byte.  All values are in [0, 255].
    __device__ __forceinline__ void px_at(const uchar* s, uchar* d, int x) const
    {
        const float two23 = 8388608.0f;
        float h = __fsub_rn(__uint_as_float(0x4B000000u | s[0]), two23);
        float sv = __fmul_rn(__fsub_rn(__uint_as_float(0x4B000000u | s[1]), two23), 1.0f / 255.0f);
        float v = __fmul_rn(__fsub_rn(__uint_as_float(0x4B000000u | s[2]), two23), 1.0f / 255.0f);
        h = __fmul_rn(h, hscale);
        const float hm = __fadd_rz(h, two23);                  // 2^23 + trunc(h), exact
        const float pre = __fsub_rn(hm, two23);
        const int ipre = (int)(__float_as_uint(hm) & 0xffu);   // h * hscale <= 8.5
        h = __fsub_rn(h, pre);
        float tab0 = v;
        float tab1 = __fmul_rn(v, __fsub_rn(1.0f, sv));
        // the reference's AVX2 unit is compiled with -mfma and GCC contracts 1 - s*h into a single fnmadd
        float tab2 = __fmul_rn(v, __fmaf_rn(-sv, h, 1.0f));
        float tab3 = __fmul_rn(v, __fmaf_rn(-sv, __fsub_rn(1.0f, h), 1.0f));
        // sector = pre - 6 * trunc(pre * (1/6.f)); pre is an integer in [0, 8]
        const int sector = ipre >= 6 ? ipre - 6 : ipre;
        // sector_data rows {b,g,r} = {1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}
        // as a two-level multiplexer on (sector & 1, sector >> 1) with two shared first-level selections
        const bool odd = sector & 1, mid = (sector >> 1) == 1, hi = (sector >> 1) == 2;
        const float X = odd ? tab0 : tab3, Y = odd ? tab2 : tab0;
        float b = hi ? Y : (mid ? X : tab1);
        float g = hi ? tab1 : (mid ? Y : X);
        float r = hi ? X : (mid ? tab1 : Y);
        b = __fmul_rn(b, 255.0f); g = __fmul_rn(g, 255.0f); r = __fmul_rn(r, 255.0f);
        uint32_t ub, ug, ur;
        if (x < trunc_cols) {      // v_trunc + saturating pack
            ub = __float_as_uint(__fadd_rz(b, two23)); ug = __float_as_uint(__fadd_rz(g, two23)); ur = __float_as_uint(__fadd_rz(r, two23));
        } else {                   // saturate_cast<uchar>(float)
            ub = __float_as_uint(__fadd_rn(b, two23)); ug = __float_as_uint(__fadd_rn(g, two23)); ur = __float_as_uint(__fadd_rn(r, two23));
        }
        d[bidx] = (uchar)ub; d[1] = (uchar)ug; d[bidx ^ 2] = (uchar)ur; d[3] = 255;
    }
};

// ---- generic streaming kernel -----------------------------------------------------------------------------------

template <int N> struct Bytes {
    uint32_t w[(N + 3) / 4];
    __device__ __forceinline__ uchar get(int i) const { return (uchar)(w[i >> 2] >> ((i & 3) * 8)); }
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int i = 0; i < (N + 3) / 4; i++) w[i] = 0;
    }
    __device__ __forceinline__ void set(int i, uchar v) { w[i >> 2] |= (uint32_t)v << ((i & 3) * 8); }
};

template <int SCN, int DCN, class Op, bool POS>
__device__ __forceinline__ void convert_px(const Op& op, const uchar* s, uchar* d, int x)
{
    if constexpr (POS) op.px_at(s, d, x);
    else op.px(s, d);
}

template <int SCN, int DCN, class Op, bool POS, bool HSV_TABLES>
__global__ void __launch_bounds__(256) cvt_kernel(Img src, Img dst, Op op, int nxblk, int vec_ok)
{
    __shared__ int s_sdiv[HSV_TABLES ? 256 : 1];
    __shared__ int s_hdiv[HSV_TABLES ? 256 : 1];
    if constexpr (HSV_TABLES) {
        s_sdiv[threadIdx.x] = g_sdiv_table[threadIdx.x];
        s_hdiv[threadIdx.x] = (op.hrange == 180 ? g_hdiv_table180 : g_hdiv_table256)[threadIdx.x];
        op.sdiv = s_sdiv;
        op.hdiv = s_hdiv;
        __syncthreads();
    }
    const int f = blockIdx.y;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned y = idx / (unsigned)nxblk;
    if (y >= (unsigned)src.rows) return;
    const int x0 = (int)(idx - y * (unsigned)nxblk) * PPT;
    const uchar* sp = src.row<uchar>(f, (int)y) + (size_t)x0 * SCN;
    uchar* dp = dst.row<uchar>(f, (int)y) + (size_t)x0 * DCN;
    const int n = min(PPT, src.cols - x0);

    // the vector path below exchanges data inside the warp when DCN >= 3: it is taken by whole warps only (a warp that holds a row's ragged last
    // item or runs past the last row goes the scalar way for all its lanes -- a few warps per image)
    const bool vec_warp = (DCN >= 3 && SCN == 1) ? __all_sync(__activemask(), vec_ok && n == PPT) && __activemask() == 0xffffffffu : (vec_ok && n == PPT);
    if (vec_warp) {
        if constexpr (POS) {
            // position-dependent ops switch behaviour at a multiple of 32 pixels: uniform over this thread's 16 pixels
            if (x0 < op.trunc_cols) op.trunc_cols = 0x7fffffff; else op.trunc_cols = 0;
        }
        uint4 in[SCN];
#pragma unroll
        for (int i = 0; i < SCN; i++) in[i] = ldg_stream((const uint4*)sp + i);
        uint4 out[DCN];
        const uchar* ib = (const uchar*)in;   // register arrays: all indices below are compile-time constants
        uchar* ob = (uchar*)out;
#pragma unroll
        for (int p = 0; p < PPT; p++) {
            uchar s[4], d[4];
#pragma unroll
            for (int c = 0; c < SCN; c++) s[c] = ib[p * SCN + c];
            convert_px<SCN, DCN, Op, POS>(op, s, d, x0 + p);
#pragma unroll
            for (int c = 0; c < DCN; c++) ob[p * DCN + c] = d[c];
        }
        if constexpr (DCN >= 3 && SCN == 1) {      // (3 -> 3 conversions gain ~1 %, and the 12 KB of shared memory cost BGR2HSV occupancy: 0.67 -> 0.64)
            // A thread's DCN vectors are 16 DCN bytes apart from its neighbour's: stored directly, every store instruction touches 32 separate
            // 16-byte pieces (half or a quarter of each sector).  When the whole warp sits in one row on the vector path its output is one
            // contiguous 512 DCN-byte run: exchange through shared memory and let store i write 32 ADJACENT vectors (full lines).
            __shared__ __align__(16) uint4 s_out[256 * DCN];
            const unsigned y0w = __shfl_sync(0xffffffffu, y, 0);
            const bool whole = __all_sync(0xffffffffu, y == y0w);                 // every lane took this branch (checked by the caller's ballot below)
            if (whole) {
                const int lane = threadIdx.x & 31, wbase = (threadIdx.x >> 5) * 32 * DCN;
#pragma unroll
                for (int i = 0; i < DCN; i++) s_out[wbase + lane * DCN + i] = out[i];
                __syncwarp();
                uint4* wp = (uint4*)(dp - (size_t)lane * PPT * DCN);              // the warp's first output byte
#pragma unroll
                for (int i = 0; i < DCN; i++) stg_stream(wp + i * 32 + lane, s_out[wbase + i * 32 + lane]);
                __syncwarp();
                return;
            }
        }
#pragma unroll
        for (int i = 0; i < DCN; i++) stg_stream((uint4*)dp + i, out[i]);
    } else {
        for (int p = 0; p < n; p++) {
            uchar s[4], d[4];
#pragma unroll
            for (int c = 0; c < SCN; c++) s[c] = sp[p * SCN + c];
            convert_px<SCN, DCN, Op, POS>(op, s, d, x0 + p);
#pragma unroll
            for (int c = 0; c < DCN; c++) dp[p * DCN + c] = d[c];
        }
    }
}

template <int SCN, int DCN, class Op, bool POS = false, bool HSV_TABLES = false>
static int launch_cvt(const Img& src, const Img& dst, const Op& op, cudaStream_t st)
{
    int nxblk = (int)div_up((unsigned)src.cols, PPT);
    unsigned long long total = (unsigned long long)nxblk * (unsigned)src.rows;
    if (total > 0x7fffffffULL) { set_error("image too large"); return B200CV_ERR_BAD_ARG; }
    int vec_ok = (((uintptr_t)src.data | src.step | src.fstep | (uintptr_t)dst.data | dst.step | dst.fstep) & 15) == 0;
    dim3 grid(div_up((unsigned)total, 256), (unsigned)src.frames);
    cvt_kernel<SCN, DCN, Op, POS, HSV_TABLES><<<grid, 256, 0, st>>>(src, dst, op, nxblk, vec_ok);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

static int ensure_hsv_tables()
{
    static PerDeviceFlag done_pd; bool& done = done_pd.cur();     // benign race: every thread writes identical tables
    if (done) return B200CV_OK;
    int sdiv[256], h180[256], h256[256];
    sdiv[0] = h180[0] = h256[0] = 0;
    for (int i = 1; i < 256; i++) {
        sdiv[i] = (int)lrint((255 << 12) / (1. * i));
        h180[i] = (int)lrint((180 << 12) / (6. * i));
        h256[i] = (int)lrint((256 << 12) / (6. * i));
    }
    B200_CUDA(cudaMemcpyToSymbol(g_sdiv_table, sdiv, sizeof(sdiv)));
    B200_CUDA(cudaMemcpyToSymbol(g_hdiv_table180, h180, sizeof(h180)));
    B200_CUDA(cudaMemcpyToSymbol(g_hdiv_table256, h256, sizeof(h256)));
    done = true;
    return B200CV_OK;
}

}  // namespace b200cv

using namespace b200cv;

// number of leading pixels per row that the reference converts in its 32-pixel AVX2 vector body (HSV2RGB_b)
static inline int hsv_trunc_cols(int width) { return width >= 32 ? (width / 32) * 32 : 0; }

extern "C" int b200cv_cvt_color_two_plane(const b200cvMat* ysrc, const b200cvMat* uvsrc, const b200cvMat* dst, int code, void* stream)
{
    int rc;
    if ((rc = check_mat(ysrc, "src1")) || (rc = check_mat(uvsrc, "src2")) || (rc = check_mat(dst, "dst"))) return rc;
    if (B200CV_DEPTH(ysrc->type) != B200CV_8U || B200CV_DEPTH(uvsrc->type) != B200CV_8U || B200CV_DEPTH(dst->type) != B200CV_8U) return B200CV_NOT_IMPLEMENTED;
    return cvt_color_two_plane(ysrc, uvsrc, dst, code, as_stream(stream));
}

extern "C" int b200cv_cvt_color(const b200cvMat* src, const b200cvMat* dst, int code, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    if ((code >= 90 && code <= 134) || (code >= 143 && code <= 154)) {      // subsampled-YUV wire formats: source and destination sizes differ (cvtcolor_yuv.cu)
        B200_REQUIRE((src->frames > 1 ? src->frames : 1) == (dst->frames > 1 ? dst->frames : 1), "src/dst batch mismatch");
        if (B200CV_DEPTH(src->type) != B200CV_8U || B200CV_DEPTH(dst->type) != B200CV_8U) return B200CV_NOT_IMPLEMENTED;
        B200_REQUIRE(src->data != dst->data, "cvtColor: in-place is not supported");
        return cvt_color_yuv(src, dst, code, as_stream(stream));
    }
    B200_REQUIRE(src->cols == dst->cols && src->rows == dst->rows, "src/dst size mismatch");
    B200_REQUIRE((src->frames > 1 ? src->frames : 1) == (dst->frames > 1 ? dst->frames : 1), "src/dst batch mismatch");
    if ((code >= 46 && code <= 49) || (code >= 135 && code <= 142)) {     // Bayer mosaics, bilinear and edge-aware, 8- and 16-bit (demosaic.cu)
        B200_REQUIRE(src->data != dst->data, "cvtColor: in-place is not supported");
        return demosaic_bilinear(src, dst, code, as_stream(stream));
    }
    if ((code >= 62 && code <= 65) || (code >= 86 && code <= 89)) {       // Bayer VNG, 8-bit (demosaic_vng.cu); Bayer to GRAY, 8- and 16-bit (demosaic.cu)
        B200_REQUIRE(src->data != dst->data, "cvtColor: in-place is not supported");
        return code <= 65 ? demosaic_vng(src, dst, code, as_stream(stream)) : demosaic_gray(src, dst, code, as_stream(stream));
    }
    if (B200CV_DEPTH(src->type) != B200CV_8U || B200CV_DEPTH(dst->type) != B200CV_8U) return cvt_color_depth(src, dst, code, as_stream(stream));   // 16U / 32F: cvtcolor_depth.cu
    const int scn = B200CV_CN(src->type), dcn = B200CV_CN(dst->type);
    Img s = make_img(src), d = make_img(dst);
    cudaStream_t st = as_stream(stream);

    if (code >= 32 && code <= 35) {                                       // CIE XYZ (cvtcolor_lab.cu)
        B200_REQUIRE(src->data != dst->data, "cvtColor: in-place is not supported");
        return cvt_color_xyz(src, dst, code, st);
    }
    if (code == 44 || code == 45 || code == 74 || code == 75 || code == 56 || code == 57 || code == 78 || code == 79) {     // CIE Lab (cvtcolor_lab.cu)
        B200_REQUIRE(src->data != dst->data, "cvtColor: in-place is not supported");
        return cvt_color_lab(src, dst, code, st);
    }
#define NEED(sc_ok, dc_ok) B200_REQUIRE((sc_ok) && (dc_ok), "channel count does not match the colour code")
    switch (code) {
    case 0: case 1: case 2: case 3: case 4: case 5: {   // BGR2BGRA BGRA2BGR BGR2RGBA RGBA2BGR BGR2RGB BGRA2RGBA
        int want_s = (code == 0 || code == 2 || code == 4) ? 3 : 4;
        int want_d = (code == 1 || code == 3 || code == 4) ? 3 : 4;
        NEED(scn == want_s, dcn == want_d);
        switch (code) {
        case 0: return launch_cvt<3, 4>(s, d, OpBGR2BGR<0, 0>(), st);
        case 1: return launch_cvt<4, 3>(s, d, OpBGR2BGR<0, 1>(), st);
        case 2: return launch_cvt<3, 4>(s, d, OpBGR2BGR<1, 0>(), st);
        case 3: return launch_cvt<4, 3>(s, d, OpBGR2BGR<1, 1>(), st);
        case 4: return launch_cvt<3, 3>(s, d, OpBGR2BGR<1, 0>(), st);
        default: return launch_cvt<4, 4>(s, d, OpBGR2BGR<1, 1>(), st);
        }
    }
    case 6: case 7: case 10: case 11: {   // BGR2GRAY RGB2GRAY BGRA2GRAY RGBA2GRAY
        NEED(scn == ((code == 6 || code == 7) ? 3 : 4), dcn == 1);
        bool rgb = (code == 7 || code == 11);
        OpBGR2Gray op;
        op.cg = 19235;
        op.cb = rgb ? 9798 : 3735;   // coefficient applied to channel 0
        op.cr = rgb ? 3735 : 9798;   // coefficient applied to channel 2
        return scn == 3 ? launch_cvt<3, 1>(s, d, op, st) : launch_cvt<4, 1>(s, d, op, st);
    }
    case 8: case 9: {   // GRAY2BGR GRAY2BGRA
        NEED(scn == 1, dcn == (code == 8 ? 3 : 4));
        OpGray2BGR op;
        return dcn == 3 ? launch_cvt<1, 3>(s, d, op, st) : launch_cvt<1, 4>(s, d, op, st);
    }
    case 36: case 37: case 82: case 83: {   // BGR2YCrCb RGB2YCrCb BGR2YUV RGB2YUV
        NEED(scn == 3 || scn == 4, dcn == 3);
        bool isCrCb = (code == 36 || code == 37);
        int bidx = (code == 36 || code == 82) ? 0 : 2;
        int c[5] = {4899, 9617, 1868, isCrCb ? 11682 : 14369, isCrCb ? 9241 : 8061};
        if (bidx == 0) { int t = c[0]; c[0] = c[2]; c[2] = t; }
#define GO(B, Y) do { OpBGR2YCrCb<B, Y> op; op.c0 = c[0]; op.c1 = c[1]; op.c2 = c[2]; op.c3 = c[3]; op.c4 = c[4]; \
                      return scn == 3 ? launch_cvt<3, 3>(s, d, op, st) : launch_cvt<4, 3>(s, d, op, st); } while (0)
        if (bidx == 0 && isCrCb) GO(0, 0);
        if (bidx == 0) GO(0, 1);
        if (isCrCb) GO(2, 0);
        GO(2, 1);
#undef GO
    }
    case 38: case 39: case 84: case 85: {   // YCrCb2BGR YCrCb2RGB YUV2BGR YUV2RGB
        NEED(scn == 3, dcn == 3 || dcn == 4);
        bool isCrCb = (code == 38 || code == 39);
        int bidx = (code == 38 || code == 84) ? 0 : 2;
#define GO(B, Y) do { OpYCrCb2BGR<B, Y> op; op.c0 = isCrCb ? 22987 : 18678; op.c1 = isCrCb ? -11698 : -9519; \
                      op.c2 = isCrCb ? -5636 : -6472; op.c3 = isCrCb ? 29049 : 33292; \
                      return dcn == 3 ? launch_cvt<3, 3>(s, d, op, st) : launch_cvt<3, 4>(s, d, op, st); } while (0)
        if (bidx == 0 && isCrCb) GO(0, 0);
        if (bidx == 0) GO(0, 1);
        if (isCrCb) GO(2, 0);
        GO(2, 1);
#undef GO
    }
    case 40: case 41: case 66: case 67: {   // BGR2HSV RGB2HSV BGR2HSV_FULL RGB2HSV_FULL
        NEED(scn == 3 || scn == 4, dcn == 3);
        if ((rc = ensure_hsv_tables())) return rc;
        int hrange = (code == 40 || code == 41) ? 180 : 256;
#define GO(B) do { OpBGR2HSV<B> op; op.hrange = hrange; op.sdiv = op.hdiv = nullptr; \
                   return scn == 3 ? launch_cvt<3, 3, OpBGR2HSV<B>, false, true>(s, d, op, st) \
                                   : launch_cvt<4, 3, OpBGR2HSV<B>, false, true>(s, d, op, st); } while (0)
        if (code == 40 || code == 66) GO(0);
        GO(2);
#undef GO
    }
    case 54: case 55: case 70: case 71: {   // HSV2BGR HSV2RGB HSV2BGR_FULL HSV2RGB_FULL
        NEED(scn == 3, dcn == 3 || dcn == 4);
        float hscale = 6.0f / ((code == 54 || code == 55) ? 180 : 255);   // inverse _FULL uses 255 (color_hsv.simd.hpp:1302)
#define GO(B) do { OpHSV2BGR<B> op; op.hscale = hscale; op.trunc_cols = hsv_trunc_cols(src->cols); \
                   return dcn == 3 ? launch_cvt<3, 3, OpHSV2BGR<B>, true>(s, d, op, st) : launch_cvt<3, 4, OpHSV2BGR<B>, true>(s, d, op, st); } while (0)
        if (code == 54 || code == 70) GO(0);
        GO(2);
#undef GO
    }
    default:
        return B200CV_NOT_IMPLEMENTED;
    }
#undef NEED
}
