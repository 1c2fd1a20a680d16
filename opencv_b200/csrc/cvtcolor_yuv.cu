// cvtcolor_yuv.cu -- cv::cvtColor for the subsampled-YUV wire formats (what a video decoder hands to the path).
//
//   4:2:0 two-plane  NV12 / NV21 -> RGB / BGR / RGBA / BGRA       codes 90-97    (color_yuv.simd.hpp:1196-1318)
//   4:2:0 three-plane YV12 / IYUV -> RGB / BGR / RGBA / BGRA      codes 98-105   (:1320-1448, plane layout :2074-2106)
//   4:2:0 -> GRAY (the Y plane)                                    code 106       (color.cpp:337)
//   4:2:2 UYVY / YUY2 / YVYU -> RGB / BGR / RGBA / BGRA, -> GRAY   codes 107-124  (:1733-1858, color.cpp:346-380)
//   RGB / BGR / RGBA / BGRA -> IYUV (I420) / YV12                  codes 127-134  (:1473-1730)
//   RGB / BGR / RGBA / BGRA -> UYVY / YUY2 / YVYU                  codes 143-154  (:1862-1958)
//
// BT.601 limited range in 20-bit fixed point, all integer, bit-exact (the reference's SIMD bodies and scalar tails agree):
//   ruv = 2^19 + 1673527 (v-128);  guv = 2^19 - 852492 (v-128) - 409993 (u-128);  buv = 2^19 + 2116026 (u-128)
//   c = saturate((max(0, y-16) * 1220542 + cuv) >> 20)
//   Y = (269484 r + 528482 g + 102760 b + 2^19 + (16 << 20)) >> 20;  U, V from the even-row, even-column pixel only.
// A 4:2:0 image of W x H pixels is ONE 8-bit plane of H*3/2 rows: H luma rows, then H/2 interleaved chroma rows of W bytes (NV) or
// H planar half rows of W/2 bytes, two to a row, the first plane's H/2 half rows before the second's (so the second plane starts in
// the middle of a row when H % 4 == 2).
// One thread = 8 pixels of a row pair (4:2:0) or of one row (4:2:2): 8-/16-byte loads and stores when the addresses allow, bytes
// otherwise.  Pure streaming: the bound is HBM (1.5 + 3 bytes per pixel for NV12 -> BGR).
#include "common.cuh"
#include "bytes.cuh"

namespace b200cv {

namespace {

struct UvTerm { int r, g, b; };

__device__ __forceinline__ UvTerm uv_term(int u, int v)
{
    const int uu = u - 128, vv = v - 128;
    UvTerm t;
    t.r = (1 << 19) + 1673527 * vv;
    t.g = (1 << 19) - 852492 * vv - 409993 * uu;
    t.b = (1 << 19) + 2116026 * uu;
    return t;
}

// one pixel: d[0..DCN-1] in the destination's channel order (bidx = position of blue)
template <int DCN>
__device__ __forceinline__ void yuv_pixel(int y, const UvTerm& t, int bidx, uchar* d)
{
    const int yy = max(0, y - 16) * 1220542;
    const uchar r = sat_u8((yy + t.r) >> 20), g = sat_u8((yy + t.g) >> 20), b = sat_u8((yy + t.b) >> 20);
    d[0] = bidx ? r : b;
    d[1] = g;
    d[2] = bidx ? b : r;
    if constexpr (DCN == 4) d[3] = 255;
}

// ---- 4:2:0 -> BGR family ---------------------------------------------------------------------------------------------------------
// ysrc: the H luma rows; csrc: the chroma rows that follow them (interleaved rows of W bytes, or planar half rows, two to a row) -- a view
// into the same buffer for cv::cvtColor, a buffer of its own for cv::cvtColorTwoPlane
template <int DCN, bool PLANAR>
__global__ void __launch_bounds__(256) yuv420_to_bgr_kernel(Img ysrc, Img csrc, Img dst, int W, int H, int bidx, int uidx)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const int j = blockIdx.y * blockDim.y + threadIdx.y;              // row pair
    const int f = blockIdx.z;
    if (x0 >= W || 2 * j >= H) return;
    const int n = min(8, W - x0);                                     // even: W is even
    uchar ya[8], yb[8], cu[4], cv[4];
    load_bytes<8>(ysrc.row<uchar>(f, 2 * j) + x0, n, ya);
    load_bytes<8>(ysrc.row<uchar>(f, 2 * j + 1) + x0, n, yb);
    if constexpr (PLANAR) {
        const int k0 = j, k1 = H / 2 + j;                             // half-row index in the first / second chroma plane
        uchar pa[4], pb[4];
        load_bytes<4>(csrc.row<uchar>(f, k0 / 2) + (k0 & 1) * (W / 2) + x0 / 2, n / 2, pa);
        load_bytes<4>(csrc.row<uchar>(f, k1 / 2) + (k1 & 1) * (W / 2) + x0 / 2, n / 2, pb);
#pragma unroll
        for (int i = 0; i < 4; i++) { cu[i] = uidx ? pb[i] : pa[i]; cv[i] = uidx ? pa[i] : pb[i]; }
    } else {
        uchar c[8];
        load_bytes<8>(csrc.row<uchar>(f, j) + x0, n, c);
#pragma unroll
        for (int i = 0; i < 4; i++) { cu[i] = uidx ? c[2 * i + 1] : c[2 * i]; cv[i] = uidx ? c[2 * i] : c[2 * i + 1]; }
    }
    uchar o0[8 * DCN], o1[8 * DCN];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const UvTerm t = uv_term(cu[i], cv[i]);
        yuv_pixel<DCN>(ya[2 * i], t, bidx, o0 + (2 * i) * DCN);
        yuv_pixel<DCN>(ya[2 * i + 1], t, bidx, o0 + (2 * i + 1) * DCN);
        yuv_pixel<DCN>(yb[2 * i], t, bidx, o1 + (2 * i) * DCN);
        yuv_pixel<DCN>(yb[2 * i + 1], t, bidx, o1 + (2 * i + 1) * DCN);
    }
    store_bytes<8 * DCN>(dst.row<uchar>(f, 2 * j) + x0 * DCN, n * DCN, o0);
    store_bytes<8 * DCN>(dst.row<uchar>(f, 2 * j + 1) + x0 * DCN, n * DCN, o1);
}

// ---- 4:2:2 -> BGR family: 4 source bytes = 2 pixels.  fmt 0 = YUY2 (Y0 U Y1 V), 1 = YVYU (Y0 V Y1 U), 2 = UYVY (U Y0 V Y1) -----------------
template <int DCN>
__global__ void __launch_bounds__(256) yuv422_to_bgr_kernel(Img src, Img dst, int W, int H, int bidx, int fmt)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int f = blockIdx.z;
    if (x0 >= W || y >= H) return;
    const int n = min(8, W - x0);
    uchar s[16];
    load_bytes<16>(src.row<uchar>(f, y) + x0 * 2, n * 2, s);
    uchar o[8 * DCN];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int q0 = s[4 * i], q1 = s[4 * i + 1], q2 = s[4 * i + 2], q3 = s[4 * i + 3];      // selects, not run-time indices (registers)
        const int ly0 = fmt == 2 ? q1 : q0, ly1 = fmt == 2 ? q3 : q2;
        const int u = fmt == 2 ? q0 : fmt == 1 ? q3 : q1, v = fmt == 2 ? q2 : fmt == 1 ? q1 : q3;
        const UvTerm t = uv_term(u, v);
        yuv_pixel<DCN>(ly0, t, bidx, o + (2 * i) * DCN);
        yuv_pixel<DCN>(ly1, t, bidx, o + (2 * i + 1) * DCN);
    }
    store_bytes<8 * DCN>(dst.row<uchar>(f, y) + x0 * DCN, n * DCN, o);
}

// ---- luma extraction: STRIDE 1 = the Y plane of a 4:2:0 image, STRIDE 2 = every second byte of a 4:2:2 row (from byte `off`) ----------
template <int STRIDE>
__global__ void __launch_bounds__(256) yuv_luma_kernel(Img src, Img dst, int W, int H, int off)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int f = blockIdx.z;
    if (x0 >= W || y >= H) return;
    const int n = min(8, W - x0);
    uchar s[8 * STRIDE], o[8];
    load_bytes<8 * STRIDE>(src.row<uchar>(f, y) + x0 * STRIDE, n * STRIDE, s);
#pragma unroll
    for (int i = 0; i < 8; i++) {
        if constexpr (STRIDE == 2) o[i] = off ? s[2 * i + 1] : s[2 * i];
        else o[i] = s[i];
    }
    store_bytes<8>(dst.row<uchar>(f, y) + x0, n, o);
}

// ---- BGR family -> IYUV / YV12 -----------------------------------------------------------------------------------------------------
template <int SCN>
__global__ void __launch_bounds__(256) bgr_to_yuv420_kernel(Img src, Img dst, int W, int H, int bidx, int yv12)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const int j = blockIdx.y * blockDim.y + threadIdx.y;
    const int f = blockIdx.z;
    if (x0 >= W || 2 * j >= H) return;
    const int n = min(8, W - x0);
    uchar a[8 * SCN], b[8 * SCN], y0[8], y1[8], uo[4], vo[4];
    load_bytes<8 * SCN>(src.row<uchar>(f, 2 * j) + x0 * SCN, n * SCN, a);
    load_bytes<8 * SCN>(src.row<uchar>(f, 2 * j + 1) + x0 * SCN, n * SCN, b);
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int ba = bidx ? a[i * SCN + 2] : a[i * SCN], ga = a[i * SCN + 1], ra = bidx ? a[i * SCN] : a[i * SCN + 2];
        const int bb = bidx ? b[i * SCN + 2] : b[i * SCN], gb = b[i * SCN + 1], rb = bidx ? b[i * SCN] : b[i * SCN + 2];
        y0[i] = sat_u8((269484 * ra + 528482 * ga + 102760 * ba + (1 << 19) + (16 << 20)) >> 20);
        y1[i] = sat_u8((269484 * rb + 528482 * gb + 102760 * bb + (1 << 19) + (16 << 20)) >> 20);
        if ((i & 1) == 0) {
            uo[i / 2] = sat_u8((-155188 * ra - 305135 * ga + 460324 * ba + (1 << 19) + (128 << 20)) >> 20);
            vo[i / 2] = sat_u8((460324 * ra - 385875 * ga - 74448 * ba + (1 << 19) + (128 << 20)) >> 20);
        }
    }
    store_bytes<8>(dst.row<uchar>(f, 2 * j) + x0, n, y0);
    store_bytes<8>(dst.row<uchar>(f, 2 * j + 1) + x0, n, y1);
    const int ku = j + (yv12 ? H / 2 : 0), kv = j + (yv12 ? 0 : H / 2);
    store_bytes<4>(dst.row<uchar>(f, H + ku / 2) + (ku & 1) * (W / 2) + x0 / 2, n / 2, uo);
    store_bytes<4>(dst.row<uchar>(f, H + kv / 2) + (kv & 1) * (W / 2) + x0 / 2, n / 2, vo);
}

// ---- BGR family -> 4:2:2 (color_yuv.simd.hpp:1862-1958; 14-bit fixed point; U, V from the SUM of the two pixels with halved coefficients) ----
// fmt 0 = YUY2 (Y0 U Y1 V), 1 = YVYU (Y0 V Y1 U), 2 = UYVY (U Y0 V Y1)
template <int SCN>
__global__ void __launch_bounds__(256) bgr_to_yuv422_kernel(Img src, Img dst, int W, int H, int bidx, int fmt)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int f = blockIdx.z;
    if (x0 >= W || y >= H) return;
    const int n = min(8, W - x0);
    uchar a[8 * SCN], o[16];
    load_bytes<8 * SCN>(src.row<uchar>(f, y) + x0 * SCN, n * SCN, a);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uchar* p = a + 2 * i * SCN;
        const int b1 = bidx ? p[2] : p[0], g1 = p[1], r1 = bidx ? p[0] : p[2];
        const int b2 = bidx ? p[SCN + 2] : p[SCN], g2 = p[SCN + 1], r2 = bidx ? p[SCN] : p[SCN + 2];
        const uchar ya = sat_u8(((1 << 13) + r1 * 4211 + g1 * 8258 + b1 * 1606 + (1 << 14) * 16) >> 14);
        const uchar yb = sat_u8(((1 << 13) + r2 * 4211 + g2 * 8258 + b2 * 1606 + (1 << 14) * 16) >> 14);
        const int sr = r1 + r2, sg = g1 + g2, sb = b1 + b2;
        const uchar u = sat_u8(((1 << 13) + sr * -1212 + sg * -2384 + sb * 3596 + (1 << 13) * 256) >> 14);
        const uchar v = sat_u8(((1 << 13) + sr * 3596 + sg * -3015 + sb * -582 + (1 << 13) * 256) >> 14);
        o[4 * i] = fmt == 2 ? u : ya;
        o[4 * i + 1] = fmt == 2 ? ya : fmt == 1 ? v : u;
        o[4 * i + 2] = fmt == 2 ? v : yb;
        o[4 * i + 3] = fmt == 2 ? yb : fmt == 1 ? u : v;
    }
    store_bytes<16>(dst.row<uchar>(f, y) + x0 * 2, n * 2, o);
}

static dim3 yuv_grid(int W, int rows, int frames, dim3 block)
{
    return dim3(div_up(div_up((unsigned)W, 8), block.x), div_up((unsigned)rows, block.y), (unsigned)frames);
}

}  // namespace

// called by b200cv_cvt_color for codes 90-134; src / dst already validated as 8-bit matrices with equal batch sizes
int cvt_color_yuv(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st)
{
    const int scn = B200CV_CN(src->type), dcn = B200CV_CN(dst->type);
    Img s = make_img(src), d = make_img(dst);
    if (s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    const dim3 block(32, 8);
    if (code >= 90 && code <= 106) {
        const int W = dst->cols, H = dst->rows;
        B200_REQUIRE(scn == 1 && src->cols == W && src->rows == H * 3 / 2 && (W & 1) == 0 && (H & 1) == 0 && W > 0 && H > 0,
                     "4:2:0 source must be one 8-bit plane of (height * 3 / 2) x width with even width and height");
        if (code == 106) {
            B200_REQUIRE(dcn == 1, "COLOR_YUV2GRAY_420 needs a 1-channel destination");
            const dim3 grid = yuv_grid(W, H, s.frames, block);
            if (grid.y >= 65536) return B200CV_NOT_IMPLEMENTED;
            yuv_luma_kernel<1><<<grid, block, 0, st>>>(s, d, W, H, 0);
            B200_LAUNCH_CHECK();
            return B200CV_OK;
        }
        B200_REQUIRE(dcn == 3 || dcn == 4, "4:2:0 -> BGR needs a 3- or 4-channel destination");
        const bool planar = code >= 98;
        int rgb, uidx;                                                 // uidx 1: V before U (NV21, YV12)
        if (!planar) { const int c = code - 90; rgb = !(c & 1); uidx = (c >> 1) & 1; B200_REQUIRE((c >= 4) == (dcn == 4), "channel count does not match the colour code"); }
        else { const int c = code - 98; rgb = !(c & 1); uidx = (c & 3) < 2; B200_REQUIRE((c >= 4) == (dcn == 4), "channel count does not match the colour code"); }
        const int bidx = rgb ? 2 : 0;
        const dim3 grid = yuv_grid(W, H / 2, s.frames, block);
        if (grid.y >= 65536) return B200CV_NOT_IMPLEMENTED;
        Img c = s;                                                     // the chroma rows follow the H luma rows in the same buffer
        c.data += (size_t)H * s.step; c.rows = H / 2;
        if (planar) {
            if (dcn == 3) yuv420_to_bgr_kernel<3, true><<<grid, block, 0, st>>>(s, c, d, W, H, bidx, uidx);
            else yuv420_to_bgr_kernel<4, true><<<grid, block, 0, st>>>(s, c, d, W, H, bidx, uidx);
        } else {
            if (dcn == 3) yuv420_to_bgr_kernel<3, false><<<grid, block, 0, st>>>(s, c, d, W, H, bidx, uidx);
            else yuv420_to_bgr_kernel<4, false><<<grid, block, 0, st>>>(s, c, d, W, H, bidx, uidx);
        }
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }
    if (code >= 107 && code <= 124) {
        if (code == 109 || code == 110 || code == 113 || code == 114) return B200CV_NOT_IMPLEMENTED;      // VYUY: not in the reference either
        const int W = dst->cols, H = dst->rows;
        B200_REQUIRE(scn == 2 && src->cols == W && src->rows == H && (W & 1) == 0 && W > 0 && H > 0, "4:2:2 source must be 8UC2 with an even width");
        const dim3 grid = yuv_grid(W, H, s.frames, block);
        if (grid.y >= 65536) return B200CV_NOT_IMPLEMENTED;
        if (code >= 123) {
            B200_REQUIRE(dcn == 1, "COLOR_YUV2GRAY_* needs a 1-channel destination");
            yuv_luma_kernel<2><<<grid, block, 0, st>>>(s, d, W, H, code == 123 ? 1 : 0);
            B200_LAUNCH_CHECK();
            return B200CV_OK;
        }
        const bool uyvy = code == 107 || code == 108 || code == 111 || code == 112;
        const bool yvyu = code == 117 || code == 118 || code == 121 || code == 122;
        const bool rgb = code == 107 || code == 111 || code == 115 || code == 117 || code == 119 || code == 121;
        const bool four = code == 111 || code == 112 || (code >= 119 && code <= 122);
        B200_REQUIRE(dcn == (four ? 4 : 3), "channel count does not match the colour code");
        const int fmt = uyvy ? 2 : yvyu ? 1 : 0;                       // byte positions: color_yuv.simd.hpp:1751-1756
        if (dcn == 3) yuv422_to_bgr_kernel<3><<<grid, block, 0, st>>>(s, d, W, H, rgb ? 2 : 0, fmt);
        else yuv422_to_bgr_kernel<4><<<grid, block, 0, st>>>(s, d, W, H, rgb ? 2 : 0, fmt);
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }
    if (code >= 127 && code <= 134) {
        const int W = src->cols, H = src->rows;
        B200_REQUIRE((scn == 3 || scn == 4) && dcn == 1 && dst->cols == W && dst->rows == H * 3 / 2 && (W & 1) == 0 && (H & 1) == 0 && W > 0 && H > 0,
                     "BGR -> 4:2:0 needs an even-sized 3-/4-channel source and one 8-bit plane of (height * 3 / 2) x width");
        const int c = (code - 127) & 3;
        const int bidx = (c & 1) ? 0 : 2, yv12 = code >= 131;          // the channel count is the source's (color.cpp passes scn through)
        const dim3 grid = yuv_grid(W, H / 2, s.frames, block);
        if (grid.y >= 65536) return B200CV_NOT_IMPLEMENTED;
        if (scn == 3) bgr_to_yuv420_kernel<3><<<grid, block, 0, st>>>(s, d, W, H, bidx, yv12);
        else bgr_to_yuv420_kernel<4><<<grid, block, 0, st>>>(s, d, W, H, bidx, yv12);
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }
    if (code >= 143 && code <= 154) {
        const int W = src->cols, H = src->rows;
        B200_REQUIRE((scn == 3 || scn == 4) && dcn == 2 && dst->cols == W && dst->rows == H && (W & 1) == 0 && W > 0 && H > 0,
                     "BGR -> 4:2:2 needs a 3-/4-channel source of even width and an 8UC2 destination of the same size");
        const bool uyvy = code <= 146, yvyu = code == 149 || code == 150 || code == 153 || code == 154;
        const int bidx = (code & 1) ? 2 : 0;                           // odd codes are the RGB(A) ones; the channel count is the source's
        const dim3 grid = yuv_grid(W, H, s.frames, block);
        if (grid.y >= 65536) return B200CV_NOT_IMPLEMENTED;
        if (scn == 3) bgr_to_yuv422_kernel<3><<<grid, block, 0, st>>>(s, d, W, H, bidx, uyvy ? 2 : yvyu ? 1 : 0);
        else bgr_to_yuv422_kernel<4><<<grid, block, 0, st>>>(s, d, W, H, bidx, uyvy ? 2 : yvyu ? 1 : 0);
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }
    return B200CV_NOT_IMPLEMENTED;
}

// cv::cvtColorTwoPlane (color.cpp:171-185): NV12 / NV21 with the luma plane (8UC1, W x H) and the interleaved chroma plane (8UC2,
// W/2 x H/2) in buffers of their own, each with its own pitch -- what hardware decoders hand out.  Codes 90-97 only, as in the reference.
int cvt_color_two_plane(const b200cvMat* ysrc, const b200cvMat* uvsrc, const b200cvMat* dst, int code, cudaStream_t st)
{
    if (code < 90 || code > 97) return B200CV_NOT_IMPLEMENTED;
    const int W = dst->cols, H = dst->rows, dcn = B200CV_CN(dst->type);
    B200_REQUIRE(B200CV_CN(ysrc->type) == 1 && ysrc->cols == W && ysrc->rows == H && (W & 1) == 0 && (H & 1) == 0 && W > 0 && H > 0,
                 "cvtColorTwoPlane: the luma plane must be 8UC1 of the destination's (even) size");
    B200_REQUIRE(B200CV_CN(uvsrc->type) == 2 && uvsrc->cols == W / 2 && uvsrc->rows == H / 2, "cvtColorTwoPlane: the chroma plane must be 8UC2 of half the size");
    const int c = code - 90, rgb = !(c & 1), uidx = (c >> 1) & 1;
    B200_REQUIRE((c >= 4) == (dcn == 4) && (dcn == 3 || dcn == 4), "channel count does not match the colour code");
    Img y = make_img(ysrc), uv = make_img(uvsrc), d = make_img(dst);
    B200_REQUIRE(y.frames == uv.frames && y.frames == d.frames, "src/dst batch mismatch");
    if (y.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    const dim3 block(32, 8);
    const dim3 grid = yuv_grid(W, H / 2, y.frames, block);
    if (grid.y >= 65536) return B200CV_NOT_IMPLEMENTED;
    if (dcn == 3) yuv420_to_bgr_kernel<3, false><<<grid, block, 0, st>>>(y, uv, d, W, H, rgb ? 2 : 0, uidx);
    else yuv420_to_bgr_kernel<4, false><<<grid, block, 0, st>>>(y, uv, d, W, H, rgb ? 2 : 0, uidx);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace b200cv
