// demosaic.cu -- cv::cvtColor / cv::demosaicing for the Bayer patterns, bilinear and edge-aware interpolation, 8- and 16-bit (the
// wire format of a raw sensor).  Codes COLOR_BayerBG/GB/RG/GR2BGR = 46..49 (the 2RGB names are the same numbers permuted), 2BGRA = 139..142,
// 2BGR_EA = 135..138, and Bayer to GRAY, 2GRAY = 86..89 (VNG, 62..65, is demosaic_vng.cu).
//
// Reference (demosaicing.cpp:806-1056, Bayer2RGB_Invoker / Bayer2RGB_): for every interior pixel of the mosaic
//   at a red / blue site:  that colour = the sample, green = (4 edge neighbours + 2) >> 2, the other colour = (4 diagonal neighbours + 2) >> 2
//   at a green site:       one colour = (left + right + 1) >> 1, the other = (up + down + 1) >> 1, green = the sample
// the first / last columns repeat their interior neighbour, then the first / last rows repeat theirs (:989-1008, :1041-1055), so every
// border pixel equals the value computed at the nearest interior site -- which is how the kernel evaluates it.  All integer: bit-exact.
// Edge-aware (Bayer2RGB_EdgeAware_T_Invoker, demosaicing.cpp:1592-1737): the same, except green at a red / blue site =
//   |left - right| > |down - up| ? (up + down + 1) >> 1 : (left + right + 1) >> 1          (3-channel destinations only)
// 16-bit mosaics run the same expressions (the reference's scalar interpolator); both pinned on the CPU against the compiled reference.
// `blue` (+1 / -1: which of the two colours the non-green sites of the first interior row carry) and `start_with_green` alternate row by row.
// Eight destination pixels per thread (one 24- / 32-byte store when aligned), 3 x 3 byte neighbourhoods through L1: the bound is HBM
// (1 + 3 bytes per pixel).
#include "common.cuh"
#include "bytes.cuh"

namespace b200cv {

namespace {

template <typename T, int DCN, bool EA>
__global__ void __launch_bounds__(256) bayer_bilinear_kernel(Img src, Img dst, int W, int H, int blue0, int swg0)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;          // 8 destination pixels per thread, one 24- / 32-byte row piece out
    const int y = blockIdx.y, f = blockIdx.z;
    if (x0 >= W) return;
    const int n = min(8, W - x0);
    const int yi = min(max(y, 1), H - 2);                                 // border pixels repeat the nearest interior site
    const int i = yi - 1;                                                 // interior row, 0-based
    const int blue = (i & 1) ? -blue0 : blue0;
    const bool swg = ((i & 1) != 0) != (swg0 != 0);                       // this interior row starts with a green site
    const T* q0 = src.row<T>(f, yi - 1);
    const T* q1 = src.row<T>(f, yi);
    const T* q2 = src.row<T>(f, yi + 1);
    union { T e[8 * DCN]; uchar b[8 * DCN * sizeof(T)]; } o;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int xi = min(max(min(x0 + j, W - 1), 1), W - 2), k = xi - 1;  // interior column, 0-based (columns past the row end are computed but not stored)
        const bool green = ((k & 1) == 0) == swg;
        const T *r0 = q0 + xi, *r1 = q1 + xi, *r2 = q2 + xi;
        int c_lo, c_hi, g;                                                // channel 1 - blue, channel 1 + blue, green
        if (green) {
            c_lo = (r0[0] + r2[0] + 1) >> 1;                              // vertical neighbours
            c_hi = (r1[-1] + r1[1] + 1) >> 1;                             // horizontal neighbours
            g = r1[0];
        } else {
            c_lo = (r0[-1] + r0[1] + r2[-1] + r2[1] + 2) >> 2;            // diagonals
            if constexpr (EA) g = (abs((int)r1[-1] - (int)r1[1]) > abs((int)r2[0] - (int)r0[0]) ? r2[0] + r0[0] + 1 : r1[-1] + r1[1] + 1) >> 1;
            else g = (r0[0] + r1[-1] + r1[1] + r2[0] + 2) >> 2;           // edge neighbours
            c_hi = r1[0];
        }
        o.e[j * DCN] = (T)(blue > 0 ? c_lo : c_hi);
        o.e[j * DCN + 1] = (T)g;
        o.e[j * DCN + 2] = (T)(blue > 0 ? c_hi : c_lo);
        if constexpr (DCN == 4) o.e[j * DCN + 3] = (T)(sizeof(T) == 1 ? 255 : 65535);
    }
    if constexpr (sizeof(T) == 1) store_bytes<8 * DCN>(dst.row<uchar>(f, y) + (size_t)x0 * DCN, n * DCN, o.b);
    else {      // 16-bit: two halves of 8 * DCN bytes each
        uchar* dp = dst.row<uchar>(f, y) + (size_t)x0 * DCN * 2;
        const int nb = n * DCN * 2;
        uchar lo[8 * DCN], hi[8 * DCN];
#pragma unroll
        for (int k = 0; k < 8 * DCN; k++) { lo[k] = o.b[k]; hi[k] = o.b[8 * DCN + k]; }
        store_bytes<8 * DCN>(dp, min(nb, 8 * DCN), lo);
        if (nb > 8 * DCN) store_bytes<8 * DCN>(dp + 8 * DCN, nb - 8 * DCN, hi);
    }
}

// Bayer2Gray_ (demosaicing.cpp:652-792): at a red / blue site (4 diagonal neighbours * rcoeff + 4 edge neighbours * G2Y + 4 * sample * bcoeff
// + 2^15) >> 16, at a green site (2 vertical neighbours * rcoeff + 2 horizontal neighbours * bcoeff + 2 * G2Y * sample + 2^14) >> 15; rcoeff
// and bcoeff swap and start_with_green flips every interior row.  Unsigned sums: a 16-bit mosaic reaches 4 294 934 528 > INT_MAX.  The
// reference's 8-bit vector body (:180-272) is the same arithmetic scaled by 2.  Border pixels repeat the nearest interior site; an image
// with W <= 2 or H <= 2 is all zero (:695-699, :789-791).  Eight destination pixels per thread.
template <typename T>
__global__ void __launch_bounds__(256) bayer_gray_kernel(Img src, Img dst, int W, int H, unsigned b0, unsigned r0, int swg0)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x0 >= W) return;
    const int n = min(8, W - x0);
    union { T e[8]; uchar b[8 * sizeof(T)]; } o;
    if (W <= 2 || H <= 2) {
#pragma unroll
        for (int j = 0; j < 8; j++) o.e[j] = 0;
    } else {
        const unsigned G2Y = 9617;
        const int yi = min(max(y, 1), H - 2), i = yi - 1;
        const unsigned bco = (i & 1) ? r0 : b0, rco = (i & 1) ? b0 : r0;
        const bool swg = ((i & 1) != 0) != (swg0 != 0);
        const T* q0 = src.row<T>(f, yi - 1);
        const T* q1 = src.row<T>(f, yi);
        const T* q2 = src.row<T>(f, yi + 1);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int xi = min(max(min(x0 + j, W - 1), 1), W - 2), k = xi - 1;
            const T *r0p = q0 + xi, *r1 = q1 + xi, *r2 = q2 + xi;
            unsigned v;
            if (((k & 1) == 0) == swg)
                v = ((unsigned)(r0p[0] + r2[0]) * rco + (unsigned)(r1[-1] + r1[1]) * bco + (unsigned)r1[0] * (2 * G2Y) + (1u << 14)) >> 15;
            else
                v = ((unsigned)(r0p[-1] + r0p[1] + r2[-1] + r2[1]) * rco + (unsigned)(r0p[0] + r1[-1] + r1[1] + r2[0]) * G2Y + (unsigned)r1[0] * (4 * bco)
                     + (1u << 15)) >> 16;
            o.e[j] = (T)v;
        }
    }
    uchar* dp = dst.row<uchar>(f, y) + (size_t)x0 * sizeof(T);
    if constexpr (sizeof(T) == 1) store_bytes<8>(dp, n, o.b);
    else store_bytes<16>(dp, n * 2, o.b);
}

}  // namespace

// called by b200cv_cvt_color for codes 86-89 (matrices of equal size and batch, not in place, already checked); 8- and 16-bit
int demosaic_gray(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st)
{
    const int depth = B200CV_DEPTH(src->type);
    if ((depth != B200CV_8U && depth != B200CV_16U) || B200CV_DEPTH(dst->type) != depth) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(B200CV_CN(src->type) == 1 && B200CV_CN(dst->type) == 1, "Bayer -> GRAY needs a 1-channel mosaic and a 1-channel destination");
    Img s = make_img(src), d = make_img(dst);
    const int W = src->cols, H = src->rows;
    if (H >= 65536 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    const unsigned R2Y = 4899, B2Y = 1868;
    const int c = code - 86;                                            // 0 BG, 1 GB, 2 RG, 3 GR
    const unsigned b0 = c < 2 ? B2Y : R2Y, r0 = c < 2 ? R2Y : B2Y;
    const dim3 block(256);
    const dim3 grid(div_up(div_up((unsigned)W, 8), 256), (unsigned)H, (unsigned)s.frames);
    if (depth == B200CV_8U) bayer_gray_kernel<uchar><<<grid, block, 0, st>>>(s, d, W, H, b0, r0, c & 1);
    else bayer_gray_kernel<unsigned short><<<grid, block, 0, st>>>(s, d, W, H, b0, r0, c & 1);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

// called by b200cv_cvt_color for codes 46-49, 135-138 (edge-aware) and 139-142 (matrices of equal size and batch already checked); 8- and 16-bit
int demosaic_bilinear(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st)
{
    const int scn = B200CV_CN(src->type), dcn = B200CV_CN(dst->type), depth = B200CV_DEPTH(src->type);
    const bool four = code >= 139, ea = code >= 135 && code <= 138;
    if ((depth != B200CV_8U && depth != B200CV_16U) || B200CV_DEPTH(dst->type) != depth) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(scn == 1 && dcn == (four ? 4 : 3), "Bayer -> BGR needs a 1-channel mosaic and a 3-channel (BGRA codes: 4-channel) destination");
    const int W = src->cols, H = src->rows;
    if (W < 3 || H < 3) return B200CV_NOT_IMPLEMENTED;                  // the reference zero-fills such images (demosaicing.cpp:836-851, :1051-1055, :1697-1701)
    Img s = make_img(src), d = make_img(dst);
    if (H >= 65536 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    const int c = four ? code - 139 : ea ? code - 135 : code - 46;      // 0 BG, 1 GB, 2 RG, 3 GR
    const int blue0 = c < 2 ? -1 : 1, swg0 = (c & 1);
    const dim3 block(256);
    const dim3 grid(div_up(div_up((unsigned)W, 8), 256), (unsigned)H, (unsigned)s.frames);
    if (depth == B200CV_8U) {
        if (ea) bayer_bilinear_kernel<uchar, 3, true><<<grid, block, 0, st>>>(s, d, W, H, blue0, swg0);
        else if (dcn == 3) bayer_bilinear_kernel<uchar, 3, false><<<grid, block, 0, st>>>(s, d, W, H, blue0, swg0);
        else bayer_bilinear_kernel<uchar, 4, false><<<grid, block, 0, st>>>(s, d, W, H, blue0, swg0);
    } else {
        if (ea) bayer_bilinear_kernel<unsigned short, 3, true><<<grid, block, 0, st>>>(s, d, W, H, blue0, swg0);
        else if (dcn == 3) bayer_bilinear_kernel<unsigned short, 3, false><<<grid, block, 0, st>>>(s, d, W, H, blue0, swg0);
        else bayer_bilinear_kernel<unsigned short, 4, false><<<grid, block, 0, st>>>(s, d, W, H, blue0, swg0);
    }
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace b200cv
