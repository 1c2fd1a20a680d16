// cvtcolor_lab.cu -- cv::cvtColor BGR / RGB <-> CIE Lab for 8-bit images: codes 44 BGR2Lab, 45 RGB2Lab, 74 LBGR2Lab,
// 75 LRGB2Lab, 56 Lab2BGR, 57 Lab2RGB, 78 Lab2LBGR, 79 Lab2LRGB.
//
// The reference's 8-bit paths are integer arithmetic around a handful of tables (color_lab.cpp):
//   to Lab   (RGB2Lab_b :1573-1890): g = gamma table (sRGB curve at 255*8 resolution, or linear); X, Y, Z = (R*C0 + G*C1 + B*C2 + 2^11) >> 12 with
//            the sRGB -> XYZ matrix divided by the D65 white point; f = cube-root table at 2^15 scale;
//            L = (296 f(Y) + Lshift + 2^14) >> 15,  a = (500 (f(X) - f(Y)) + 128 * 2^15 + 2^14) >> 15,  b = (200 (f(Y) - f(Z)) + ...) >> 15
//   from Lab (Lab2RGBinteger :2399-2700): (y, fy) = LabToYF_b[L]; x = abToXZ_b[fy + adiv(a)], z = abToXZ_b[fy - bdiv(b)] (piecewise linear /
//            cubic in 14-bit fixed point); rgb = (C * xyz + 2^13) >> 14 clipped to [0, 4095]; inverse-gamma table, or (v * 255) >> 12.
// The tables (:1225-1308, :1086-1107) are built on the host once, with the reference's expressions; its softfloat cbrt (core/src/softfloat.cpp:
// 3897-3930: a rational polynomial whose result mantissa is TRUNCATED) is restated bit for bit, pow goes through libm.  The port, which
// shares these expressions, equals the reference on all 2^24 colours in both directions (tests/test_oracle.py): bit-exact.
// Eight pixels per thread (24- / 32-byte vector accesses when the addresses allow), table lookups through L1 / L2 (the tables total 165 KB):
// streaming, HBM-bound (6 bytes per pixel).
#include <math.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "common.cuh"
#include "bytes.cuh"

namespace b200cv {

namespace {

enum { LAB_CBRT_N = 256 * 3 / 2 * 8, LAB_INVG_N = 4096, LAB_BASE = 1 << 14, LAB_MIN_AB = -8145, LAB_ABXZ_N = LAB_BASE * 9 / 4 };

__device__ unsigned short g_lab_gamma[256];
__device__ unsigned short g_lab_cbrt[LAB_CBRT_N];
__device__ unsigned short g_lab_yf[512];
__device__ unsigned short g_lab_invgamma[LAB_INVG_N];
__device__ int g_lab_abxz[LAB_ABXZ_N];

// cv::cbrt(softfloat): exponent split by three, quartic rational polynomial of the mantissa in double, result mantissa truncated to 23 bits
float soft_cbrtf(float x)
{
    uint32_t v; memcpy(&v, &x, 4);
    if ((v & 0x7fffffffu) == 0) return 0.f;
    const uint32_t s = v >> 31;
    int ex = (int)((v >> 23) & 255) - 127, shx = ex % 3;
    shx -= shx >= 0 ? 3 : 0;
    ex = (ex - shx) / 3 - 1;
    const uint64_t fv = ((uint64_t)(shx + 1023) << 52) | ((uint64_t)(v & 0x7fffffu) << 29);
    double fr; memcpy(&fr, &fv, 8);
    static const uint64_t K[9] = {0x4046a09e6653ba70ull, 0x406808f46c6116e0ull, 0x405dca97439cae14ull, 0x402add70d2827500ull, 0x3fc4f15f83f55d2dull,
                                  0x402d9e20660edb21ull, 0x4062ff15c0285815ull, 0x406510d06a8112ceull, 0x4040fecbc9e2c375ull};
    double A[9]; memcpy(A, K, sizeof(A));
    volatile double num = A[0] * fr; num = num + A[1]; num = num * fr; num = num + A[2]; num = num * fr; num = num + A[3]; num = num * fr; num = num + A[4];
    volatile double den = A[5] * fr; den = den + A[6]; den = den * fr; den = den + A[7]; den = den * fr; den = den + A[8]; den = den * fr; den = den + 1.0;
    const double q = num / den;
    uint64_t r; memcpy(&r, &q, 8);
    const uint32_t y = (s << 31) | ((uint32_t)(ex + 127) << 23) | (uint32_t)((r & 0xFFFFFFFFFFFFFull) >> 29);
    float out; memcpy(&out, &y, 4);
    return out;
}

struct LabHostTabs {
    std::vector<unsigned short> gamma, cbrt, yf, invgamma;
    std::vector<int> abxz;
};

void build_lab_tabs(LabHostTabs& t)          // createLabTabs, color_lab.cpp:1225-1308 (the 8-bit tables)
{
    t.gamma.resize(256); t.cbrt.resize(LAB_CBRT_N); t.yf.resize(512); t.invgamma.resize(LAB_INVG_N); t.abxz.resize(LAB_ABXZ_N);
    const float intScale = 255 * 8;
    for (int i = 0; i < 256; i++) {
        const float x = (float)i / 255.f;
        const double xd = x;
        const float g = (float)(xd <= 809. / 20000. ? xd / (323. / 25.) : pow((xd + 11. / 200.) / (1. + 11. / 200.), 12. / 5.));
        t.gamma[i] = (unsigned short)lrintf(intScale * g);
    }
    const float cbScale = 1.f / (255.f * 8), lthresh = 216.f / 24389.f, lscale = 841.f / 108.f, lbias = 16.f / 116.f, lshift2 = 32768.f;
    for (int i = 0; i < LAB_CBRT_N; i++) {
        const float x = cbScale * (float)i;
        const float f = x < lthresh ? fmaf(x, lscale, lbias) : soft_cbrtf(x);
        t.cbrt[i] = (unsigned short)lrintf(lshift2 * f);
    }
    for (int i = 0; i < 256; i++) {
        int yv, ify;
        if (i <= 20) {
            yv = (int)lrintf((float)(i * LAB_BASE * 20 * 9) / (float)(17 * 29 * 29 * 29));
            ify = (int)lrintf((float)LAB_BASE * ((float)16 / (float)116 + (float)(i * 5) / (float)(3 * 17 * 29)));
        } else {
            const float fy = (float)(i * 100 * LAB_BASE) / (float)(255 * 116) + (float)(16 * LAB_BASE) / (float)116;
            ify = (int)lrintf(fy);
            volatile float f2 = fy * fy; volatile float f3 = f2 * fy;
            yv = (int)lrintf(f3 / (float)(LAB_BASE * LAB_BASE));
        }
        t.yf[2 * i] = (unsigned short)yv; t.yf[2 * i + 1] = (unsigned short)ify;
    }
    for (int i = 0; i < LAB_INVG_N; i++) {
        const float x = (1.f / 4096.f) * (float)i;
        const double xd = x;
        const float ig = (float)(xd <= 7827. / 2500000. ? xd * (323. / 25.) : pow(xd, 1. / (12. / 5.)) * (1. + 11. / 200.) - 11. / 200.);
        t.invgamma[i] = (unsigned short)lrintf(255.f * ig);
    }
    for (int i = LAB_MIN_AB; i < LAB_ABXZ_N + LAB_MIN_AB; i++)
        t.abxz[i - LAB_MIN_AB] = i <= 3390 ? i * 108 / 841 - LAB_BASE * 16 / 116 * 108 / 841 : i * i / LAB_BASE * i / LAB_BASE;
}

int ensure_lab_tables()
{
    static PerDeviceFlag done_pd; bool& done = done_pd.cur();
    if (done) return B200CV_OK;
    LabHostTabs t;
    build_lab_tabs(t);
    B200_CUDA(cudaMemcpyToSymbol(g_lab_gamma, t.gamma.data(), t.gamma.size() * sizeof(unsigned short)));
    B200_CUDA(cudaMemcpyToSymbol(g_lab_cbrt, t.cbrt.data(), t.cbrt.size() * sizeof(unsigned short)));
    B200_CUDA(cudaMemcpyToSymbol(g_lab_yf, t.yf.data(), t.yf.size() * sizeof(unsigned short)));
    B200_CUDA(cudaMemcpyToSymbol(g_lab_invgamma, t.invgamma.data(), t.invgamma.size() * sizeof(unsigned short)));
    B200_CUDA(cudaMemcpyToSymbol(g_lab_abxz, t.abxz.data(), t.abxz.size() * sizeof(int)));
    done = true;
    return B200CV_OK;
}

struct LabCoef { int c[9]; };

// 8 pixels per thread: 24- / 32-byte row pieces through bytes.cuh (vector accesses when aligned and complete, bytes otherwise)
enum { LAB_PX = 8 };

template <int SCN>
__global__ void __launch_bounds__(256) bgr_to_lab_kernel(Img src, Img dst, int W, LabCoef k, int srgb)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * LAB_PX;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x0 >= W) return;
    const int n = min((int)LAB_PX, W - x0);
    uchar s[LAB_PX * SCN], o[LAB_PX * 3];
    load_bytes<LAB_PX * SCN>(src.row<uchar>(f, y) + (size_t)x0 * SCN, n * SCN, s);
    const int Lscale = (116 * 255 + 50) / 100, Lshift = -((16 * 255 * (1 << 15) + 50) / 100);
#pragma unroll
    for (int i = 0; i < LAB_PX; i++) {
        const int c0 = s[i * SCN], c1 = s[i * SCN + 1], c2 = s[i * SCN + 2];
        const int R = srgb ? g_lab_gamma[c0] : c0 * 8, G = srgb ? g_lab_gamma[c1] : c1 * 8, B = srgb ? g_lab_gamma[c2] : c2 * 8;
        const int fX = g_lab_cbrt[(R * k.c[0] + G * k.c[1] + B * k.c[2] + (1 << 11)) >> 12];
        const int fY = g_lab_cbrt[(R * k.c[3] + G * k.c[4] + B * k.c[5] + (1 << 11)) >> 12];
        const int fZ = g_lab_cbrt[(R * k.c[6] + G * k.c[7] + B * k.c[8] + (1 << 11)) >> 12];
        o[i * 3] = sat_u8((Lscale * fY + Lshift + (1 << 14)) >> 15);
        o[i * 3 + 1] = sat_u8((500 * (fX - fY) + 128 * (1 << 15) + (1 << 14)) >> 15);
        o[i * 3 + 2] = sat_u8((200 * (fY - fZ) + 128 * (1 << 15) + (1 << 14)) >> 15);
    }
    store_bytes<LAB_PX * 3>(dst.row<uchar>(f, y) + (size_t)x0 * 3, n * 3, o);
}

template <int DCN>
__global__ void __launch_bounds__(256) lab_to_bgr_kernel(Img src, Img dst, int W, LabCoef k, int srgb)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * LAB_PX;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x0 >= W) return;
    const int n = min((int)LAB_PX, W - x0);
    uchar s[LAB_PX * 3], o[LAB_PX * DCN];
    load_bytes<LAB_PX * 3>(src.row<uchar>(f, y) + (size_t)x0 * 3, n * 3, s);
#pragma unroll
    for (int i = 0; i < LAB_PX; i++) {
        const int LL = s[i * 3], aa = s[i * 3 + 1], bb = s[i * 3 + 2];
        const int yv = g_lab_yf[LL * 2], ify = g_lab_yf[LL * 2 + 1];
        const int adiv = ((5 * aa * 53687 + (1 << 7)) >> 13) - 128 * LAB_BASE / 500, bdiv = ((bb * 41943 + (1 << 4)) >> 9) - 128 * LAB_BASE / 200 + 1;
        const int xv = g_lab_abxz[ify + adiv - LAB_MIN_AB], zv = g_lab_abxz[ify - bdiv - LAB_MIN_AB];
        int ro = (k.c[0] * xv + k.c[1] * yv + k.c[2] * zv + (1 << 13)) >> 14;
        int go = (k.c[3] * xv + k.c[4] * yv + k.c[5] * zv + (1 << 13)) >> 14;
        int bo = (k.c[6] * xv + k.c[7] * yv + k.c[8] * zv + (1 << 13)) >> 14;
        ro = min(max(ro, 0), LAB_INVG_N - 1); go = min(max(go, 0), LAB_INVG_N - 1); bo = min(max(bo, 0), LAB_INVG_N - 1);
        if (srgb) { ro = g_lab_invgamma[ro]; go = g_lab_invgamma[go]; bo = g_lab_invgamma[bo]; }
        else { ro = ((ro << 8) - ro) >> 12; go = ((go << 8) - go) >> 12; bo = ((bo << 8) - bo) >> 12; }
        o[i * DCN] = sat_u8(bo); o[i * DCN + 1] = sat_u8(go); o[i * DCN + 2] = sat_u8(ro);      // the matrix rows were placed by blueIdx (color_lab.cpp:2434-2436)
        if constexpr (DCN == 4) o[i * DCN + 3] = 255;
    }
    store_bytes<LAB_PX * DCN>(dst.row<uchar>(f, y) + (size_t)x0 * DCN, n * DCN, o);
}

// BGR / RGB <-> CIE XYZ (RGB2XYZ_i<uchar> color_lab.cpp:250-330, XYZ2RGB_i<uchar> :650-730): out = saturate((M * in + 2^11) >> 12), 12-bit integer matrices
template <int SCN, int DCN>
__global__ void __launch_bounds__(256) xyz_matrix_kernel(Img src, Img dst, int W, LabCoef k)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * LAB_PX;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x0 >= W) return;
    const int n = min((int)LAB_PX, W - x0);
    uchar s[LAB_PX * SCN], o[LAB_PX * DCN];
    load_bytes<LAB_PX * SCN>(src.row<uchar>(f, y) + (size_t)x0 * SCN, n * SCN, s);
#pragma unroll
    for (int i = 0; i < LAB_PX; i++) {
        const int s0 = s[i * SCN], s1 = s[i * SCN + 1], s2 = s[i * SCN + 2];
#pragma unroll
        for (int r = 0; r < 3; r++) o[i * DCN + r] = sat_u8((s0 * k.c[3 * r] + s1 * k.c[3 * r + 1] + s2 * k.c[3 * r + 2] + (1 << 11)) >> 12);
        if constexpr (DCN == 4) o[i * DCN + 3] = 255;
    }
    store_bytes<LAB_PX * DCN>(dst.row<uchar>(f, y) + (size_t)x0 * DCN, n * DCN, o);
}

}  // namespace

// codes 32 BGR2XYZ, 33 RGB2XYZ, 34 XYZ2BGR, 35 XYZ2RGB (8-bit)
int cvt_color_xyz(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st)
{
    const int scn = B200CV_CN(src->type), dcn = B200CV_CN(dst->type);
    const bool to_xyz = code == 32 || code == 33, bgr = code == 32 || code == 34;
    B200_REQUIRE(to_xyz ? ((scn == 3 || scn == 4) && dcn == 3) : (scn == 3 && (dcn == 3 || dcn == 4)), "channel count does not match the colour code");
    static const int fwd[9] = {1689, 1465, 739, 871, 2929, 296, 79, 488, 3892}, inv[9] = {13273, -6296, -2042, -3970, 7684, 170, 228, -836, 4331};   // color_lab.cpp:132-144
    LabCoef k;
    for (int i = 0; i < 9; i++) k.c[i] = to_xyz ? fwd[i] : inv[i];
    if (bgr) {
        if (to_xyz) for (int r = 0; r < 3; r++) std::swap(k.c[3 * r], k.c[3 * r + 2]);       // BGR source: swap the matrix columns
        else for (int c = 0; c < 3; c++) std::swap(k.c[c], k.c[6 + c]);                     // BGR destination: swap the rows
    }
    Img s = make_img(src), d = make_img(dst);
    if (s.rows >= 65536 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    const dim3 block(256);
    const dim3 grid(div_up(div_up((unsigned)src->cols, LAB_PX), 256), (unsigned)src->rows, (unsigned)s.frames);
    if (scn == 3 && dcn == 3) xyz_matrix_kernel<3, 3><<<grid, block, 0, st>>>(s, d, src->cols, k);
    else if (scn == 4) xyz_matrix_kernel<4, 3><<<grid, block, 0, st>>>(s, d, src->cols, k);
    else xyz_matrix_kernel<3, 4><<<grid, block, 0, st>>>(s, d, src->cols, k);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

// called by b200cv_cvt_color for codes 44, 45, 74, 75, 56, 57, 78, 79 (8-bit matrices of equal size and batch already checked)
int cvt_color_lab(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st)
{
    const int scn = B200CV_CN(src->type), dcn = B200CV_CN(dst->type);
    const bool to_lab = code == 44 || code == 45 || code == 74 || code == 75;
    const bool srgb = code < 70;
    const int bidx = (code == 44 || code == 74 || code == 56 || code == 78) ? 0 : 2;
    Img s = make_img(src), d = make_img(dst);
    if (s.rows >= 65536 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    int rc = ensure_lab_tables();
    if (rc) return rc;
    static const double wp[3] = {0.950456, 1., 1.088754};
    LabCoef k;
    const dim3 block(256);
    const dim3 grid(div_up(div_up((unsigned)src->cols, LAB_PX), 256), (unsigned)src->rows, (unsigned)s.frames);
    if (to_lab) {
        B200_REQUIRE((scn == 3 || scn == 4) && dcn == 3, "BGR -> Lab needs a 3-/4-channel source and a 3-channel destination");
        static const double M[9] = {0.412453, 0.357580, 0.180423, 0.212671, 0.715160, 0.072169, 0.019334, 0.119193, 0.950227};
        for (int i = 0; i < 3; i++) {
            k.c[i * 3 + (bidx ^ 2)] = (int)nearbyint(4096. * M[i * 3] / wp[i]);
            k.c[i * 3 + 1] = (int)nearbyint(4096. * M[i * 3 + 1] / wp[i]);
            k.c[i * 3 + bidx] = (int)nearbyint(4096. * M[i * 3 + 2] / wp[i]);
        }
        if (scn == 3) bgr_to_lab_kernel<3><<<grid, block, 0, st>>>(s, d, src->cols, k, srgb ? 1 : 0);
        else bgr_to_lab_kernel<4><<<grid, block, 0, st>>>(s, d, src->cols, k, srgb ? 1 : 0);
    } else {
        B200_REQUIRE(scn == 3 && (dcn == 3 || dcn == 4), "Lab -> BGR needs a 3-channel source and a 3-/4-channel destination");
        static const double M[9] = {3.240479, -1.53715, -0.498535, -0.969256, 1.875991, 0.041556, 0.055648, -0.204043, 1.057311};
        for (int i = 0; i < 3; i++) {
            k.c[i + bidx * 3] = (int)nearbyint(4096. * M[i] * wp[i]);
            k.c[i + 3] = (int)nearbyint(4096. * M[i + 3] * wp[i]);
            k.c[i + (bidx ^ 2) * 3] = (int)nearbyint(4096. * M[i + 6] * wp[i]);
        }
        if (dcn == 3) lab_to_bgr_kernel<3><<<grid, block, 0, st>>>(s, d, src->cols, k, srgb ? 1 : 0);
        else lab_to_bgr_kernel<4><<<grid, block, 0, st>>>(s, d, src->cols, k, srgb ? 1 : 0);
    }
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace b200cv
