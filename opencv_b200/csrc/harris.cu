// harris.cu -- cv::cornerHarris / cv::cornerMinEigenVal / cv::goodFeaturesToTrack.
//
// Reference pipeline (cornerEigenValsVecs, modules/imgproc/src/corner.cpp:237-322): five full-frame single-threaded
// passes -- Sobel x, Sobel y (scaled, CV_32F), products (dx^2, dx*dy, dy^2), un-normalised blockSize^2 box sum (f64
// accumulators, box_filter.simd.hpp:1255-1264), response (calcHarris :104-155 / calcMinEigenVal :55-101).
// Here: ONE kernel.  A CTA stages the source tile + apron in shared memory, evaluates both scaled Sobel derivatives and
// the three products for every position of the box apron, resolves the box filter's border on the *product* image
// (exactly where the reference applies it: cv::boxFilter extrapolates cov, not the source), sums the block in fp64 and
// writes the response: 1 byte (or 4) read and 4 bytes written per pixel, no intermediate ever reaches HBM.
//
// goodFeaturesToTrack (modules/imgproc/src/featureselect.cpp:382-548): response map -> per-frame max (warp-shuffle +
// atomic reduction) -> threshold at max*quality (TOZERO) -> 3x3 non-maximum test (== dilate + compare) -> compaction of
// (value, position) candidates on the device; the ordered part (sort by value then address, greedy min-distance
// acceptance on a cell grid) runs on the host over the compacted list, as it is inherently sequential.  The list holds 2^20 candidates
// per frame; a frame with more (a noise frame at 8K has ~2 10^6, a plateau frame up to (W - 2)(H - 2)) makes the list grow to the
// largest count and the candidates be found a second time, so no candidate is ever dropped.
#include <algorithm>
#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cub/device/device_radix_sort.cuh>
#include "common.cuh"

namespace b200cv {

int sobel_taps(int dx, int dy, int ksize, double scale, std::vector<float>& kx, std::vector<float>& ky);

struct HarrisParams {
    float dxk_x[8], dxk_y[8];   // Dx = row pass with dxk_x, column pass with dxk_y
    float dyk_x[8], dyk_y[8];
    int ks;                     // taps per direction (3 for ksize 1|3, 5, 7)
    int bs, ba;                 // box size and anchor (bs/2)
    int border;
    float k;
    int op;                     // 0 = Harris, 1 = min eigen value
    int skip_interior;          // the tile kernel leaves the tiles harris_fast_kernel owns alone
};

constexpr int H_TW = 128, H_TH = 16;
// tiles of harris_fast_kernel (below): columns per warp (32 lanes x 4), rows per warp; the predicate says which tiles it owns
constexpr int HF_W = 128, HF_SEG = 64;
__host__ __device__ __forceinline__ bool harris_fast_tile(int x0, int y0, int W, int H, int bs)
{
    const int R = bs + 2;                    // products reach bs - 1 - ba <= bs, the Sobel one more
    return x0 - R - 4 >= 0 && x0 + HF_W + R + 4 <= W && y0 - R >= 0 && y0 + HF_SEG + R <= H;
}

// KS = Sobel taps per direction (3 / 5 / 7), BS = box size when small (2 / 3 / 5), 0 = run-time box size
template <typename ST, int KS, int BS>
__global__ void __launch_bounds__(256) harris_kernel(Img src, Img dst, const __grid_constant__ HarrisParams p)
{
    extern __shared__ __align__(16) float smem[];
    constexpr int rs = KS / 2;
    const int bs = BS ? BS : p.bs;
    const int cw = H_TW + bs - 1, ch = H_TH + bs - 1;             // product (cov) region
    const int sw_ = cw + 2 * rs, sh_ = ch + 2 * rs;               // source region
    float* s_src = smem;                                          // sh_ x sw_
    float* s_rx = s_src + sw_ * sh_;                              // sh_ x cw : row pass with the Dx row taps
    float* s_ry = s_rx + sh_ * cw;                                // sh_ x cw : row pass with the Dy row taps
    // the three product images (float); rows padded to an even length so that pairs load as 64-bit words
    const int cwp = cw + (cw & 1);
    float* s_a = s_ry + sh_ * cw + ((sw_ * sh_ + 2 * sh_ * cw) & 1);   // ch x cwp : dx*dx   (8-byte aligned)
    float* s_b = s_a + cwp * ch;                                  //            dx*dy
    float* s_c = s_b + cwp * ch;                                  //            dy*dy
    const int f = blockIdx.z, x0 = blockIdx.x * H_TW, y0 = blockIdx.y * H_TH;
    const int cx0 = x0 - p.ba, cy0 = y0 - p.ba;                   // image coordinates of cov region origin
    const int W = src.cols, H = src.rows;
    if (p.skip_interior && harris_fast_tile(x0, (y0 / HF_SEG) * HF_SEG, W, H, bs)) return;       // harris_fast_kernel's tile

    // one warp per staged row, lanes over columns (no per-element division); interior tiles skip the border arithmetic
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool interior = cx0 - rs >= 0 && cy0 - rs >= 0 && cx0 - rs + sw_ <= W && cy0 - rs + sh_ <= H;
    for (int r = warp; r < sh_; r += 8) {
        const int sy = interior ? cy0 - rs + r : border_interpolate(cy0 - rs + r, H, p.border);
        const ST* srow = sy >= 0 ? src.row<ST>(f, sy) : nullptr;
        float* drow = s_src + r * sw_;
        for (int c = lane; c < sw_; c += 32) {
            const int sx = interior ? cx0 - rs + c : border_interpolate(cx0 - rs + c, W, p.border);
            float v = 0.f;
            if (srow && sx >= 0) {
                if constexpr (sizeof(ST) == 1) v = __fsub_rn(__uint_as_float(0x4B000000u | (uint32_t)srow[sx]), 8388608.0f);   // byte -> float through the mantissa of 2^23 (I2F is quarter rate)
                else v = (float)srow[sx];
            }
            drow[c] = v;
        }
    }
    __syncthreads();
    // row pass (both derivative filters share the staged source row)
    for (int r = warp; r < sh_; r += 8)
    for (int c = lane; c < cw; c += 32) {
        const int idx = r * cw + c;
        const float* row = s_src + r * sw_ + c;
        float rx = 0.f, ry = 0.f;
        // Same operation order as the reference's Sobel = sepFilter2D (filter.simd.hpp, see sep_f32.cu): 8-bit rows and 7-tap float
        // rows in tap order with FMA; 3/5-tap float rows centre-out (Dx row kernel antisymmetric, Dy row kernel symmetric)
        if constexpr (sizeof(ST) == 4 && KS <= 5) {
            constexpr int m = KS / 2;
            rx = __fmul_rn(__fsub_rn(row[m + 1], row[m - 1]), p.dxk_x[m + 1]);
            ry = fmaf(row[m], p.dyk_x[m], __fmul_rn(__fadd_rn(row[m - 1], row[m + 1]), p.dyk_x[m + 1]));
            if constexpr (KS == 5) {
                rx = fmaf(__fsub_rn(row[m + 2], row[m - 2]), p.dxk_x[m + 2], rx);
                ry = fmaf(__fadd_rn(row[m - 2], row[m + 2]), p.dyk_x[m + 2], ry);
            }
        } else {
#pragma unroll
            for (int i = 0; i < KS; i++) { rx = fmaf(row[i], p.dxk_x[i], rx); ry = fmaf(row[i], p.dyk_x[i], ry); }
        }
        s_rx[idx] = rx; s_ry[idx] = ry;
    }
    __syncthreads();
    // column pass + products at the in-image positions of the cov region
    for (int r = warp; r < ch; r += 8)
    for (int c = lane; c < cw; c += 32) {
        const int idx = r * cwp + c;
        int gx = cx0 + c, gy = cy0 + r;
        if ((unsigned)gx >= (unsigned)W || (unsigned)gy >= (unsigned)H) continue;
        // columns: mirrored rows first (Dx column kernel symmetric, Dy column kernel antisymmetric; delta = 0)
        constexpr int m = KS / 2;
        float dx = fmaf(p.dxk_y[m], s_rx[(r + m) * cw + c], 0.f), dy = 0.f;
#pragma unroll
        for (int j = 1; j <= m; j++) {
            dx = fmaf(p.dxk_y[m + j], __fadd_rn(s_rx[(r + m + j) * cw + c], s_rx[(r + m - j) * cw + c]), dx);
            dy = fmaf(p.dyk_y[m + j], __fsub_rn(s_ry[(r + m + j) * cw + c], s_ry[(r + m - j) * cw + c]), dy);
        }
        s_a[idx] = __fmul_rn(dx, dx); s_b[idx] = __fmul_rn(dx, dy); s_c[idx] = __fmul_rn(dy, dy);
    }
    __syncthreads();
    // the box filter's border: out-of-image positions take the products of the border-interpolated position (or 0);
    // only CTAs on the image boundary have any
    if (cx0 < 0 || cy0 < 0 || cx0 + cw > W || cy0 + ch > H) {
        for (int i = threadIdx.x; i < cw * ch; i += 256) {
            int r = i / cw, c = i - r * cw;
            const int idx = r * cwp + c;
            int gx = cx0 + c, gy = cy0 + r;
            if ((unsigned)gx < (unsigned)W && (unsigned)gy < (unsigned)H) continue;
            int qx = border_interpolate(gx, W, p.border), qy = border_interpolate(gy, H, p.border);
            int qc = qx - cx0, qr = qy - cy0;
            if (qx < 0 || qy < 0 || qc < 0 || qc >= cw || qr < 0 || qr >= ch) { s_a[idx] = s_b[idx] = s_c[idx] = 0.f; continue; }
            int q = qr * cwp + qc;
            s_a[idx] = s_a[q]; s_b[idx] = s_b[q]; s_c[idx] = s_c[q];
        }
        __syncthreads();
    }
    auto response = [&](double a, double b, double cc) -> float {
        float fa = (float)a, fb = (float)b, fc = (float)cc;
        if (p.op == 0) {
            float acbb = __fsub_rn(__fmul_rn(fa, fc), __fmul_rn(fb, fb));
            float ac = __fadd_rn(fa, fc);
            return __fsub_rn(acbb, __fmul_rn(p.k, __fmul_rn(ac, ac)));     // calcHarrisLine_AVX: k * ((a+c)*(a+c)), no FMA (corner.avx.cpp:145-160)
        }
        float ha = __fmul_rn(fa, 0.5f), hc = __fmul_rn(fc, 0.5f);
        float t = __fsub_rn(ha, hc);
        t = __fadd_rn(__fmul_rn(fb, fb), __fmul_rn(t, t));
        return __fsub_rn(__fadd_rn(ha, hc), __fsqrt_rn(t));
    };
    if constexpr (BS == 2 || BS == 3) {
        // four adjacent outputs per thread: the 4 + BS - 1 products of a row are loaded once (64-bit words), converted once (F2F.F64.F32 issues at
        // 16 lanes / clk / SM: 4 BS^2 conversions per pixel and array were a third of the kernel) and shared by the four horizontal sums
        // (added left to right, then rows top to bottom: the order of the scalar loop below); one 16-byte store
        for (int item = threadIdx.x; item < (H_TW / 4) * H_TH; item += 256) {
            const int r = item / (H_TW / 4), c = (item - r * (H_TW / 4)) * 4;
            const int gx = x0 + c, gy = y0 + r;
            if (gx >= W || gy >= H) continue;
            double sa[4] = {0, 0, 0, 0}, sb[4] = {0, 0, 0, 0}, sc[4] = {0, 0, 0, 0};
#pragma unroll
            for (int j = 0; j < BS; j++) {
                const int o = (r + j) * cwp + c;                  // even: 8-byte aligned
                double va[6], vb[6], vc[6];
#pragma unroll
                for (int q = 0; q < 3; q++) {
                    const float2 ta = *(const float2*)(s_a + o + 2 * q), tb = *(const float2*)(s_b + o + 2 * q), tc = *(const float2*)(s_c + o + 2 * q);
                    va[2 * q] = ta.x; vb[2 * q] = tb.x; vc[2 * q] = tc.x;
                    if (2 * q + 1 < 4 + BS - 1) { va[2 * q + 1] = ta.y; vb[2 * q + 1] = tb.y; vc[2 * q + 1] = tc.y; }
                }
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    double ra = va[i], rb = vb[i], rc = vc[i];
#pragma unroll
                    for (int t = 1; t < BS; t++) { ra += va[i + t]; rb += vb[i + t]; rc += vc[i + t]; }
                    sa[i] += ra; sb[i] += rb; sc[i] += rc;
                }
            }
            float o4[4];
#pragma unroll
            for (int i = 0; i < 4; i++) o4[i] = response(sa[i], sb[i], sc[i]);
            float* dp = dst.row<float>(f, gy) + gx;
            if (gx + 4 <= W && ((uintptr_t)dp & 15) == 0) *(float4*)dp = make_float4(o4[0], o4[1], o4[2], o4[3]);
            else for (int i = 0; i < 4 && gx + i < W; i++) dp[i] = o4[i];
        }
    } else {
        for (int idx = threadIdx.x; idx < H_TW * H_TH; idx += 256) {
            int r = idx / H_TW, c = idx - r * H_TW;
            int gx = x0 + c, gy = y0 + r;
            if (gx >= W || gy >= H) continue;
            double a = 0, b = 0, cc = 0;
            for (int j = 0; j < bs; j++) {
                int o = (r + j) * cwp + c;
                double ra = 0, rb = 0, rc = 0;
                for (int i = 0; i < bs; i++) { ra += (double)s_a[o + i]; rb += (double)s_b[o + i]; rc += (double)s_c[o + i]; }
                a += ra; b += rb; cc += rc;
            }
            dst.row<float>(f, gy)[gx] = response(a, b, cc);
        }
    }
}

// ---- second version for the common case (3-tap Sobel, block size 2 or 3): register marching, interior tiles only ------------------------------
// The tile kernel above spends ~140 thread instructions per pixel on staging, three shared-memory passes and 4 BS^2 float -> double conversions
// (issue-bound at 25 % occupancy).  Here a THREAD owns 4 adjacent output columns and walks down HF_SEG rows:
// the 3-row windows of the two row-filtered derivative images, the current product row and the horizontal box sums of the previous BS - 1
// product rows all live in registers (the row loop is unrolled by 6 = lcm(3, 2) so every ring index is a compile-time constant); a product is
// converted to double once; no shared memory, no barrier; one 16-byte store per thread and row.  Arithmetic and operation order are the tile
// kernel's (= the reference's): same Sobel chains, products rounded to float, box sums left to right then top to bottom in f64.
// Tiles that touch the image border (where the box filter's border rule lands on the PRODUCT image) stay with the tile kernel: it skips the
// tiles this kernel owns (HarrisParams::skip_interior).
template <typename ST, int BS>
__global__ void __launch_bounds__(128) harris_fast_kernel(Img src, Img dst, const __grid_constant__ HarrisParams p)
{
    constexpr int BA = BS / 2, NP = 4 + BS - 1, NS = NP + 2;           // product columns / source columns per thread
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tx = blockIdx.x * 4 + warp;                                 // 4 strips per CTA
    const int x0 = tx * HF_W, y0 = blockIdx.y * HF_SEG, f = blockIdx.z;
    if (x0 >= src.cols || !harris_fast_tile(x0, y0, src.cols, src.rows, BS)) return;
    const int X = x0 + 4 * lane;                                          // first output column
    const int xs = X - BA - 1;                                            // first source column
    // source row -> NS floats in two steps, so that the NEXT row's loads are in flight while this row is processed (the first version consumed
    // each load at once: 43 % of its stall samples sat on the first instruction after the LDG): fetch = raw words / floats, decode = bytes
    // through the mantissa of 2^23 (the thread's bytes sit in 3 aligned words: one funnel shift each, then compile-time PRMTs)
    constexpr int NRAW = sizeof(ST) == 1 ? 4 : NS;
    const int a0 = (xs & ~3);
    auto fetch = [&](int gy, unsigned* raw) {
        if constexpr (sizeof(ST) == 1) {
            const uchar* rp = src.row<uchar>(f, gy);
            if ((((uintptr_t)rp) & 3) == 0) {
#pragma unroll
                for (int i = 0; i < 4; i++) raw[i] = __ldg((const unsigned*)(rp + a0) + i);
            } else {
#pragma unroll
                for (int i = 0; i < 4; i++) raw[i] = (unsigned)rp[a0 + 4 * i] | ((unsigned)rp[a0 + 4 * i + 1] << 8) | ((unsigned)rp[a0 + 4 * i + 2] << 16) | ((unsigned)rp[a0 + 4 * i + 3] << 24);
            }
        } else {
            const float* rp = src.row<float>(f, gy) + xs;
#pragma unroll
            for (int j = 0; j < NS; j++) raw[j] = __float_as_uint(__ldg(rp + j));
        }
    };
    auto decode = [&](const unsigned* raw, float* sv) {
        if constexpr (sizeof(ST) == 1) {
            const unsigned sh8 = 8u * (unsigned)(xs - a0);                // the same for every lane (X % 4 == 0)
            unsigned v[3];
#pragma unroll
            for (int i = 0; i < 3; i++) v[i] = __funnelshift_r(raw[i], raw[i + 1], sh8);
#pragma unroll
            for (int j = 0; j < NS; j++) sv[j] = __fsub_rn(__uint_as_float(__byte_perm(v[j >> 2], 0x4B000000u, 0x7650 + (j & 3))), 8388608.0f);
        } else {
#pragma unroll
            for (int j = 0; j < NS; j++) sv[j] = __uint_as_float(raw[j]);
        }
    };
    // row pass of one source row: the two derivative row filters at the NP product columns
    auto row_pass = [&](const float* sv, float* rx, float* ry) {
#pragma unroll
        for (int j = 0; j < NP; j++) {
            if constexpr (sizeof(ST) == 4) {       // float source, 3 taps: centre-out (SymmRowSmallVec_32f order, as the tile kernel)
                rx[j] = __fmul_rn(__fsub_rn(sv[j + 2], sv[j]), p.dxk_x[2]);
                ry[j] = fmaf(sv[j + 1], p.dyk_x[1], __fmul_rn(__fadd_rn(sv[j], sv[j + 2]), p.dyk_x[2]));
            } else {                               // 8-bit source: tap order with FMA from 0
                float a = 0.f, b = 0.f;
#pragma unroll
                for (int i = 0; i < 3; i++) { a = fmaf(sv[j + i], p.dxk_x[i], a); b = fmaf(sv[j + i], p.dyk_x[i], b); }
                rx[j] = a; ry[j] = b;
            }
        }
    };
    float rxw[3][NP], ryw[3][NP];                  // row-filtered rows r - 2, r - 1, r (ring by r % 3)
    double hb[BS > 1 ? BS - 1 : 1][4][3];          // horizontal box sums of the previous BS - 1 product rows (ring by q % (BS - 1))
    // source rows: products exist from row y0 - BA (needs source rows y0 - BA - 1 ..); walk r = first source row ...
    const int r_first = y0 - BA - 1, r_last = y0 + HF_SEG - 1 + (BS - 1 - BA) + 1;      // inclusive
    float sv[NS];
    unsigned raw[2][NRAW];
    int r = r_first;
    fetch(r, raw[0]);
    // the unrolled-by-6 loop body handles source row r with compile-time ring slots it % 3 and it % (BS - 1)
#pragma unroll 1
    for (int base = 0; r <= r_last; base += 6) {
#pragma unroll
        for (int it = 0; it < 6; it++, r++) {
            if (r > r_last) break;
            if (r < r_last) fetch(r + 1, raw[(it + 1) % 2]);
            decode(raw[it % 2], sv);
            row_pass(sv, rxw[it % 3], ryw[it % 3]);
            const int n = base + it;                                  // source rows seen before this one
            if (n < 2) continue;                                      // need rows r - 2 .. r
            // product row q = r - 1: column pass (mirrored rows first) + products
            const int q = r - 1;
            const float* rm = rxw[(it + 1) % 3]; const float* rc = rxw[(it + 2) % 3]; const float* rp_ = rxw[it % 3];       // rows r - 2, r - 1, r
            const float* sm = ryw[(it + 1) % 3]; const float* sp_ = ryw[it % 3];
            double pa[NP], pb[NP], pc[NP];
#pragma unroll
            for (int j = 0; j < NP; j++) {
                float dx = fmaf(p.dxk_y[1], rc[j], 0.f);
                dx = fmaf(p.dxk_y[2], __fadd_rn(rp_[j], rm[j]), dx);
                float dy = fmaf(p.dyk_y[2], __fsub_rn(sp_[j], sm[j]), 0.f);
                pa[j] = (double)__fmul_rn(dx, dx); pb[j] = (double)__fmul_rn(dx, dy); pc[j] = (double)__fmul_rn(dy, dy);
            }
            // horizontal sums of this product row at the 4 output columns
            double ha[4], hbv[4], hc[4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                double a = pa[i], b = pb[i], c = pc[i];
#pragma unroll
                for (int t = 1; t < BS; t++) { a += pa[i + t]; b += pb[i + t]; c += pc[i + t]; }
                ha[i] = a; hbv[i] = b; hc[i] = c;
            }
            // output row y = q - (BS - 1 - BA): its box = product rows y - BA .. q, top to bottom
            const int y = q - (BS - 1 - BA);
            const int nq = n - 2;                                     // product rows seen before this one
            if (nq >= BS - 1 && y >= y0 && y < y0 + HF_SEG) {
                float o4[4];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    double a = 0, b = 0, c = 0;
#pragma unroll
                    for (int t = BS - 1; t >= 1; t--) {               // oldest first: product row q - t sits in ring slot (nq - t) % (BS - 1)
                        constexpr int M = BS > 1 ? BS - 1 : 1;
                        const int slot = ((it + 6 * 4 - 2 - t) % M);   // (nq - t) % M with nq = base + it - 2 and base % 6 == 0, 6 % M == 0
                        a += hb[slot][i][0]; b += hb[slot][i][1]; c += hb[slot][i][2];
                    }
                    a += ha[i]; b += hbv[i]; c += hc[i];
                    const float fa = (float)a, fb = (float)b, fc = (float)c;
                    if (p.op == 0) {
                        const float acbb = __fsub_rn(__fmul_rn(fa, fc), __fmul_rn(fb, fb));
                        const float ac = __fadd_rn(fa, fc);
                        o4[i] = __fsub_rn(acbb, __fmul_rn(p.k, __fmul_rn(ac, ac)));
                    } else {
                        const float hA = __fmul_rn(fa, 0.5f), hC = __fmul_rn(fc, 0.5f);
                        float t = __fsub_rn(hA, hC);
                        t = __fadd_rn(__fmul_rn(fb, fb), __fmul_rn(t, t));
                        o4[i] = __fsub_rn(__fadd_rn(hA, hC), __fsqrt_rn(t));
                    }
                }
                float* dp = dst.row<float>(f, y) + X;
                if ((((uintptr_t)dp) & 15) == 0) *(float4*)dp = make_float4(o4[0], o4[1], o4[2], o4[3]);
                else { dp[0] = o4[0]; dp[1] = o4[1]; dp[2] = o4[2]; dp[3] = o4[3]; }
            }
            if constexpr (BS > 1) {
                constexpr int M = BS - 1;
                const int slot = (it + 6 * 4 - 2) % M;                // nq % M
#pragma unroll
                for (int i = 0; i < 4; i++) { hb[slot][i][0] = ha[i]; hb[slot][i][1] = hbv[i]; hb[slot][i][2] = hc[i]; }
            }
        }
    }
}

template <typename ST, int KS, int BS>
static int launch_harris(const Img& s, const Img& d, const HarrisParams& p, cudaStream_t st)
{
    const int rs = KS / 2, cw = H_TW + p.bs - 1, ch = H_TH + p.bs - 1, sw_ = cw + 2 * rs, sh_ = ch + 2 * rs;
    const int cwp = cw + (cw & 1);
    size_t smem = ((size_t)sw_ * sh_ + 2 * (size_t)sh_ * cw + 1 + 3 * (size_t)cwp * ch) * sizeof(float);
    auto kern = harris_kernel<ST, KS, BS>;
    static PerDeviceFlag a_pd; bool& a = a_pd.cur();
    if (!a) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); a = true; }
    if (smem > 200 * 1024) return B200CV_NOT_IMPLEMENTED;
    dim3 grid(div_up((unsigned)s.cols, H_TW), div_up((unsigned)s.rows, H_TH), (unsigned)s.frames);
    kern<<<grid, 256, smem, st>>>(s, d, p);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

template <typename ST, int KS>
static int launch_harris_bs(const Img& s, const Img& d, const HarrisParams& p, cudaStream_t st)
{
    if constexpr (KS == 3) {
        // 3-tap Sobel with a 2 x 2 or 3 x 3 block (cornerHarris / goodFeaturesToTrack defaults): interior tiles on the register-marching kernel,
        // the border ring on the tile kernel (B200CV_HARRIS_PATH=tile: everything on the tile kernel)
        const char* path = getenv("B200CV_HARRIS_PATH");
        const bool any_fast = s.cols >= HF_W + 2 * (p.bs + 6) && s.rows >= HF_SEG + 2 * (p.bs + 2);
        if ((p.bs == 2 || p.bs == 3) && any_fast && !(path && !strcmp(path, "tile"))) {
            HarrisParams q = p;
            q.skip_interior = 1;
            dim3 grid(div_up(div_up((unsigned)s.cols, HF_W), 4), div_up((unsigned)s.rows, HF_SEG), (unsigned)s.frames);
            if (p.bs == 2) harris_fast_kernel<ST, 2><<<grid, 128, 0, st>>>(s, d, q);
            else harris_fast_kernel<ST, 3><<<grid, 128, 0, st>>>(s, d, q);
            B200_LAUNCH_CHECK();
            return p.bs == 2 ? launch_harris<ST, KS, 2>(s, d, q, st) : launch_harris<ST, KS, 3>(s, d, q, st);
        }
    }
    switch (p.bs) {
    case 2: return launch_harris<ST, KS, 2>(s, d, p, st);
    case 3: return launch_harris<ST, KS, 3>(s, d, p, st);
    case 5: return launch_harris<ST, KS, 5>(s, d, p, st);
    default: return launch_harris<ST, KS, 0>(s, d, p, st);
    }
}

template <typename ST>
static int launch_harris_ks(const Img& s, const Img& d, const HarrisParams& p, cudaStream_t st)
{
    switch (p.ks) {
    case 3: return launch_harris_bs<ST, 3>(s, d, p, st);
    case 5: return launch_harris_bs<ST, 5>(s, d, p, st);
    case 7: return launch_harris_bs<ST, 7>(s, d, p, st);
    }
    return B200CV_NOT_IMPLEMENTED;
}

int corner_response(const b200cvMat* src, const b200cvMat* dst, int block_size, int ksize, double k, int border, int op, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->cols == dst->cols && src->rows == dst->rows, "src/dst size mismatch");
    B200_REQUIRE(dst->type == B200CV_MAKETYPE(B200CV_32F, 1), "corner response must be CV_32FC1");
    B200_REQUIRE(src->type == B200CV_MAKETYPE(B200CV_8U, 1) || src->type == B200CV_MAKETYPE(B200CV_32F, 1), "source must be CV_8UC1 or CV_32FC1");
    B200_REQUIRE(block_size > 0, "blockSize must be positive");
    border &= ~B200CV_BORDER_ISOLATED;
    if (border < 0 || border > B200CV_BORDER_REFLECT_101 || border == B200CV_BORDER_WRAP) return B200CV_NOT_IMPLEMENTED;
    if (block_size > 31 || (ksize != 1 && ksize != 3 && ksize != 5 && ksize != 7)) return B200CV_NOT_IMPLEMENTED;   // Scharr (ksize<0): next
    const bool u8 = B200CV_DEPTH(src->type) == B200CV_8U;
    // corner.cpp:247-252
    double scale = (double)(1 << (ksize - 1)) * block_size;
    if (u8) scale *= 255.0;
    scale = 1.0 / scale;
    std::vector<float> xkx, xky, ykx, yky;
    if ((rc = sobel_taps(1, 0, ksize, scale, xkx, xky)) || (rc = sobel_taps(0, 1, ksize, scale, ykx, yky))) return rc;
    HarrisParams p;
    memset(&p, 0, sizeof(p));
    // ksize 1: 3 taps along the derivative, 1 across; embed the 1-tap kernels centred in 3 taps
    int ks = (int)std::max(std::max(xkx.size(), xky.size()), std::max(ykx.size(), yky.size()));
    auto put = [&](float* d, const std::vector<float>& v) { int o = (ks - (int)v.size()) / 2; for (size_t i = 0; i < v.size(); i++) d[o + i] = v[i]; };
    put(p.dxk_x, xkx); put(p.dxk_y, xky); put(p.dyk_x, ykx); put(p.dyk_y, yky);
    p.ks = ks; p.bs = block_size; p.ba = block_size / 2; p.border = border; p.k = (float)k; p.op = op;
    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    cudaStream_t st = as_stream(stream);
    return u8 ? launch_harris_ks<uchar>(s, d, p, st) : launch_harris_ks<float>(s, d, p, st);
}

// ---- goodFeaturesToTrack device side --------------------------------------------------------------------------------
// order-preserving float <-> uint mapping for atomicMax
__device__ __forceinline__ unsigned f2ord(float v) { unsigned u = __float_as_uint(v); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__host__ __device__ __forceinline__ float ord2f(unsigned o) {
    unsigned u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

// eig is the function's own response map: base and pitch are multiples of 256 bytes, so 4-column groups load as one float4
__device__ __forceinline__ float4 eig_ld4(const float* r, int x, int W)
{
    if (x + 3 < W) return __ldg(reinterpret_cast<const float4*>(r + x));
    float4 v = {0.f, 0.f, 0.f, 0.f};
    if (x < W) v.x = __ldg(r + x);
    if (x + 1 < W) v.y = __ldg(r + x + 1);
    if (x + 2 < W) v.z = __ldg(r + x + 2);
    return v;
}
__global__ void __launch_bounds__(256) frame_max_kernel(Img eig, unsigned* maxord)
{
    const int f = blockIdx.y, W = eig.cols;
    unsigned best = 0;    // below every real value's code
    for (int y = blockIdx.x; y < eig.rows; y += gridDim.x) {
        const float* r = eig.row<float>(f, y);
        for (int x = threadIdx.x * 4; x < W; x += 1024) {
            if (x + 3 < W) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(r + x));
                best = max(max(best, f2ord(v.x)), max(f2ord(v.y), max(f2ord(v.z), f2ord(v.w))));
            } else
                for (int i = x; i < W; i++) best = max(best, f2ord(__ldg(r + i)));
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((threadIdx.x & 31) == 0) atomicMax(maxord + f, best);
}

// candidate key: order-preserving bits of the response in the high word, row-major position in the low word.  Sorting keys
// descending = strongest first, equal responses: larger address first (featureselect.cpp:55-60).
typedef unsigned long long CandKey;
constexpr int GF_BINS = 4096, GF_TOP_MIN = 1 << 15, GF_TOP_CAP = 1 << 17;
constexpr int GC_R = 8;        // rows per tile of the candidate kernel (4 columns x GC_R rows per thread: one bit each in a 32-bit mask)

// Candidates = pixels that survive threshold(eig, max * quality, TOZERO) and equal the 3x3 maximum of the thresholded map (dilate + compare,
// modules/imgproc/src/featureselect.cpp:127-166), 1-pixel frame excluded.  A thread walks down GC_R rows of 4 columns with the three window rows in
// registers; the block reserves its output range with ONE atomic per 1024 x GC_R tile (a per-candidate atomic on the frame's counter serialises
// on a noisy frame with many candidates); the histogram of the response codes' top 12 bits (for the top-K
// preselection below) is kept in shared memory and flushed once per block.
__global__ void __launch_bounds__(256) gftt_candidates_kernel(Img eig, const unsigned* maxord, double quality, CandKey* out, int cap, int* counts, unsigned* hist)
{
    __shared__ unsigned s_hist[GF_BINS];
    __shared__ int s_warp[8];
    __shared__ int s_base;
    const int f = blockIdx.y, W = eig.cols, H = eig.rows;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (hist) {
        for (int i = tid; i < GF_BINS; i += 256) s_hist[i] = 0;
        __syncthreads();
    }
    const float thr = (float)((double)ord2f(maxord[f]) * quality);            // threshold(eig, maxVal*qualityLevel, TOZERO) compares in float
    const int tx = (W + 1023) / 1024, ty = (H + GC_R - 1) / GC_R;
    // columns x0-1 .. x0+4 of row y, thresholded; rows / columns outside the image only feed centres that are excluded anyway
    auto load_row = [&](int y, int x0, float (&a)[6]) {
        if (y < 0 || y >= H || x0 >= W) { a[0] = a[1] = a[2] = a[3] = a[4] = a[5] = 0.f; return; }
        const float* r = eig.row<float>(f, y);
        const float4 v = eig_ld4(r, x0, W);
        a[0] = x0 > 0 ? __ldg(r + x0 - 1) : 0.f;
        a[1] = v.x; a[2] = v.y; a[3] = v.z; a[4] = v.w;
        a[5] = x0 + 4 < W ? __ldg(r + x0 + 4) : 0.f;
#pragma unroll
        for (int i = 0; i < 6; i++) a[i] = a[i] > thr ? a[i] : 0.f;
    };
    for (int t = blockIdx.x; t < tx * ty; t += gridDim.x) {
        const int y0 = (t / tx) * GC_R, x0 = (t % tx) * 1024 + tid * 4;
        unsigned mask = 0;
        if (x0 < W) {
            float a[6], b[6], c[6];
            load_row(y0 - 1, x0, a);
            load_row(y0, x0, b);
#pragma unroll
            for (int r = 0; r < GC_R; r++) {
                const int y = y0 + r;
                load_row(y + 1, x0, c);
                float m[6];
#pragma unroll
                for (int i = 0; i < 6; i++) m[i] = fmaxf(fmaxf(a[i], b[i]), c[i]);
                if (y >= 1 && y < H - 1) {
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const float v = b[j + 1];
                        const int x = x0 + j;
                        if (v != 0.f && x >= 1 && x < W - 1 && !(fmaxf(fmaxf(m[j], m[j + 1]), m[j + 2]) > v)) mask |= 1u << (r * 4 + j);
                    }
                }
#pragma unroll
                for (int i = 0; i < 6; i++) { a[i] = b[i]; b[i] = c[i]; }
            }
        }
        const int cnt = __popc(mask);
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
        if (lane == 31) s_warp[wid] = incl;
        __syncthreads();
        if (tid == 0) {
            int tot = 0;
#pragma unroll
            for (int w = 0; w < 8; w++) { const int c = s_warp[w]; s_warp[w] = tot; tot += c; }
            s_base = tot ? atomicAdd(counts + f, tot) : 0;
        }
        __syncthreads();
        int slot = s_base + s_warp[wid] + incl - cnt;
        while (mask) {
            const int bit = __ffs(mask) - 1;
            mask &= mask - 1;
            const int y = y0 + (bit >> 2), x = x0 + (bit & 3);
            const unsigned code = f2ord(__ldg(eig.row<float>(f, y) + x));
            if (slot < cap) {
                out[(size_t)f * cap + slot] = ((CandKey)code << 32) | (unsigned)(y * W + x);
                if (hist) atomicAdd(&s_hist[code >> 20], 1u);
            }
            slot++;
        }
    }
    if (hist) {
        __syncthreads();
        for (int i = tid; i < GF_BINS; i += 256)
            if (s_hist[i]) atomicAdd(hist + (size_t)f * GF_BINS + i, s_hist[i]);
    }
}

// ---- top-K preselection: the greedy walk normally stops after a few thousand candidates, a noisy 4K frame has ~10^6 -----------------------
// histogram of the top 12 bits of the (order-preserving) response code -> the highest bins that hold at least GF_TOP_MIN candidates ->
// compaction of exactly those candidates.  Sorting them gives the PREFIX of the full descending order (every stronger candidate is in), so
// the walk is the reference's as long as it ends inside the prefix; if it runs out, the frame is redone with the full sort.
__global__ void __launch_bounds__(128) gftt_select_kernel(const unsigned* hist, int* thr_bin)
{
    __shared__ unsigned part[128];
    const int f = blockIdx.x, t = threadIdx.x;
    const unsigned* h = hist + (size_t)f * GF_BINS;
    unsigned sum = 0;
    for (int i = 0; i < 32; i++) sum += h[t * 32 + i];
    part[t] = sum;
    __syncthreads();
    if (t) return;
    unsigned cum = 0;
    int g = 127;
    for (; g > 0 && cum + part[g] < (unsigned)GF_TOP_MIN; g--) cum += part[g];
    int b = g * 32 + 31;
    for (; b > g * 32; b--) { cum += h[b]; if (cum >= (unsigned)GF_TOP_MIN) break; }
    thr_bin[f] = b;
}
__global__ void __launch_bounds__(256) gftt_filter_kernel(const CandKey* cand, const int* counts, int cap, const int* thr_bin, CandKey* top, int* top_cnt)
{
    const int f = blockIdx.y, n = min(counts[f], cap), tb = thr_bin[f];
    const CandKey* c = cand + (size_t)f * cap;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
        const CandKey k = c[i];
        if ((int)(k >> 52) >= tb) {
            const int slot = atomicAdd(top_cnt + f, 1);
            if (slot < GF_TOP_CAP) top[(size_t)f * GF_TOP_CAP + slot] = k;
        }
    }
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_corner_harris(const b200cvMat* src, const b200cvMat* dst, int block_size, int ksize, double k, int border, void* stream)
{
    return corner_response(src, dst, block_size, ksize, k, border, 0, stream);
}

extern "C" int b200cv_corner_min_eigen_val(const b200cvMat* src, const b200cvMat* dst, int block_size, int ksize, int border, void* stream)
{
    return corner_response(src, dst, block_size, ksize, 0.0, border, 1, stream);
}

extern "C" int b200cv_good_features_to_track(const b200cvMat* src, float* corners, float* quality, int max_out, int* counts,
                                             int max_corners, double quality_level, double min_distance, int block_size,
                                             int gradient_size, int use_harris, double k, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src"))) return rc;
    B200_REQUIRE(corners && counts && max_out > 0, "bad output arguments");
    B200_REQUIRE(quality_level > 0 && min_distance >= 0 && max_corners >= 0, "bad parameters");
    const int W = src->cols, H = src->rows, frames = src->frames > 1 ? src->frames : 1;
    cudaStream_t st = as_stream(stream);
    // workspace: response map + per-frame max + candidate list
    float* d_eig = nullptr; unsigned* d_max = nullptr; int* d_cnt = nullptr; CandKey* d_cand = nullptr; CandKey* d_sorted = nullptr; void* d_tmp = nullptr;
    size_t pitch = ((size_t)W * 4 + 255) & ~(size_t)255;
    int cap = (int)std::min<long long>((long long)W * H, 1 << 20);
    auto cleanup = [&]() {
        cudaFreeAsync(d_eig, st); cudaFreeAsync(d_max, st); cudaFreeAsync(d_cnt, st); cudaFreeAsync(d_cand, st);
        if (d_sorted) cudaFreeAsync(d_sorted, st);
        if (d_tmp) cudaFreeAsync(d_tmp, st);
    };
#define TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { cleanup(); return cuda_fail(e_, #call, __FILE__, __LINE__); } } while (0)
    TRY(cudaMallocAsync(&d_eig, pitch * H * frames, st));
    TRY(cudaMallocAsync(&d_max, sizeof(unsigned) * frames, st));
    TRY(cudaMallocAsync(&d_cnt, sizeof(int) * frames, st));
    TRY(cudaMallocAsync(&d_cand, sizeof(CandKey) * (size_t)cap * frames, st));
    TRY(cudaMemsetAsync(d_max, 0, sizeof(unsigned) * frames, st));
    b200cvMat eig = {d_eig, pitch, W, H, B200CV_MAKETYPE(B200CV_32F, 1), frames, pitch * H};
    rc = corner_response(src, &eig, block_size, gradient_size, k, B200CV_BORDER_REFLECT_101, use_harris ? 0 : 1, stream);
    if (rc) { cleanup(); return rc; }
    Img e = make_img(&eig);
    frame_max_kernel<<<dim3(std::min((unsigned)H, (unsigned)num_sms() * 8u), frames), 256, 0, st>>>(e, d_max);
    count_launch();
    // top-K preselection (all frames, before the one synchronisation that brings the counts back)
    unsigned* d_hist = nullptr; int* d_thr = nullptr; int* d_topcnt = nullptr; CandKey* d_top = nullptr;
    auto cleanup2 = [&]() { cudaFreeAsync(d_hist, st); cudaFreeAsync(d_thr, st); cudaFreeAsync(d_topcnt, st); cudaFreeAsync(d_top, st); cleanup(); };
#undef TRY
#define TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { cleanup2(); return cuda_fail(e_, #call, __FILE__, __LINE__); } } while (0)
    const char* ps_env = getenv("B200CV_GFTT_PRESELECT");                        // "0": always sort every candidate (A/B and the parity test)
    const bool preselect = max_corners > 0 && !(ps_env && ps_env[0] == '0');
    if (preselect) {
        TRY(cudaMallocAsync(&d_hist, sizeof(unsigned) * GF_BINS * frames, st));
        TRY(cudaMallocAsync(&d_thr, sizeof(int) * frames, st));
        TRY(cudaMallocAsync(&d_topcnt, sizeof(int) * frames, st));
        TRY(cudaMallocAsync(&d_top, sizeof(CandKey) * (size_t)GF_TOP_CAP * frames, st));
    }
    std::vector<int> hcnt(frames), hsel(frames, 0);
    // candidates (and the preselection) of every frame, then one synchronisation that brings the counts back.  The kernel counts every
    // candidate but stores only the first `cap` of a frame
    auto find_candidates = [&]() -> cudaError_t {
        cudaError_t ce = cudaMemsetAsync(d_cnt, 0, sizeof(int) * frames, st);
        if (ce == cudaSuccess && preselect) ce = cudaMemsetAsync(d_hist, 0, sizeof(unsigned) * GF_BINS * frames, st);
        if (ce == cudaSuccess && preselect) ce = cudaMemsetAsync(d_topcnt, 0, sizeof(int) * frames, st);
        if (ce != cudaSuccess) return ce;
        const unsigned tiles = div_up(W, 1024) * div_up(H, GC_R);
        gftt_candidates_kernel<<<dim3(std::min(tiles, (unsigned)num_sms() * 8u), frames), 256, 0, st>>>(e, d_max, quality_level, d_cand, cap, d_cnt, d_hist);
        count_launch();
        if ((ce = cudaGetLastError()) != cudaSuccess) return ce;
        if (preselect) {
            gftt_select_kernel<<<frames, 128, 0, st>>>(d_hist, d_thr);
            gftt_filter_kernel<<<dim3(128, frames), 256, 0, st>>>(d_cand, d_cnt, cap, d_thr, d_top, d_topcnt);
            count_launch(2);
            if ((ce = cudaGetLastError()) != cudaSuccess) return ce;
        }
        if ((ce = cudaMemcpyAsync(hcnt.data(), d_cnt, sizeof(int) * frames, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return ce;
        if (preselect && (ce = cudaMemcpyAsync(hsel.data(), d_topcnt, sizeof(int) * frames, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return ce;
        return cudaStreamSynchronize(st);
    };
    TRY(find_candidates());
    // a frame with more candidates than the list holds (noise or plateaus at 8K: up to (W - 2)(H - 2)): every candidate is kept -- the
    // list grows to the largest count and the candidates are found again (the common case keeps one pass and the 2^20-entry list)
    const int most = *std::max_element(hcnt.begin(), hcnt.end());
    if (most > cap) {
        TRY(cudaFreeAsync(d_cand, st));
        d_cand = nullptr;
        cap = most;
        TRY(cudaMallocAsync(&d_cand, sizeof(CandKey) * (size_t)cap * frames, st));
        TRY(find_candidates());
    }
    // order the candidates on the device (library radix sort: not per-pixel work), then walk them on the host in chunks --
    // the greedy minimum-distance selection is sequential and normally stops after a short prefix
    int nmax = 0;
    std::vector<int> nwalk(frames);
    std::vector<char> partial(frames, 0);
    for (int f = 0; f < frames; f++) {
        hcnt[f] = std::min(hcnt[f], cap);
        nwalk[f] = hcnt[f];
        if (preselect && hsel[f] < hcnt[f] && hsel[f] <= GF_TOP_CAP && hsel[f] > 0) { partial[f] = 1; nwalk[f] = hsel[f]; }
        nmax = std::max(nmax, hcnt[f]);
    }
    // the strongest CHUNK candidates of EVERY frame come back with one synchronisation (page-locked staging); the walk fetches further chunks
    // only if it gets that far (it normally stops after a short prefix)
    const int CHUNK = 1 << 14;
    static thread_local CandKey* h_stage = nullptr;
    static thread_local size_t h_stage_cap = 0;
    const size_t need = (size_t)CHUNK * frames;
    if (h_stage_cap < need) {
        if (h_stage) cudaFreeHost(h_stage);
        h_stage = nullptr; h_stage_cap = 0;
        TRY(cudaHostAlloc((void**)&h_stage, need * sizeof(CandKey), cudaHostAllocDefault));
        h_stage_cap = need;
    }
    // a radix sort of 10^4..10^5 keys is ten launches of a few microseconds each: the frames' sorts (and the copies of their heads) run on
    // side streams next to each other, forked from / joined to the caller's stream with events
    constexpr int NSIDE = 4;
    struct Side { int dev = -1; cudaStream_t s[NSIDE]; cudaEvent_t fork, join[NSIDE]; };
    static thread_local Side side;
    int cur_dev = 0;
    TRY(cudaGetDevice(&cur_dev));
    const int ns = std::min(frames, NSIDE);
    if (ns > 1 && side.dev != cur_dev) {
        if (side.dev >= 0) { for (int i = 0; i < NSIDE; i++) { cudaStreamDestroy(side.s[i]); cudaEventDestroy(side.join[i]); } cudaEventDestroy(side.fork); side.dev = -1; }
        for (int i = 0; i < NSIDE; i++) { TRY(cudaStreamCreateWithFlags(&side.s[i], cudaStreamNonBlocking)); TRY(cudaEventCreateWithFlags(&side.join[i], cudaEventDisableTiming)); }
        TRY(cudaEventCreateWithFlags(&side.fork, cudaEventDisableTiming));
        side.dev = cur_dev;
    }
    size_t tmp_bytes = 0;
    if (nmax) {
        TRY(cub::DeviceRadixSort::SortKeysDescending(nullptr, tmp_bytes, d_cand, d_sorted, nmax, 0, 64, st));
        tmp_bytes = (tmp_bytes + 255) & ~(size_t)255;
        TRY(cudaMallocAsync(&d_tmp, tmp_bytes * ns, st));
        TRY(cudaMallocAsync(&d_sorted, sizeof(CandKey) * (size_t)cap * frames, st));
        if (ns > 1) {
            TRY(cudaEventRecord(side.fork, st));
            for (int i = 0; i < ns; i++) TRY(cudaStreamWaitEvent(side.s[i], side.fork, 0));
        }
        for (int f = 0; f < frames; f++)
            if (nwalk[f]) {
                cudaStream_t sf = ns > 1 ? side.s[f % ns] : st;
                const CandKey* in = partial[f] ? d_top + (size_t)f * GF_TOP_CAP : d_cand + (size_t)f * cap;
                TRY(cub::DeviceRadixSort::SortKeysDescending((char*)d_tmp + tmp_bytes * (f % ns), tmp_bytes, in, d_sorted + (size_t)f * cap, nwalk[f], 0, 64, sf));
                count_launch();
                TRY(cudaMemcpyAsync(h_stage + (size_t)f * CHUNK, d_sorted + (size_t)f * cap, sizeof(CandKey) * std::min(CHUNK, nwalk[f]), cudaMemcpyDeviceToHost, sf));
            }
        if (ns > 1)
            for (int i = 0; i < ns; i++) { TRY(cudaEventRecord(side.join[i], side.s[i])); TRY(cudaStreamWaitEvent(st, side.join[i], 0)); }
    }
    TRY(cudaStreamSynchronize(st));
    std::vector<CandKey> chunk;
    std::vector<int> head, nxt;                  // accepted corners per grid cell: singly linked lists in flat arrays
    std::vector<float> ax, ay;
    for (int f = 0; f < frames; f++) {
      for (int attempt = 0; attempt < 2; attempt++) {
        const int n = nwalk[f];
        int fetched = std::min(CHUNK, n), base = 0;                  // candidates [base, fetched) are in `cur`
        const CandKey* cur = h_stage + (size_t)f * CHUNK;
        // the i-th strongest candidate; fetches another chunk when the walk gets there
        auto fetch = [&](int i) -> cudaError_t {
            if (i < fetched) return cudaSuccess;
            const int m = std::min(CHUNK, n - fetched);
            chunk.resize(m);
            cudaError_t ce = cudaMemcpyAsync(chunk.data(), d_sorted + (size_t)f * cap + fetched, sizeof(CandKey) * m, cudaMemcpyDeviceToHost, st);
            if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
            base = fetched; fetched += m; cur = chunk.data();
            return ce;
        };
        float* outp = corners + (size_t)f * max_out * 2;
        float* outq = quality ? quality + (size_t)f * max_out : nullptr;
        int accepted = 0;
        auto emit = [&](int x, int y, float v) {
            if (accepted < max_out) { outp[2 * accepted] = (float)x; outp[2 * accepted + 1] = (float)y; if (outq) outq[accepted] = v; }
            accepted++;
        };
        if (min_distance >= 1) {
            const int cell = (int)lrint(min_distance);
            const int gw = (W + cell - 1) / cell, gh = (H + cell - 1) / cell;
            head.assign((size_t)gw * gh, -1);
            nxt.clear(); ax.clear(); ay.clear();
            const double md2 = min_distance * min_distance;
            for (int i = 0; i < n; i++) {
                TRY(fetch(i));
                const CandKey key = cur[i - base];
                const int pos = (int)(unsigned)key;
                int y = pos / W, x = pos - y * W;
                int cx = x / cell, cy = y / cell;
                bool keep = true;
                for (int yy = std::max(0, cy - 1); keep && yy <= std::min(gh - 1, cy + 1); yy++)
                    for (int xx = std::max(0, cx - 1); keep && xx <= std::min(gw - 1, cx + 1); xx++)
                        for (int q = head[(size_t)yy * gw + xx]; q >= 0; q = nxt[q]) {
                            float ddx = x - ax[q], ddy = y - ay[q];
                            if (ddx * ddx + ddy * ddy < md2) { keep = false; break; }
                        }
                if (!keep) continue;
                nxt.push_back(head[(size_t)cy * gw + cx]);
                head[(size_t)cy * gw + cx] = (int)ax.size();
                ax.push_back((float)x); ay.push_back((float)y);
                emit(x, y, ord2f((unsigned)(key >> 32)));
                if (max_corners > 0 && accepted == max_corners) break;
            }
        } else {
            for (int i = 0; i < n; i++) {
                TRY(fetch(i));
                const CandKey key = cur[i - base];
                const int pos = (int)(unsigned)key;
                int y = pos / W, x = pos - y * W;
                emit(x, y, ord2f((unsigned)(key >> 32)));
                if (max_corners > 0 && accepted == max_corners) break;
            }
        }
        counts[f] = accepted;
        if (!partial[f] || accepted >= max_corners) break;
        // the preselected prefix ran out before max_corners corners were accepted: this frame again, with every candidate in order
        partial[f] = 0; nwalk[f] = hcnt[f];
        TRY(cub::DeviceRadixSort::SortKeysDescending(d_tmp, tmp_bytes, d_cand + (size_t)f * cap, d_sorted + (size_t)f * cap, hcnt[f], 0, 64, st));
        count_launch();
        TRY(cudaMemcpyAsync(h_stage + (size_t)f * CHUNK, d_sorted + (size_t)f * cap, sizeof(CandKey) * std::min(CHUNK, hcnt[f]), cudaMemcpyDeviceToHost, st));
        TRY(cudaStreamSynchronize(st));
      }
    }
#undef TRY
    cleanup2();
    return B200CV_OK;
}
