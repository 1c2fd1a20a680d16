// matchtemplate.cu -- cv::matchTemplate (1-channel CV_8U / CV_32F images, all six methods, no mask).
//
// Reference (modules/imgproc/src/templmatch.cpp): crossCorr (:566-760) computes the raw correlation with a block DFT
// in float (u8) or double (f32) on ONE thread; common_matchTemplate (:906-1029) then normalises it from f64 integral
// images.  Here:
//   * numerator  R(x,y) = sum_{u,v} T(u,v) * I(x+u, y+v)   -- direct dense contraction.
//       u8 : exact integers, 4 MACs per IDP4A (dp4a) with 4x4 register blocking per thread: a CTA stages a
//            (64+w-1) x (64+h-1) byte tile in shared memory and produces 64 x 64 outputs; every staged image word is
//            reused for 4 template rows and every template word for 4 outputs.  (The reference's result is the exact
//            value +- DFT round-off ~1e-7 relative; its own test tolerance is 1e-3, test_templmatch.cpp:333.)
//       f32: same blocking with FFMA.
//   * window sums  sum I, sum I^2 over each w x h window in f64 (exact for u8): separable sliding sums.
//   * normalisation: the formulas and clamps of common_matchTemplate :975-1026, in f64, per output.
#include <cstdlib>
#include <cstring>
#include <vector>
#include "common.cuh"

namespace b200cv {

int ccorr_u8_tensor(const Img& im, const Img& tp, const Img& rs, int w, int h, cudaStream_t st);

constexpr int MT_T = 64;     // outputs per CTA side
constexpr int MT_R = 4;      // outputs per thread side

struct TemplStats {          // produced on the device, consumed by the normalisation kernel
    double mean, norm, sum2, inv_area;
    int flat;                // CCOEFF_NORMED on a constant template: result = 1 everywhere
};

// ---- template statistics (meanStdDev semantics, modules/core/src/mean.dispatch.cpp) --------------------------------------
template <typename T>
__global__ void templ_stats_kernel(Img templ, int method, TemplStats* out)
{
    __shared__ double s_sum[256], s_sq[256];
    double s = 0, q = 0;
    const int n = templ.cols * templ.rows;
    for (int i = threadIdx.x; i < n; i += 256) {
        int y = i / templ.cols, x = i - y * templ.cols;
        double v = (double)templ.row<T>(0, y)[x];
        s += v; q += v * v;
    }
    s_sum[threadIdx.x] = s; s_sq[threadIdx.x] = q;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (threadIdx.x < o) { s_sum[threadIdx.x] += s_sum[threadIdx.x + o]; s_sq[threadIdx.x] += s_sq[threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double scale = 1. / n;
        double mean = s_sum[0] * scale;
        double var = fmax(s_sq[0] * scale - mean * mean, 0.);
        double sdv = sqrt(var);
        double templNorm = sdv * sdv;
        TemplStats r;
        r.inv_area = 1. / ((double)templ.rows * templ.cols);
        r.flat = (templNorm < 2.220446049250313e-16 && method == B200CV_TM_CCOEFF_NORMED);
        double templSum2 = templNorm + mean * mean;
        const int numType = (method == B200CV_TM_CCORR || method == B200CV_TM_CCORR_NORMED) ? 0 : (method == B200CV_TM_CCOEFF || method == B200CV_TM_CCOEFF_NORMED) ? 1 : 2;
        if (numType != 1) { mean = 0; templNorm = templSum2; }
        templSum2 /= r.inv_area;
        templNorm = sqrt(templNorm);
        templNorm /= sqrt(r.inv_area);
        r.mean = mean; r.norm = templNorm; r.sum2 = templSum2;
        *out = r;
    }
}

// ---- window sums -------------------------------------------------------------------------------------------------------
// pass 1: rs[y][x] = sum_{i<w} I[y][x+i] (and squares), x in [0, W-w]; one thread walks 32 consecutive outputs
template <typename T>
__global__ void __launch_bounds__(256) wnd_rows_kernel(Img img, int w, int ow, double* rs, double* rq, size_t pitch_d)
{
    const int f = blockIdx.z;
    const int y = blockIdx.y;
    const int x0 = (blockIdx.x * 256 + threadIdx.x) * 32;
    if (x0 >= ow) return;
    const T* row = img.row<T>(f, y);
    double s = 0, q = 0;
    for (int i = 0; i < w; i++) { double v = (double)row[x0 + i]; s += v; q += v * v; }
    double* ps = rs + ((size_t)f * img.rows + y) * pitch_d;
    double* pq = rq + ((size_t)f * img.rows + y) * pitch_d;
    const int n = min(32, ow - x0);
    for (int k = 0; k < n; k++) {
        ps[x0 + k] = s; pq[x0 + k] = q;
        if (k + 1 < n) {
            double a = (double)row[x0 + k + w], b = (double)row[x0 + k];
            s += a - b; q += a * a - b * b;
        }
    }
}

// pass 2: ws[y][x] = sum_{j<h} rs[y+j][x]; one thread walks 32 consecutive output rows of one column
__global__ void __launch_bounds__(256) wnd_cols_kernel(const double* rs, const double* rq, double* ws, double* wq, size_t pitch_d,
                                                        int rows, int h, int ow, int oh)
{
    const int f = blockIdx.z;
    const int x = blockIdx.x * 256 + threadIdx.x;
    const int y0 = blockIdx.y * 32;
    if (x >= ow || y0 >= oh) return;
    const double* ps = rs + (size_t)f * rows * pitch_d + x;
    const double* pq = rq + (size_t)f * rows * pitch_d + x;
    double s = 0, q = 0;
    for (int j = 0; j < h; j++) { s += ps[(size_t)(y0 + j) * pitch_d]; q += pq[(size_t)(y0 + j) * pitch_d]; }
    const int n = min(32, oh - y0);
    for (int k = 0; k < n; k++) {
        ws[((size_t)f * oh + y0 + k) * pitch_d + x] = s;
        wq[((size_t)f * oh + y0 + k) * pitch_d + x] = q;
        if (k + 1 < n) {
            s += ps[(size_t)(y0 + k + h) * pitch_d] - ps[(size_t)(y0 + k) * pitch_d];
            q += pq[(size_t)(y0 + k + h) * pitch_d] - pq[(size_t)(y0 + k) * pitch_d];
        }
    }
}

// ---- numerator: u8, dp4a ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ccorr_u8_kernel(Img img, Img templ, Img res, int w, int h, int wpad)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tstride = wpad;                               // template row stride (bytes, multiple of 4)
    const int istride = MT_T + wpad + 4;                    // image tile row stride (bytes, multiple of 4)
    const int irows = MT_T + h - 1;
    unsigned char* s_t = smem_raw;                          // h x tstride
    unsigned char* s_i = smem_raw + (((size_t)h * tstride + 15) & ~(size_t)15);
    const int f = blockIdx.z, x0 = blockIdx.x * MT_T, y0 = blockIdx.y * MT_T;
    for (int idx = threadIdx.x; idx < h * tstride; idx += 256) {
        int r = idx / tstride, c = idx - r * tstride;
        s_t[idx] = c < w ? templ.row<uchar>(0, r)[c] : (uchar)0;
    }
    for (int idx = threadIdx.x; idx < irows * istride; idx += 256) {
        int r = idx / istride, c = idx - r * istride;
        int gy = y0 + r, gx = x0 + c;
        s_i[idx] = (gy < img.rows && gx < img.cols) ? img.row<uchar>(f, gy)[gx] : (uchar)0;
    }
    __syncthreads();
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;     // 16 x 16 threads, 4 x 4 outputs each
    unsigned acc[MT_R][MT_R];
#pragma unroll
    for (int a = 0; a < MT_R; a++)
#pragma unroll
        for (int b = 0; b < MT_R; b++) acc[a][b] = 0;
    const int nwords = wpad / 4;
    // image rows r = ty*4 .. ty*4 + 3 + h - 1 feed output rows o (0..3) with template row r - ty*4 - o
    for (int rr = 0; rr < h + MT_R - 1; rr++) {
        const unsigned* irow = (const unsigned*)(s_i + (ty * MT_R + rr) * istride + tx * MT_R);
        for (int g = 0; g < nwords; g++) {
            unsigned w0 = irow[g], w1 = irow[g + 1];
            unsigned win[MT_R];
            win[0] = w0;
            win[1] = __byte_perm(w0, w1, 0x4321);
            win[2] = __byte_perm(w0, w1, 0x5432);
            win[3] = __byte_perm(w0, w1, 0x6543);
#pragma unroll
            for (int o = 0; o < MT_R; o++) {
                int tr = rr - o;
                if (tr >= 0 && tr < h) {
                    unsigned tw = *(const unsigned*)(s_t + tr * tstride + g * 4);
#pragma unroll
                    for (int b = 0; b < MT_R; b++) acc[o][b] = __dp4a(win[b], tw, acc[o][b]);
                }
            }
        }
    }
#pragma unroll
    for (int o = 0; o < MT_R; o++) {
        int gy = y0 + ty * MT_R + o;
        if (gy >= res.rows) break;
        float* rp = res.row<float>(f, gy);
#pragma unroll
        for (int b = 0; b < MT_R; b++) {
            int gx = x0 + tx * MT_R + b;
            if (gx < res.cols) rp[gx] = (float)acc[o][b];
        }
    }
}

// ---- numerator: f32 ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ccorr_f32_kernel(Img img, Img templ, Img res, int w, int h)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int istride = MT_T + w + 3;
    const int irows = MT_T + h - 1;
    float* s_t = (float*)smem_raw;                          // h x w
    float* s_i = s_t + (size_t)h * w;
    const int f = blockIdx.z, x0 = blockIdx.x * MT_T, y0 = blockIdx.y * MT_T;
    for (int idx = threadIdx.x; idx < h * w; idx += 256) s_t[idx] = templ.row<float>(0, idx / w)[idx % w];
    for (int idx = threadIdx.x; idx < irows * istride; idx += 256) {
        int r = idx / istride, c = idx - r * istride;
        int gy = y0 + r, gx = x0 + c;
        s_i[idx] = (gy < img.rows && gx < img.cols) ? img.row<float>(f, gy)[gx] : 0.f;
    }
    __syncthreads();
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[MT_R][MT_R];
#pragma unroll
    for (int a = 0; a < MT_R; a++)
#pragma unroll
        for (int b = 0; b < MT_R; b++) acc[a][b] = 0.f;
    for (int rr = 0; rr < h + MT_R - 1; rr++) {
        const float* irow = s_i + (ty * MT_R + rr) * istride + tx * MT_R;
        for (int u = 0; u < w; u++) {
            float v[MT_R];
#pragma unroll
            for (int b = 0; b < MT_R; b++) v[b] = irow[u + b];
#pragma unroll
            for (int o = 0; o < MT_R; o++) {
                int tr = rr - o;
                if (tr >= 0 && tr < h) {
                    float t = s_t[tr * w + u];
#pragma unroll
                    for (int b = 0; b < MT_R; b++) acc[o][b] = fmaf(v[b], t, acc[o][b]);
                }
            }
        }
    }
#pragma unroll
    for (int o = 0; o < MT_R; o++) {
        int gy = y0 + ty * MT_R + o;
        if (gy >= res.rows) break;
        float* rp = res.row<float>(f, gy);
#pragma unroll
        for (int b = 0; b < MT_R; b++) {
            int gx = x0 + tx * MT_R + b;
            if (gx < res.cols) rp[gx] = acc[o][b];
        }
    }
}

// ---- normalisation (common_matchTemplate :975-1026) ------------------------------------------------------------------
__global__ void __launch_bounds__(256) mt_normalize_kernel(Img res, const double* ws, const double* wq, size_t pitch_d, int method,
                                                            const TemplStats* stats)
{
    const int f = blockIdx.z;
    const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
    if (x >= res.cols) return;
    const TemplStats st = *stats;
    float* rp = res.row<float>(f, y) + x;
    if (st.flat) { *rp = 1.f; return; }
    const int numType = (method == B200CV_TM_CCORR || method == B200CV_TM_CCORR_NORMED) ? 0 : (method == B200CV_TM_CCOEFF || method == B200CV_TM_CCOEFF_NORMED) ? 1 : 2;
    const bool isNormed = method == B200CV_TM_CCORR_NORMED || method == B200CV_TM_SQDIFF_NORMED || method == B200CV_TM_CCOEFF_NORMED;
    double num = (double)*rp, t;
    double wndMean2 = 0, wndSum2 = 0;
    const size_t o = ((size_t)f * res.rows + y) * pitch_d + x;
    if (numType == 1) {
        t = ws[o];
        wndMean2 += t * t;
        num -= t * st.mean;
        wndMean2 *= st.inv_area;
    }
    if (isNormed || numType == 2) {
        wndSum2 += wq[o];
        if (numType == 2) { num = wndSum2 - 2 * num + st.sum2; num = fmax(num, 0.); }
    }
    if (isNormed) {
        double diff2 = fmax(wndSum2 - wndMean2, 0.);
        if (diff2 <= fmin(0.5, 10 * 1.1920928955078125e-07 * wndSum2)) t = 0;
        else t = sqrt(diff2) * st.norm;
        if (fabs(num) < t) num /= t;
        else if (fabs(num) < t * 1.125) num = num > 0 ? 1 : -1;
        else num = method != B200CV_TM_SQDIFF_NORMED ? 0 : 1;
    }
    *rp = (float)num;
}


// ---- 8-bit images: window sums + normalisation in ONE kernel, no intermediate planes ----------------------------------------------------
// The window sums of an 8-bit image are exact integers (sum <= 255 w h, sum of squares <= 65025 w h < 2^32 for every template the numerator
// kernels accept): the reference's f64 integral-image differences (templmatch.cpp:930-1004) have exactly these values.  One thread owns 4
// adjacent result columns and walks down a segment of rows keeping the 4 window sums and sums of squares in u32 registers: a row enters
// (and, h rows later, leaves) as 4 horizontal sums over w bytes, computed from the aligned words of the image row -- the words all 4 windows
// share once (IDP4A against 1s for the sum, against the word itself for the squares), the one or two words at either end per window through
// byte masks.  Every image row is read twice, the numerator once; nothing else touches HBM (the first version wrote and re-read four f64
// planes).
__device__ __forceinline__ unsigned mt_mask_ge(int k) { return k >= 4 ? 0u : (k <= 0 ? 0xFFFFFFFFu : 0xFFFFFFFFu << (8 * k)); }
__device__ __forceinline__ unsigned mt_mask_lt(int n) { return n <= 0 ? 0u : (n >= 4 ? 0xFFFFFFFFu : (1u << (8 * n)) - 1u); }

// sums over bytes [k, k + w) of the row for k = 0..3, relative to the aligned word pointer wp; words with index > jmax lie outside the row
__device__ __forceinline__ void mt_row4(const unsigned* __restrict__ wp, int w, int jmax, unsigned s[4], unsigned q[4])
{
    const int nw = min((w + 2) / 4, jmax);            // last word index any of the 4 windows touches
    const int jfull = min((w - 4) >> 2, jmax);        // words 1..jfull lie inside all 4 windows
    unsigned ms = 0, mq = 0;
#pragma unroll 4
    for (int j = 1; j <= jfull; j++) {
        const unsigned v = __ldg(wp + j);
        ms = __dp4a(v, 0x01010101u, ms);
        mq = __dp4a(v, v, mq);
    }
    const unsigned v0 = jmax >= 0 ? __ldg(wp) : 0u;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const unsigned vm = v0 & mt_mask_ge(k) & mt_mask_lt(k + w);
        s[k] = __dp4a(vm, 0x01010101u, ms);
        q[k] = __dp4a(vm, v0, mq);
    }
    for (int j = max(jfull + 1, 1); j <= nw; j++) {
        const unsigned v = __ldg(wp + j);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const unsigned vm = v & mt_mask_lt(k + w - 4 * j);
            s[k] = __dp4a(vm, 0x01010101u, s[k]);
            q[k] = __dp4a(vm, v, q[k]);
        }
    }
}

// the same for a template width of 4 * WW bytes, everything at compile time: words 1 .. WW-1 lie inside all four windows, word 0 loses its
// first k bytes and word WW contributes its first k bytes (no loop, no run-time masks; the caller guarantees that word WW is inside the row)
template <int WW>
__device__ __forceinline__ void mt_row4_fixed(const unsigned* __restrict__ wp, unsigned s[4], unsigned q[4])
{
    unsigned v[WW + 1];
#pragma unroll
    for (int j = 0; j <= WW; j++) v[j] = __ldg(wp + j);
    unsigned ms = 0, mq = 0;
#pragma unroll
    for (int j = 1; j < WW; j++) { ms = __dp4a(v[j], 0x01010101u, ms); mq = __dp4a(v[j], v[j], mq); }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const unsigned m0 = k == 0 ? 0xFFFFFFFFu : 0xFFFFFFFFu << (8 * k), m1 = ~m0;
        const unsigned a = v[0] & m0, b = v[WW] & m1;
        s[k] = __dp4a(b, 0x01010101u, __dp4a(a, 0x01010101u, ms));
        q[k] = __dp4a(b, v[WW], __dp4a(a, v[0], mq));
    }
}

__device__ __forceinline__ float mt_normalize_one(double num, double ws, double wq, int numType, bool isNormed, int method, const TemplStats& st)
{
    double t, wndMean2 = 0, wndSum2 = 0;
    if (numType == 1) {
        t = ws;
        wndMean2 += t * t;
        num -= t * st.mean;
        wndMean2 *= st.inv_area;
    }
    if (isNormed || numType == 2) {
        wndSum2 += wq;
        if (numType == 2) { num = wndSum2 - 2 * num + st.sum2; num = fmax(num, 0.); }
    }
    if (isNormed) {
        double diff2 = fmax(wndSum2 - wndMean2, 0.);
        if (diff2 <= fmin(0.5, 10 * 1.1920928955078125e-07 * wndSum2)) t = 0;
        else t = sqrt(diff2) * st.norm;
        if (fabs(num) < t) num /= t;
        else if (fabs(num) < t * 1.125) num = num > 0 ? 1 : -1;
        else num = method != B200CV_TM_SQDIFF_NORMED ? 0 : 1;
    }
    return (float)num;
}

constexpr int MTF_SEG = 128;     // result rows per thread

template <int WW>      // template width / 4 when it is a multiple of 4 in {16, 32, 64, 128} bytes, 0 = any width
__global__ void __launch_bounds__(128) mt_fused_u8_kernel(Img img, Img res, int w, int h, int method, const TemplStats* __restrict__ stats)
{
    const int f = blockIdx.z;
    const int x0 = (blockIdx.x * 128 + threadIdx.x) * 4;
    const int ys = blockIdx.y * MTF_SEG, ye = min(ys + MTF_SEG, res.rows);
    if (x0 >= res.cols) return;
    const TemplStats st = *stats;
    const int numType = (method == B200CV_TM_CCORR || method == B200CV_TM_CCORR_NORMED) ? 0 : (method == B200CV_TM_CCOEFF || method == B200CV_TM_CCOEFF_NORMED) ? 1 : 2;
    const bool isNormed = method == B200CV_TM_CCORR_NORMED || method == B200CV_TM_SQDIFF_NORMED || method == B200CV_TM_CCOEFF_NORMED;
    const int jmax = (img.cols - x0 + 3) / 4 - 1;                    // last word of the row that still holds image bytes
    const int n = min(4, res.cols - x0);
    const bool fixed = WW > 0 && jmax >= WW;                          // all WW + 1 words inside the row: the compile-time variant
    auto row4 = [&](int y, unsigned* s, unsigned* q) {
        const unsigned* wp = (const unsigned*)(img.row<uchar>(f, y) + x0);
        if constexpr (WW > 0) { if (fixed) { mt_row4_fixed<WW>(wp, s, q); return; } }
        mt_row4(wp, w, jmax, s, q);
    };
    unsigned ws[4] = {0, 0, 0, 0}, wq[4] = {0, 0, 0, 0};
    for (int j = 0; j < h; j++) {
        unsigned s[4], q[4];
        row4(ys + j, s, q);
#pragma unroll
        for (int k = 0; k < 4; k++) { ws[k] += s[k]; wq[k] += q[k]; }
    }
    for (int y = ys; y < ye; y++) {
        float* rp = res.row<float>(f, y) + x0;
        const bool vec = n == 4 && (((uintptr_t)rp) & 15) == 0;
        float num[4];
        if (vec) { const float4 t = *(const float4*)rp; num[0] = t.x; num[1] = t.y; num[2] = t.z; num[3] = t.w; }
        else for (int k = 0; k < n; k++) num[k] = rp[k];
        float out[4];
        if (st.flat) { out[0] = out[1] = out[2] = out[3] = 1.f; }
        else {
#pragma unroll
            for (int k = 0; k < 4; k++) out[k] = k < n ? mt_normalize_one((double)num[k], (double)ws[k], (double)wq[k], numType, isNormed, method, st) : 0.f;
        }
        if (vec) *(float4*)rp = make_float4(out[0], out[1], out[2], out[3]);
        else for (int k = 0; k < n; k++) rp[k] = out[k];
        if (y + 1 < ye) {
            unsigned s[4], q[4], s2[4], q2[4];
            row4(y + h, s, q);
            row4(y, s2, q2);
#pragma unroll
            for (int k = 0; k < 4; k++) { ws[k] += s[k] - s2[k]; wq[k] += q[k] - q2[k]; }
        }
    }
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_match_template(const b200cvMat* image, const b200cvMat* templ, const b200cvMat* result, int method, void* stream)
{
    int rc;
    if ((rc = check_mat(image, "image")) || (rc = check_mat(templ, "templ")) || (rc = check_mat(result, "result"))) return rc;
    B200_REQUIRE(method >= 0 && method <= 5, "bad method");
    B200_REQUIRE(image->type == templ->type, "image/template type mismatch");
    if (image->type != B200CV_MAKETYPE(B200CV_8U, 1) && image->type != B200CV_MAKETYPE(B200CV_32F, 1)) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(result->type == B200CV_MAKETYPE(B200CV_32F, 1), "result must be CV_32FC1");
    const int W = image->cols, H = image->rows, w = templ->cols, h = templ->rows;
    if (w > W || h > H) return B200CV_NOT_IMPLEMENTED;      // the reference swaps roles; not on the device path
    const int ow = W - w + 1, oh = H - h + 1;
    B200_REQUIRE(result->cols == ow && result->rows == oh, "result must be (W-w+1) x (H-h+1)");
    Img im = make_img(image), tp = make_img(templ), rs = make_img(result);
    B200_REQUIRE(im.frames == rs.frames, "image/result batch mismatch");
    const bool u8 = B200CV_DEPTH(image->type) == B200CV_8U;
    cudaStream_t st = as_stream(stream);
    const int frames = im.frames;
    dim3 grid(div_up((unsigned)ow, MT_T), div_up((unsigned)oh, MT_T), (unsigned)frames);

    bool done = false;
    if (u8 && (long long)w * h <= 33025) {      // tensor-core path (matchtemplate_tc.cu): s32 accumulators stay exact (65025*w*h < 2^31)
        const char* force = getenv("B200CV_MATCHTEMPLATE_PATH");
        if (!(force && !strcmp(force, "dp4a"))) {
            rc = ccorr_u8_tensor(im, tp, rs, w, h, st);
            if (rc == B200CV_OK) done = true;
            else if (rc != B200CV_NOT_IMPLEMENTED) return rc;
        }
    }
    if (done) {
    } else if (u8) {
        if ((long long)w * h > 66051) return B200CV_NOT_IMPLEMENTED;   // u32 accumulators stay exact
        int wpad = (w + 3) & ~3;
        size_t smem = (((size_t)h * wpad + 15) & ~(size_t)15) + (size_t)(MT_T + h - 1) * (MT_T + wpad + 4) + 16;
        if (smem > 200 * 1024) return B200CV_NOT_IMPLEMENTED;
        static PerDeviceFlag a_pd; bool& a = a_pd.cur();
        if (!a) { B200_CUDA(cudaFuncSetAttribute(ccorr_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); a = true; }
        ccorr_u8_kernel<<<grid, 256, smem, st>>>(im, tp, rs, w, h, wpad);
    } else {
        size_t smem = ((size_t)h * w + (size_t)(MT_T + h - 1) * (MT_T + w + 3)) * sizeof(float);
        if (smem > 200 * 1024) return B200CV_NOT_IMPLEMENTED;
        static PerDeviceFlag a_pd; bool& a = a_pd.cur();
        if (!a) { B200_CUDA(cudaFuncSetAttribute(ccorr_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); a = true; }
        ccorr_f32_kernel<<<grid, 256, smem, st>>>(im, tp, rs, w, h);
    }
    if (!done) B200_LAUNCH_CHECK();
    if (method == B200CV_TM_CCORR) return B200CV_OK;

    const char* norm_env = getenv("B200CV_MATCHTEMPLATE_NORM");        // test hook: "planes" = the first version (f64 window-sum planes)
    if (u8 && (((uintptr_t)im.data | im.step | im.fstep) & 3) == 0 && !(norm_env && !strcmp(norm_env, "planes"))) {
        // 8-bit: exact u32 window sums and the normalisation fused into one pass (no intermediate planes)
        TemplStats* d_stats = nullptr;
        B200_CUDA(cudaMallocAsync(&d_stats, sizeof(TemplStats), st));
        templ_stats_kernel<uchar><<<1, 256, 0, st>>>(tp, method, d_stats);
        count_launch();
        const dim3 fg(div_up(div_up((unsigned)ow, 4), 128), div_up((unsigned)oh, MTF_SEG), frames);
        switch (w) {
        case 16: mt_fused_u8_kernel<4><<<fg, 128, 0, st>>>(im, rs, w, h, method, d_stats); break;
        case 32: mt_fused_u8_kernel<8><<<fg, 128, 0, st>>>(im, rs, w, h, method, d_stats); break;
        case 64: mt_fused_u8_kernel<16><<<fg, 128, 0, st>>>(im, rs, w, h, method, d_stats); break;
        case 128: mt_fused_u8_kernel<32><<<fg, 128, 0, st>>>(im, rs, w, h, method, d_stats); break;
        default: mt_fused_u8_kernel<0><<<fg, 128, 0, st>>>(im, rs, w, h, method, d_stats); break;
        }
        B200_LAUNCH_CHECK();
        B200_CUDA(cudaFreeAsync(d_stats, st));
        return B200CV_OK;
    }
    // workspace (stream-ordered): row sums, window sums, template statistics
    const size_t pitch_d = ((size_t)ow + 31) & ~(size_t)31;
    double *d_rs = nullptr, *d_rq = nullptr, *d_ws = nullptr, *d_wq = nullptr;
    TemplStats* d_stats = nullptr;
    size_t n_rows = (size_t)frames * H * pitch_d, n_wnd = (size_t)frames * oh * pitch_d;
    B200_CUDA(cudaMallocAsync(&d_rs, (2 * n_rows + 2 * n_wnd) * sizeof(double) + sizeof(TemplStats), st));
    d_rq = d_rs + n_rows; d_ws = d_rq + n_rows; d_wq = d_ws + n_wnd; d_stats = (TemplStats*)(d_wq + n_wnd);
    if (u8) {
        templ_stats_kernel<uchar><<<1, 256, 0, st>>>(tp, method, d_stats);
        wnd_rows_kernel<uchar><<<dim3(div_up(div_up((unsigned)ow, 32), 256), H, frames), 256, 0, st>>>(im, w, ow, d_rs, d_rq, pitch_d);
    } else {
        templ_stats_kernel<float><<<1, 256, 0, st>>>(tp, method, d_stats);
        wnd_rows_kernel<float><<<dim3(div_up(div_up((unsigned)ow, 32), 256), H, frames), 256, 0, st>>>(im, w, ow, d_rs, d_rq, pitch_d);
    }
    count_launch(2);
    wnd_cols_kernel<<<dim3(div_up((unsigned)ow, 256), div_up((unsigned)oh, 32), frames), 256, 0, st>>>(d_rs, d_rq, d_ws, d_wq, pitch_d, H, h, ow, oh);
    count_launch();
    mt_normalize_kernel<<<dim3(div_up((unsigned)ow, 256), oh, frames), 256, 0, st>>>(rs, d_ws, d_wq, pitch_d, method, d_stats);
    B200_LAUNCH_CHECK();
    B200_CUDA(cudaFreeAsync(d_rs, st));
    return B200CV_OK;
}
