/* oracle/port/port_laplacian.c -- cv::Laplacian restated in scalar C.  TEST INFRASTRUCTURE ONLY (see port_common.h).
 *   cv::Laplacian               modules/imgproc/src/deriv.cpp:787-876, getSobelKernels :96-160
 *   SymmRowSmallVec_32f         modules/imgproc/src/filter.simd.hpp:1746-1844, SymmRowSmallFilter :2450-2532
 *   SymmColumnVec_32f           modules/imgproc/src/filter.simd.hpp:1853-1949
 *   cvt_32f (convertTo)         modules/core/src/convert_scale.simd.hpp:91-121
 *
 * ksize 1 / 3: filter2D (port_filter2d) with the 3x3 kernel [0 1 0; 1 -4 1; 0 1 0] / [2 0 2; 0 -8 0; 2 0 2], each tap times (float)scale.
 * ksize 5..31: d2x = sepFilter(row kd, column ks), d2y = sepFilter(row ks, column kd) with kd, ks = getSobelKernels(2, 0, ksize), both
 *   into the working depth (16S for an 8-bit source at ksize 5, else 32F), through the port's separable core (port_filter.c); then
 *   d2x + d2y in that depth (saturating for 16S) and convertTo(ddepth, scale, delta):
 *     scale == 1 && delta == 0  saturate_cast (16S -> 16S and 32F -> 32F are copies)
 *     otherwise                 saturate_cast(fma((float)v, (float)scale, (float)delta)): cvt_32f's vector body is v_fma, and its scalar
 *                               tail, src*a + b, is contracted to the same FMA in the reference's AVX2 object
 *   A float source at ksize 5 is the one case the separable core does not restate: there both row kernels are 5-tap SymmRowSmall
 *   kernels, and the reference's Laplacian-specific order (lap5_f32 below) differs from the general one the core uses for every other
 *   caller.
 * Returns -1 for a ksize the reference refuses (even, < 1, > 31). */
#include "port_common.h"

int port_filter2d(const void* src, size_t sstep, void* dst, size_t dstep, int w, int h, int stype, int ddepth,
                  const float* k, int kw, int kh, int ax, int ay, double delta, int border);          /* port_filter.c */

static float mul_rn(float a, float b) { volatile float p = a * b; return p; }   /* a product rounded to float on its own */

/* getSobelKernels' taps: (1+z)^(n-d-1) (z-1)^d, rounded to float */
static void sobel_taps(int n, int d, float* out)
{
    long long p[32] = {1};
    int len = 1;
    for (int i = 0; i < n - d - 1; i++, len++) for (int j = len; j > 0; j--) p[j] += p[j - 1];
    for (int i = 0; i < d; i++, len++) { for (int j = len; j > 0; j--) p[j] = p[j - 1] - p[j]; p[0] = -p[0]; }
    for (int i = 0; i < len; i++) out[i] = (float)p[i];
}

/* One 5-tap row of a float source, output element e of a row of we elements, taps v[0..4] (v[2] the centre).
 *   kd = [1 0 -2 0 1]: SymmRowSmallVec_32f's special case fma(x0, -2, x-2 + x2), which never reads the zero taps (:1802-1815)
 *   ks = [1 4 6 4 1]:  the centre-out order fma(x-2 + x2, 1, fma(x0, 6, (x-1 + x1) * 4)) (:1816-1821)
 * The vector body covers the first we - we % 8 elements; SymmRowSmallFilter's scalar remainder (compiled with contraction) does the
 * rest: pairs of kd as fma(-2, x0, x-2) + x2 and of ks as the body, an odd last element of both as k0*x0; s = fma(k[j], x[j] + x[-j], s)
 * (:2508-2532). */
static float row5(const float* v, const float* k, int is_kd, int e, int we)
{
    const int tail = we - we % 8, last = tail + ((we - tail) & ~1);
    if (e >= last) {
        float s = mul_rn(k[2], v[2]);
        for (int j = 1; j <= 2; j++) s = fmaf(k[2 + j], v[2 + j] + v[2 - j], s);
        return s;
    }
    if (is_kd) return e >= tail ? fmaf(-2.f, v[2], v[0]) + v[4] : fmaf(v[2], -2.f, v[0] + v[4]);
    return fmaf(v[0] + v[4], k[4], fmaf(v[2], k[2], mul_rn(v[1] + v[3], k[3])));
}

/* d2x and d2y of a float source at ksize 5: the rows above, then the symmetric column order of SymmColumnVec_32f,
   s = fma(k[2], S[0], 0); s = fma(k[2+j], S[j] + S[-j], s) */
static void lap5_f32(const float* src, size_t sstep, float* d2x, float* d2y, int w, int h, int cn, int border,
                     const float* kd, const float* ks)
{
    const int we = w * cn;
    float* rd = (float*)malloc(sizeof(float) * (size_t)we * h);
    float* rs = (float*)malloc(sizeof(float) * (size_t)we * h);
    for (int y = 0; y < h; y++) {
        const float* row = (const float*)((const char*)src + (size_t)y * sstep);
        for (int x = 0; x < w; x++)
            for (int c = 0; c < cn; c++) {
                float v[5];
                for (int i = 0; i < 5; i++) {
                    int sx = port_border(x + i - 2, w, border);
                    v[i] = sx < 0 ? 0.f : row[sx * cn + c];
                }
                const int e = x * cn + c;
                rd[(size_t)y * we + e] = row5(v, kd, 1, e, we);
                rs[(size_t)y * we + e] = row5(v, ks, 0, e, we);
            }
    }
    for (int y = 0; y < h; y++)
        for (int e = 0; e < we; e++) {
            int s0 = port_border(y, h, border);
            float a = fmaf(ks[2], s0 < 0 ? 0.f : rd[(size_t)s0 * we + e], 0.f), b = fmaf(kd[2], s0 < 0 ? 0.f : rs[(size_t)s0 * we + e], 0.f);
            for (int j = 1; j <= 2; j++) {
                int p = port_border(y + j, h, border), m = port_border(y - j, h, border);
                float dp = p < 0 ? 0.f : rd[(size_t)p * we + e], dm = m < 0 ? 0.f : rd[(size_t)m * we + e];
                float sp = p < 0 ? 0.f : rs[(size_t)p * we + e], sm = m < 0 ? 0.f : rs[(size_t)m * we + e];
                a = fmaf(ks[2 + j], dp + dm, a);
                b = fmaf(kd[2 + j], sp + sm, b);
            }
            d2x[(size_t)y * we + e] = a;
            d2y[(size_t)y * we + e] = b;
        }
    free(rd);
    free(rs);
}

/* saturate_cast<uchar / short>(float) as the reference's x86 objects do it: cvRound is cvtss2si, which gives INT_MIN for NaN and for
   anything that does not fit 32 bits (an 8-bit source at large apertures reaches 2^31) */
static void lap_store(char* row, int ddepth, size_t e, float v)
{
    if (ddepth == P_32F) { ((float*)row)[e] = v; return; }
    const int r = (v >= -2147483648.f && v < 2147483648.f) ? (int)lrintf(v) : -2147483647 - 1;
    if (ddepth == P_8U) ((uchar*)row)[e] = port_sat_u8i(r);
    else ((short*)row)[e] = port_sat_s16i(r);
}

PORT_API int port_laplacian(const void* src, size_t sstep, void* dst, size_t dstep, int w, int h, int stype, int ddepth,
                            int ksize, double scale, double delta, int border)
{
    static const float K[2][9] = {{0, 1, 0, 1, -4, 1, 0, 1, 0}, {2, 0, 2, 0, -8, 0, 2, 0, 2}};
    const int sdepth = P_DEPTH(stype), cn = P_CN(stype);
    if (ddepth < 0) ddepth = sdepth;
    if (ksize < 1 || ksize > 31 || !(ksize & 1)) return -1;
    if (ksize <= 3) {
        float k[9];
        for (int i = 0; i < 9; i++) k[i] = scale != 1 ? K[ksize == 3][i] * (float)scale : K[ksize == 3][i];
        return port_filter2d(src, sstep, dst, dstep, w, h, stype, ddepth, k, 3, 3, -1, -1, delta, border);
    }
    float kd[32], ks[32];
    sobel_taps(ksize, 2, kd);
    sobel_taps(ksize, 0, ks);
    const int wdepth = sdepth == P_8U && ksize <= 5 ? P_16S : P_32F;
    const size_t we = (size_t)w * cn, wstep = we * port_esz(wdepth);
    char* d2x = (char*)malloc(wstep * h);
    char* d2y = (char*)malloc(wstep * h);
    if (sdepth == P_32F && ksize == 5) {
        lap5_f32((const float*)src, sstep, (float*)d2x, (float*)d2y, w, h, cn, border & ~16, kd, ks);
    } else {
        port_sep_filter_core(src, sstep, d2x, wstep, w, h, stype, wdepth, kd, ksize, ks, ksize, -1, -1, 0.0, border);
        port_sep_filter_core(src, sstep, d2y, wstep, w, h, stype, wdepth, ks, ksize, kd, ksize, -1, -1, 0.0, border);
    }
    const int plain = scale == 1 && delta == 0;
    const float a = (float)scale, b = (float)delta;
    for (int y = 0; y < h; y++) {
        const char *px = d2x + (size_t)y * wstep, *py = d2y + (size_t)y * wstep;
        char* drow = (char*)dst + (size_t)y * dstep;
        for (size_t e = 0; e < we; e++) {
            if (wdepth == P_16S) {
                const int v = port_sat_s16i(((const short*)px)[e] + ((const short*)py)[e]);
                lap_store(drow, ddepth, e, plain ? (float)v : fmaf((float)v, a, b));
            } else {
                const float v = ((const float*)px)[e] + ((const float*)py)[e];
                lap_store(drow, ddepth, e, plain ? v : fmaf(v, a, b));
            }
        }
    }
    free(d2x);
    free(d2y);
    return 0;
}
