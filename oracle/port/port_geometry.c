/* oracle/port/port_geometry.c -- cv::resize / cv::warpAffine / cv::warpPerspective restated in scalar C.
 * TEST INFRASTRUCTURE ONLY (see port_common.h).
 *   hal::resize               modules/imgproc/src/resize.cpp:3826-4194 (tables :4097-4190)
 *   resizeNN                  :1121-1172 ; HResizeLinear :1877-1928 ; VResizeLinear<uchar> :1963-1989
 *   HResizeCubic              :1993-2041 ; VResizeCubic + VResizeCubicVec_32s8u (SSE body) :1408-1444, :2044-2062
 *   resizeAreaFast (2x2)      :2919-3068
 *   cv::warpAffine            modules/imgproc/src/imgwarp.cpp:2788-2902, hal::warpAffine :2673-2700, blocklines :2702-2782
 *   cv::warpPerspective       :3370-3466, WarpPerspectiveInvoker :3160-3226, blocklines :3299-3365, cv::invert 3x3 core/src/lapack.cpp:944-970
 *   remapNearest/Bilinear/Bicubic :329-430, :675-904, :907-1010 ; initInterTab2D :213-287
 */
#include "port_common.h"

static int clipi(int x, int a, int b) { return x >= a ? (x < b ? x : b - 1) : a; }

static void cubic_c(float x, float* c)
{
    const float A = -0.75f;
    c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
    c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
    c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
    c[3] = 1.f - c[0] - c[1] - c[2];
}

/* interpolateLanczos4, resize.cpp:974-1003: sin / cos of the first tap's angle in double, the other seven by the 45-degree rotation table */
static void lanczos4_c(float x, float* c)
{
    static const double s45 = 0.70710678118654752440084436210485;
    static const double cs[][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
    float sum = 0;
    double y0 = -(x + 3) * 3.1415926535897932384626433832795 * 0.25, s0 = sin(y0), c0 = cos(y0);
    for (int i = 0; i < 8; i++) {
        float y0_ = (x + 3 - i);
        if (fabsf(y0_) >= 1e-6f) {
            double y = -y0_ * 3.1415926535897932384626433832795 * 0.25;
            c[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
        } else c[i] = 1e30f;
        sum += c[i];
    }
    sum = 1.f / sum;
    for (int i = 0; i < 8; i++) c[i] *= sum;
}

static short s16(float v) { return port_sat_s16i((int)lrintf(v)); }

#define SRC(y, x, c) (depth == P_8U ? (float)((const uchar*)src + (size_t)(y) * sstep)[(x) * cn + (c)] : ((const float*)((const char*)src + (size_t)(y) * sstep))[(x) * cn + (c)])

/* inv_x, inv_y: the inverse sampling scales hal::resize gets, dsize / ssize unless the caller gave fx, fy (resize.cpp:4214-4228) */
static int resize_scaled(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type, int interp,
                         double inv_x, double inv_y)
{
    int depth = P_DEPTH(type), cn = P_CN(type), es = (int)port_esz(depth) * cn;
    double scale_x = 1. / inv_x, scale_y = 1. / inv_y;
    if (depth != P_8U && depth != P_32F) return 1;
    if (dw == sw && dh == sh) {
        for (int y = 0; y < sh; y++) memcpy((char*)dst + (size_t)y * dstep, (const char*)src + (size_t)y * sstep, (size_t)sw * es);
        return 0;
    }
    if (interp == 0) {
        double ifx = 1. / inv_x, ify = 1. / inv_y;
        for (int y = 0; y < dh; y++) {
            int sy = (int)floor(y * ify); if (sy > sh - 1) sy = sh - 1;
            for (int x = 0; x < dw; x++) {
                int sx = (int)floor(x * ifx); if (sx > sw - 1) sx = sw - 1;
                memcpy((char*)dst + (size_t)y * dstep + (size_t)x * es, (const char*)src + (size_t)sy * sstep + (size_t)sx * es, es);
            }
        }
        return 0;
    }
    int isx = port_round(scale_x), isy = port_round(scale_y);
    int area_fast = fabs(scale_x - isx) < 2.220446049250313e-16 && fabs(scale_y - isy) < 2.220446049250313e-16;
    if (interp == 5 && depth == P_32F) interp = 1;       /* cv::resize, resize.cpp:4223: float data has no exact mode */
    if ((interp == 1 || interp == 3 || interp == 5) && area_fast && isx == 2 && isy == 2) {   /* LINEAR_EXACT 2 x 2: resize.cpp:3976-3981 */
        for (int y = 0; y < dh; y++)
            for (int x = 0; x < dw; x++)
                for (int c = 0; c < cn; c++) {
                    if (depth == P_8U) {
                        const uchar* s0 = (const uchar*)src + (size_t)(2 * y) * sstep + 2 * x * cn + c; const uchar* s1 = s0 + sstep;
                        ((uchar*)dst + (size_t)y * dstep)[x * cn + c] = (uchar)((s0[0] + s0[cn] + s1[0] + s1[cn] + 2) >> 2);
                    } else {
                        const float* s0 = (const float*)((const char*)src + (size_t)(2 * y) * sstep) + 2 * x * cn + c;
                        const float* s1 = (const float*)((const char*)s0 + sstep);
                        /* 4-lane SIMD body: (a+b)+(c+d); 3 channels and the single-channel remainder columns (dw % 4): scalar loop,
                         * sum = 0; sum += ((a+b)+c)+d -- -0 comes out as +0 */
                        int seq = cn == 3 || (cn == 1 && x >= (dw & ~3));
                        float sum = seq ? 0.f + (((s0[0] + s0[cn]) + s1[0]) + s1[cn]) : (s0[0] + s0[cn]) + (s1[0] + s1[cn]);
                        ((float*)((char*)dst + (size_t)y * dstep))[x * cn + c] = sum * 0.25f;
                    }
                }
        return 0;
    }
    if (interp == 6) {
        /* INTER_NEAREST_EXACT (resizeNN_bitexact, resize.cpp:1267-1288): 16.16 fixed-point source coordinate of the pixel centre */
        if (sw >= 32768 || sh >= 32768) return 1;
        int ifx = ((sw << 16) + dw / 2) / dw, ifx0 = ifx / 2 - sw % 2, ify = ((sh << 16) + dh / 2) / dh, ify0 = ify / 2 - sh % 2;
        for (int y = 0; y < dh; y++) {
            int sy = (ify * y + ify0) >> 16; if (sy > sh - 1) sy = sh - 1;
            for (int x = 0; x < dw; x++) {
                int sx = (ifx * x + ifx0) >> 16; if (sx > sw - 1) sx = sw - 1;
                memcpy((char*)dst + (size_t)y * dstep + (size_t)x * es, (const char*)src + (size_t)sy * sstep + (size_t)sx * es, es);
            }
        }
        return 0;
    }
    if (interp == 5) {
        /* INTER_LINEAR_EXACT for 8-bit data (resize_bitExact<uint8_t, interpolationLinear>, resize.cpp:776-960; fixedpoint.inl.hpp:326-374):
         * 8.8 fixed-point weights c1 = cvRound((f - floor f) * 256), c0 = 256 - c1 from f = (1/inv_scale) * (d + 0.5) - 0.5 in double;
         * positions left of the first / right of the last source sample copy it; rows: H = c0*p0 + c1*p1 (16-bit), columns:
         * (H0*b0 + H1*b1 + 2^15) >> 16, or (H + 128) >> 8 for the copied rows. */
        int* ofs[2]; unsigned short* co[2]; int mn[2], mx[2];
        for (int pass = 0; pass < 2; pass++) {
            int dn = pass ? dh : dw, sn = pass ? sh : sw; double scale = 1.0 / (pass ? inv_y : inv_x);
            ofs[pass] = (int*)calloc((size_t)dn, sizeof(int)); co[pass] = (unsigned short*)calloc((size_t)dn * 2, sizeof(unsigned short));
            int minofst = 0, maxofst = dn;
            for (int d = 0; d < dn; d++) {
                volatile double t = scale * (d + 0.5); double fval = t - 0.5;
                int ival = (int)floor(fval);
                if (ival >= 0 && sn > 1) {
                    if (ival < sn - 1) {
                        ofs[pass][d] = ival;
                        volatile double fr = fval - ival; double q = fr * 256.0;
                        co[pass][2 * d + 1] = (unsigned short)port_round(q);
                        co[pass][2 * d] = (unsigned short)(256 - co[pass][2 * d + 1]);
                    } else { ofs[pass][d] = sn - 1; if (d < maxofst) maxofst = d; }
                } else if (d + 1 > minofst) minofst = d + 1;
            }
            mn[pass] = minofst; mx[pass] = maxofst;
        }
        for (int y = 0; y < dh; y++)
            for (int x = 0; x < dw; x++)
                for (int c = 0; c < cn; c++) {
                    unsigned H[2]; int rows[2], nr;
                    if (y < mn[1]) { rows[0] = 0; nr = 1; } else if (y >= mx[1]) { rows[0] = sh - 1; nr = 1; } else { rows[0] = ofs[1][y]; rows[1] = rows[0] + 1; nr = 2; }
                    for (int r = 0; r < nr; r++) {
                        const uchar* sp = (const uchar*)src + (size_t)rows[r] * sstep;
                        if (x < mn[0]) H[r] = (unsigned)sp[c] << 8;
                        else if (x >= mx[0]) H[r] = (unsigned)sp[(sw - 1) * cn + c] << 8;
                        else {
                            unsigned a = co[0][2 * x] * sp[ofs[0][x] * cn + c], b = co[0][2 * x + 1] ? co[0][2 * x + 1] * sp[(ofs[0][x] + 1) * cn + c] : 0;
                            if (a > 65535) a = 65535; if (b > 65535) b = 65535;
                            H[r] = a + b > 65535 ? 65535 : a + b;
                        }
                    }
                    unsigned v;
                    if (nr == 1) v = ((H[0] + 128) & 0xFFFF) >> 8;
                    else v = (H[0] * co[1][2 * y] + H[1] * co[1][2 * y + 1] + 32768u) >> 16;
                    ((uchar*)dst + (size_t)y * dstep)[x * cn + c] = (uchar)(v > 255 ? 255 : v);
                }
        free(ofs[0]); free(ofs[1]); free(co[0]); free(co[1]);
        return 0;
    }
    if (interp == 3) {
        /* INTER_AREA, true area mode only (both scales >= 1; resize.cpp:4016-4064).  Integer scales: plain window sum times float(1/area)
         * (resizeAreaFast_Invoker :2969-3060; float sums in groups of four, CV_ENABLE_UNROLLED); otherwise the DecimateAlpha tables of
         * computeResizeAreaTab (:3334-3373) and ResizeArea_Invoker (:3183-3297): per source row buf = sum_k S*alpha_k, per destination
         * row sum = beta_0*buf_0, then sum += beta_j*buf_j; all in float, no fused operations; cvRound at the end for 8-bit data. */
        if (scale_x < 1 || scale_y < 1) goto area_as_linear;      /* an enlarging axis: bilinear with area-mode weights, below */
        if (area_fast) {
            const int area = isx * isy;
            const float scale = 1.f / area;
            for (int y = 0; y < dh; y++)
                for (int x = 0; x < dw; x++)
                    for (int c = 0; c < cn; c++) {
                        if (depth == P_8U) {
                            int sum = 0;
                            for (int j = 0; j < isy; j++)
                                for (int i = 0; i < isx; i++) sum += ((const uchar*)src + (size_t)(y * isy + j) * sstep)[(x * isx + i) * cn + c];
                            ((uchar*)dst + (size_t)y * dstep)[x * cn + c] = port_sat_u8f((float)sum * scale);
                        } else {
                            float v[4], sum = 0; int k = 0, n = 0;
                            for (int j = 0; j < isy; j++)
                                for (int i = 0; i < isx; i++) {
                                    float s = ((const float*)((const char*)src + (size_t)(y * isy + j) * sstep))[(x * isx + i) * cn + c];
                                    if (k <= area - 4 || n) { v[n++] = s; if (n == 4) { sum += ((v[0] + v[1]) + v[2]) + v[3]; n = 0; k += 4; } }
                                    else { sum += s; k++; }
                                }
                            ((float*)((char*)dst + (size_t)y * dstep))[x * cn + c] = sum * scale;
                        }
                    }
            return 0;
        }
        typedef struct { int si, di; float alpha; } DecAlpha;
        DecAlpha* tabs[2]; int tn[2];
        for (int pass = 0; pass < 2; pass++) {
            int ssize = pass ? sh : sw, dsize = pass ? dh : dw; double scale = pass ? scale_y : scale_x;
            DecAlpha* tab = (DecAlpha*)malloc(sizeof(DecAlpha) * (size_t)ssize * 2 + 64);
            int k = 0;
            for (int dx = 0; dx < dsize; dx++) {
                double fsx1 = dx * scale, fsx2 = fsx1 + scale, cell = scale < ssize - fsx1 ? scale : ssize - fsx1;
                int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
                if (sx2 > ssize - 1) sx2 = ssize - 1;
                if (sx1 > sx2) sx1 = sx2;
                if (sx1 - fsx1 > 1e-3) { tab[k].di = dx; tab[k].si = sx1 - 1; tab[k++].alpha = (float)((sx1 - fsx1) / cell); }
                for (int sx = sx1; sx < sx2; sx++) { tab[k].di = dx; tab[k].si = sx; tab[k++].alpha = (float)(1.0 / cell); }
                if (fsx2 - sx2 > 1e-3) {
                    double m = fsx2 - sx2 < 1. ? fsx2 - sx2 : 1.; if (cell < m) m = cell;
                    tab[k].di = dx; tab[k].si = sx2; tab[k++].alpha = (float)(m / cell);
                }
            }
            tabs[pass] = tab; tn[pass] = k;
        }
        float* buf = (float*)malloc(sizeof(float) * (size_t)dw * cn * 2); float* sum = buf + (size_t)dw * cn;
        int prev_dy = tabs[1][0].di;
        for (int e = 0; e < dw * cn; e++) sum[e] = 0;
        for (int j = 0; j <= tn[1]; j++) {
            if (j == tn[1] || tabs[1][j].di != prev_dy) {
                for (int e = 0; e < dw * cn; e++) {
                    if (depth == P_8U) ((uchar*)dst + (size_t)prev_dy * dstep)[e] = port_sat_u8f(sum[e]);
                    else ((float*)((char*)dst + (size_t)prev_dy * dstep))[e] = sum[e];
                }
                if (j == tn[1]) break;
            }
            const float beta = tabs[1][j].alpha; const int sy = tabs[1][j].si, dy = tabs[1][j].di;
            for (int e = 0; e < dw * cn; e++) buf[e] = 0;
            for (int k = 0; k < tn[0]; k++)
                for (int c = 0; c < cn; c++) {
                    float sv = depth == P_8U ? (float)((const uchar*)src + (size_t)sy * sstep)[tabs[0][k].si * cn + c]
                                             : ((const float*)((const char*)src + (size_t)sy * sstep))[tabs[0][k].si * cn + c];
                    buf[tabs[0][k].di * cn + c] += sv * tabs[0][k].alpha;
                }
            if (dy != prev_dy) { for (int e = 0; e < dw * cn; e++) sum[e] = beta * buf[e]; prev_dy = dy; }
            else for (int e = 0; e < dw * cn; e++) sum[e] += beta * buf[e];
        }
        free(buf); free(tabs[0]); free(tabs[1]);
        return 0;
    }
    if (interp == 4) {
        /* INTER_LANCZOS4 (resize.cpp:974-1003 weights, :2066-2116 rows, :2119-2157 + :1596-1621 columns): 8 taps at s-3 .. s+4 around
         * s = floor((d + 0.5) * scale - 0.5), indices clamped to the image; 8-bit: weights cvRound(w * 2048) as shorts, int sums,
         * (v + 2^21) >> 22; float: rows summed left to right, columns right to left in the 4-lane SIMD body
         * (S0*b0 + (S1*b1 + ... (S6*b6 + S7*b7))) and left to right in the last (dw * cn) % 4 elements; no fused operations. */
        int* os[2]; float* co[2];
        for (int pass = 0; pass < 2; pass++) {
            int dn = pass ? dh : dw; double sc = pass ? scale_y : scale_x;
            os[pass] = (int*)malloc(sizeof(int) * (size_t)dn); co[pass] = (float*)malloc(sizeof(float) * 8 * (size_t)dn);
            for (int d = 0; d < dn; d++) {
                float f = (float)((d + 0.5) * sc - 0.5); int s = (int)floorf(f); f -= s;
                os[pass][d] = s;
                lanczos4_c(f, co[pass] + 8 * d);
            }
        }
        const int body = ((dw * cn) / 4) * 4;
        for (int y = 0; y < dh; y++)
            for (int x = 0; x < dw; x++)
                for (int c = 0; c < cn; c++) {
                    int xi[8], yi[8], e = x * cn + c;
                    for (int j = 0; j < 8; j++) { xi[j] = clipi(os[0][x] - 3 + j, 0, sw); yi[j] = clipi(os[1][y] - 3 + j, 0, sh); }
                    const float* a = co[0] + 8 * x; const float* b = co[1] + 8 * y;
                    if (depth == P_8U) {
                        int t[8], v = 0;
                        for (int k = 0; k < 8; k++) {
                            const uchar* r = (const uchar*)src + (size_t)yi[k] * sstep; t[k] = 0;
                            for (int j = 0; j < 8; j++) t[k] += r[xi[j] * cn + c] * s16(a[j] * 2048.f);
                        }
                        for (int k = 0; k < 8; k++) v = (int)((unsigned)v + (unsigned)t[k] * (unsigned)(int)s16(b[k] * 2048.f));
                        ((uchar*)dst + (size_t)y * dstep)[e] = port_sat_u8i((int)((unsigned)v + (1u << 21)) >> 22);
                    } else {
                        float t[8], o;
                        for (int k = 0; k < 8; k++) {
                            const float* r = (const float*)((const char*)src + (size_t)yi[k] * sstep);
                            float v = r[xi[0] * cn + c] * a[0];
                            for (int j = 1; j < 8; j++) v += r[xi[j] * cn + c] * a[j];
                            t[k] = v;
                        }
                        if (e < body) { o = t[7] * b[7]; for (int k = 6; k >= 0; k--) o = t[k] * b[k] + o; }
                        else { o = t[0] * b[0]; for (int k = 1; k < 8; k++) o += t[k] * b[k]; }
                        ((float*)((char*)dst + (size_t)y * dstep))[e] = o;
                    }
                }
        free(os[0]); free(os[1]); free(co[0]); free(co[1]);
        return 0;
    }
area_as_linear:;
    /* INTER_AREA with a factor < 1 on either axis (resize.cpp:4071, :4104-4109, :4158-4163): the bilinear kernel with
     * s = floor(d * scale), f = (d + 1) - (s + 1) * inv_scale, f = f <= 0 ? 0 : f - floor(f) on BOTH axes */
    const int area_mode = interp == 3;
    if (area_mode) interp = 1;
    if (interp != 1 && interp != 2) return 1;
    int cubic = interp == 2;
    /* tables */
    int* xs = (int*)malloc(sizeof(int) * (dw + dh)); int* ys = xs + dw;
    float* xa = (float*)malloc(sizeof(float) * 4 * (dw + dh)); float* ya = xa + 4 * dw;
    for (int pass = 0; pass < 2; pass++) {
        int dn = pass ? dh : dw, sn = pass ? sh : sw; double sc = pass ? scale_y : scale_x;
        for (int d = 0; d < dn; d++) {
            float f; int s;
            if (!area_mode) { f = (float)((d + 0.5) * sc - 0.5); s = (int)floorf(f); f -= s; }
            else {
                s = (int)floor(d * sc);
                volatile double m = (s + 1) * (pass ? inv_y : inv_x);
                f = (float)((d + 1) - m);
                f = f <= 0 ? 0.f : f - floorf(f);
            }
            if (!cubic && !pass) { if (s < 0) { f = 0; s = 0; } if (s >= sn - 1) { f = 0; s = sn - 1; } }
            float* c = (pass ? ya : xa) + 4 * d;
            if (cubic) cubic_c(f, c); else { c[0] = 1.f - f; c[1] = f; c[2] = c[3] = 0; }
            (pass ? ys : xs)[d] = s;
        }
    }
    int vec8 = ((dw * cn) / 8) * 8, vec4 = ((dw * cn) / 4) * 4;
    for (int y = 0; y < dh; y++)
        for (int x = 0; x < dw; x++)
            for (int c = 0; c < cn; c++) {
                int e = x * cn + c;
                if (!cubic) {
                    int sy0 = clipi(ys[y], 0, sh), sy1 = clipi(ys[y] + 1, 0, sh), sx = xs[x], last = sx >= sw - 1;
                    if (depth == P_8U) {
                        int a0 = s16(xa[4 * x] * 2048.f), a1 = s16(xa[4 * x + 1] * 2048.f), b0 = s16(ya[4 * y] * 2048.f), b1 = s16(ya[4 * y + 1] * 2048.f);
                        const uchar* r0 = (const uchar*)src + (size_t)sy0 * sstep + sx * cn + c; const uchar* r1 = (const uchar*)src + (size_t)sy1 * sstep + sx * cn + c;
                        int t0 = last ? r0[0] * 2048 : r0[0] * a0 + r0[cn] * a1, t1 = last ? r1[0] * 2048 : r1[0] * a0 + r1[cn] * a1;
                        ((uchar*)dst + (size_t)y * dstep)[e] = (uchar)((((b0 * (t0 >> 4)) >> 16) + ((b1 * (t1 >> 4)) >> 16) + 2) >> 2);
                    } else {
                        float a0 = xa[4 * x], a1 = xa[4 * x + 1], b0 = ya[4 * y], b1 = ya[4 * y + 1];
                        const float* r0 = (const float*)((const char*)src + (size_t)sy0 * sstep) + sx * cn + c; const float* r1 = (const float*)((const char*)src + (size_t)sy1 * sstep) + sx * cn + c;
                        float t0 = last ? r0[0] : r0[0] * a0 + r0[cn] * a1, t1 = last ? r1[0] : r1[0] * a0 + r1[cn] * a1;
                        ((float*)((char*)dst + (size_t)y * dstep))[e] = t0 * b0 + t1 * b1;
                    }
                } else {
                    int xi[4], yi[4];
                    for (int j = 0; j < 4; j++) { xi[j] = clipi(xs[x] - 1 + j, 0, sw); yi[j] = clipi(ys[y] - 1 + j, 0, sh); }
                    if (depth == P_8U) {
                        int ia[4], ib[4], t[4];
                        for (int j = 0; j < 4; j++) { ia[j] = s16(xa[4 * x + j] * 2048.f); ib[j] = s16(ya[4 * y + j] * 2048.f); }
                        for (int k = 0; k < 4; k++) { const uchar* r = (const uchar*)src + (size_t)yi[k] * sstep; t[k] = 0; for (int j = 0; j < 4; j++) t[k] += r[xi[j] * cn + c] * ia[j]; }
                        uchar o;
                        if (e < vec8) {      /* SSE body: float, S0*b0 + (S1*b1 + (S2*b2 + S3*b3)), b = beta/2^22, round-half-even */
                            const float sc = 1.f / (2048.f * 2048.f);
                            float v = (float)t[3] * (ib[3] * sc);
                            v = (float)t[2] * (ib[2] * sc) + v; v = (float)t[1] * (ib[1] * sc) + v; v = (float)t[0] * (ib[0] * sc) + v;
                            o = port_sat_u8i((int)lrintf(v));
                        } else o = port_sat_u8i((t[0] * ib[0] + t[1] * ib[1] + t[2] * ib[2] + t[3] * ib[3] + (1 << 21)) >> 22);
                        ((uchar*)dst + (size_t)y * dstep)[e] = o;
                    } else {
                        float t[4];
                        for (int k = 0; k < 4; k++) {
                            const float* r = (const float*)((const char*)src + (size_t)yi[k] * sstep);
                            float v = r[xi[0] * cn + c] * xa[4 * x]; v += r[xi[1] * cn + c] * xa[4 * x + 1]; v += r[xi[2] * cn + c] * xa[4 * x + 2]; v += r[xi[3] * cn + c] * xa[4 * x + 3];
                            t[k] = v;
                        }
                        const float* b = ya + 4 * y; float o;
                        if (e < vec4) { o = t[3] * b[3]; o = t[2] * b[2] + o; o = t[1] * b[1] + o; o = t[0] * b[0] + o; }
                        else { o = t[0] * b[0]; o += t[1] * b[1]; o += t[2] * b[2]; o += t[3] * b[3]; }
                        ((float*)((char*)dst + (size_t)y * dstep))[e] = o;
                    }
                }
            }
    free(xs); free(xa);
    return 0;
}

PORT_API int port_resize(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type, int interp)
{
    return resize_scaled(src, sstep, sw, sh, dst, dstep, dw, dh, type, interp, (double)dw / sw, (double)dh / sh);
}

/* cv::resize(src, dst, Size(), fx, fy): dst is round(sw * fx) x round(sh * fy), the sampling scales stay fx, fy.  NEAREST, LINEAR and
 * CUBIC, and the exact 2 x 2 decimation on even sizes (the reference's partial last windows for odd sizes are not restated); 1 otherwise */
PORT_API int port_resize_fxfy(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type, int interp,
                              double fx, double fy)
{
    if (interp != 0 && interp != 1 && interp != 2) return 1;
    if (fx == 0.5 && fy == 0.5 && interp == 1 && (2 * dw != sw || 2 * dh != sh)) return 1;
    return resize_scaled(src, sstep, sw, sh, dst, dstep, dw, dh, type, interp, fx, fy);
}

/* ---- remap tables ---- */
static float g_lin_f[1024 * 4], g_cub_f[1024 * 16];
static short g_lin_i[1024 * 4], g_cub_i[1024 * 16];
static void build_tabs(void)
{
    static int done = 0;
    if (done) return;
    for (int ks = 2; ks <= 4; ks += 2) {
        float t1[32 * 4]; float* ft = ks == 2 ? g_lin_f : g_cub_f; short* it = ks == 2 ? g_lin_i : g_cub_i;
        for (int i = 0; i < 32; i++) { float x = i * (1.f / 32); if (ks == 2) { t1[i * 2] = 1.f - x; t1[i * 2 + 1] = x; } else cubic_c(x, t1 + i * 4); }
        for (int iy = 0; iy < 32; iy++)
            for (int ix = 0; ix < 32; ix++) {
                float* f = ft + (iy * 32 + ix) * ks * ks; short* q = it + (iy * 32 + ix) * ks * ks; int total = 0;
                for (int a = 0; a < ks; a++) for (int b = 0; b < ks; b++) { float v = t1[iy * ks + a] * t1[ix * ks + b]; f[a * ks + b] = v; q[a * ks + b] = s16(v * 32768.f); total += q[a * ks + b]; }
                int res = total - 32768;
                if (res && ks == 2) q[3] = (short)(q[3] - res);
                else if (res) {
                    int lo = 10, hi = 10; const int idx[4] = {10, 11, 14, 15};
                    for (int k = 0; k < 4; k++) { if (q[idx[k]] < q[lo]) lo = idx[k]; else if (q[idx[k]] > q[hi]) hi = idx[k]; }
                    int tg = res < 0 ? hi : lo; q[tg] = (short)(q[tg] - res);
                }
            }
    }
    done = 1;
}

/* cvRound / v_round on x86: nearest-even, 0x80000000 for NaN and values outside int32 */
static int x86_round(float v) { return fabsf(v) < 2147483648.f ? (int)lrintf(v) : (int)0x80000000; }

typedef struct { const void* m1; size_t s1; int t1; const void* m2; size_t s2; int t2; } PortMaps;

/* cv::remap coordinates (RemapInvoker, imgwarp.cpp:1164-1283): float maps are rounded (NEAREST) or scaled by 32 and rounded into a
   5-bit-fraction fixed point; fixed-point maps are used as they are (NEAREST rounds the fractions through NNDeltaTab_i) */
static void map_coords(const PortMaps* mp, int x, int y, int interp, int* sx, int* sy, int* a)
{
    *a = 0;
    if (P_DEPTH(mp->t1) == P_16S) {
        const short* xy = (const short*)((const char*)mp->m1 + (size_t)y * mp->s1) + 2 * x;
        int fr = mp->m2 ? (((const unsigned short*)((const char*)mp->m2 + (size_t)y * mp->s2))[x] & 1023) : 0;
        /* NNDeltaTab_i is filled as (fraction < 1/2) (imgwarp.cpp:237-238) -- and only once a bilinear table has been built in the process;
           before that it is all zeros.  The table as built is what is reproduced here.  Without a fraction map the coordinates are
           "already in the right format" (:1166) and the table is not consulted. */
        if (interp == 0 && !mp->m2) { *sx = xy[0]; *sy = xy[1]; }
        else if (interp == 0) { *sx = (short)(xy[0] + ((fr & 31) < 16)); *sy = (short)(xy[1] + ((fr >> 5) < 16)); }
        else { *sx = xy[0]; *sy = xy[1]; *a = fr; }
        return;
    }
    float mx, my;
    if (mp->m2) { mx = ((const float*)((const char*)mp->m1 + (size_t)y * mp->s1))[x]; my = ((const float*)((const char*)mp->m2 + (size_t)y * mp->s2))[x]; }
    else { const float* q = (const float*)((const char*)mp->m1 + (size_t)y * mp->s1) + 2 * x; mx = q[0]; my = q[1]; }
    if (interp == 0) { *sx = port_sat_s16i(x86_round(mx)); *sy = port_sat_s16i(x86_round(my)); }
    else {
        int ix = x86_round(mx * 32.f), iy = x86_round(my * 32.f);
        *sx = port_sat_s16i(ix >> 5); *sy = port_sat_s16i(iy >> 5); *a = (iy & 31) * 32 + (ix & 31);
    }
}

static int warp_impl(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type, const double* M, int persp,
                     int interp, int border, const double* bv, const PortMaps* maps)
{
    int depth = P_DEPTH(type), cn = P_CN(type);
    if (depth != P_8U && depth != P_32F) return 1;
    if (interp == 3) interp = 1;
    if (interp > 2) return 1;
    build_tabs();
    border &= ~16;
    float cvf[4]; int cvi[4];
    for (int c = 0; c < 4; c++) { cvf[c] = (float)bv[c]; cvi[c] = port_sat_u8i((int)lrint(bv[c])); }
    int bh0 = dh < 16 ? dh : 16, bw0 = 1024 / bh0; if (bw0 > dw) bw0 = dw;
    for (int y = 0; y < dh; y++)
        for (int x = 0; x < dw; x++) {
            int sx, sy, a = 0;
            if (maps) map_coords(maps, x, y, interp, &sx, &sy, &a);
            else if (!persp) {
                int rd = interp == 0 ? 512 : 16;
                int ad = port_round(M[0] * x * 1024), bd = port_round(M[3] * x * 1024);
                int X0 = port_round((M[1] * y + M[2]) * 1024) + rd, Y0 = port_round((M[4] * y + M[5]) * 1024) + rd;
                if (interp == 0) { sx = port_sat_s16i((X0 + ad) >> 10); sy = port_sat_s16i((Y0 + bd) >> 10); }
                else { int X = (X0 + ad) >> 5, Y = (Y0 + bd) >> 5; sx = port_sat_s16i(X >> 5); sy = port_sat_s16i(Y >> 5); a = (Y & 31) * 32 + (X & 31); }
            } else {
                int xb = (x / bw0) * bw0, x1 = x - xb;
                double X0 = M[0] * xb + M[1] * y + M[2], Y0 = M[3] * xb + M[4] * y + M[5], W0 = M[6] * xb + M[7] * y + M[8];
                double W = W0 + M[6] * x1; W = W ? (interp == 0 ? 1. : 32.) / W : 0;
                double fX = fmax(-2147483648.0, fmin(2147483647.0, (X0 + M[0] * x1) * W)), fY = fmax(-2147483648.0, fmin(2147483647.0, (Y0 + M[3] * x1) * W));
                int X = port_round(fX), Y = port_round(fY);
                if (interp == 0) { sx = port_sat_s16i(X); sy = port_sat_s16i(Y); } else { sx = port_sat_s16i(X >> 5); sy = port_sat_s16i(Y >> 5); a = (Y & 31) * 32 + (X & 31); }
            }
            for (int c = 0; c < cn; c++) {
                float outf = 0; int outi = 0;
#define PIX(yy, xx) (((yy) < 0 || (xx) < 0) ? (depth == P_8U ? (float)cvi[c] : cvf[c]) : SRC(yy, xx, c))
                if (interp == 0) {
                    int qx, qy;
                    if ((unsigned)sx < (unsigned)sw && (unsigned)sy < (unsigned)sh) { qx = sx; qy = sy; }
                    else if (border == PB_REPLICATE) { qx = clipi(sx, 0, sw); qy = clipi(sy, 0, sh); }
                    else if (border == PB_CONSTANT) { qx = qy = -1; }
                    else { qx = port_border(sx, sw, border); qy = port_border(sy, sh, border); }
                    outf = PIX(qy, qx); outi = (int)outf;
                } else if (interp == 1) {
                    if (border == PB_CONSTANT && (sx >= sw || sx + 1 < 0 || sy >= sh || sy + 1 < 0)) { outf = cvf[c]; outi = cvi[c]; }
                    else {
                        int x0, x1, y0, y1;
                        if ((unsigned)sx < (unsigned)(sw - 1) && (unsigned)sy < (unsigned)(sh - 1)) { x0 = sx; x1 = sx + 1; y0 = sy; y1 = sy + 1; }
                        else if (border == PB_REPLICATE) { x0 = clipi(sx, 0, sw); x1 = clipi(sx + 1, 0, sw); y0 = clipi(sy, 0, sh); y1 = clipi(sy + 1, 0, sh); }
                        else { x0 = port_border(sx, sw, border); x1 = port_border(sx + 1, sw, border); y0 = port_border(sy, sh, border); y1 = port_border(sy + 1, sh, border); }
                        float v0 = PIX(y0, x0), v1 = PIX(y0, x1), v2 = PIX(y1, x0), v3 = PIX(y1, x1);
                        if (depth == P_8U) { const short* w = g_lin_i + a * 4; outi = port_sat_u8i(((int)v0 * w[0] + (int)v1 * w[1] + (int)v2 * w[2] + (int)v3 * w[3] + (1 << 14)) >> 15); }
                        else { const float* w = g_lin_f + a * 4; outf = v0 * w[0] + v1 * w[1] + v2 * w[2] + v3 * w[3]; }
                    }
                } else {
                    int bx = sx - 1, by = sy - 1;
                    int inl = (unsigned)bx < (unsigned)(sw - 3 > 0 ? sw - 3 : 0) && (unsigned)by < (unsigned)(sh - 3 > 0 ? sh - 3 : 0);
                    if (!inl && border == PB_CONSTANT && (bx >= sw || bx + 4 <= 0 || by >= sh || by + 4 <= 0)) { outf = cvf[c]; outi = cvi[c]; }
                    else {
                        int xs4[4], ys4[4];
                        for (int i = 0; i < 4; i++) { xs4[i] = inl ? bx + i : port_border(bx + i, sw, border); ys4[i] = inl ? by + i : port_border(by + i, sh, border); }
                        if (depth == P_8U) {
                            const short* w = g_cub_i + a * 16; int sum = 0;
                            for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) sum += (int)PIX(ys4[i], xs4[j]) * w[i * 4 + j];
                            outi = port_sat_u8i((sum + (1 << 14)) >> 15);
                        } else {
                            const float* w = g_cub_f + a * 16;
                            if (inl) {
                                float sum = 0;
                                for (int i = 0; i < 4; i++) { float rs = SRC(ys4[i], xs4[0], c) * w[i * 4] + SRC(ys4[i], xs4[1], c) * w[i * 4 + 1] + SRC(ys4[i], xs4[2], c) * w[i * 4 + 2] + SRC(ys4[i], xs4[3], c) * w[i * 4 + 3]; sum = i ? sum + rs : rs; }
                                outf = sum;
                            } else {
                                float cv = cvf[c], sum = cv;
                                for (int i = 0; i < 4; i++) { if (ys4[i] < 0) continue; for (int j = 0; j < 4; j++) if (xs4[j] >= 0) sum += (SRC(ys4[i], xs4[j], c) - cv) * w[i * 4 + j]; }
                                outf = sum;
                            }
                        }
                    }
                }
                if (depth == P_8U) ((uchar*)dst + (size_t)y * dstep)[x * cn + c] = (uchar)outi;
                else ((float*)((char*)dst + (size_t)y * dstep))[x * cn + c] = outf;
            }
        }
    return 0;
}

PORT_API int port_warp_affine(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type, const double* M0,
                              int flags, int border, const double* bv)
{
    double M[9] = {M0[0], M0[1], M0[2], M0[3], M0[4], M0[5], 0, 0, 1};
    if (!(flags & 16)) {
        double D = M[0] * M[4] - M[1] * M[3]; D = D != 0 ? 1. / D : 0;
        double A11 = M[4] * D, A22 = M[0] * D;
        M[0] = A11; M[1] *= -D; M[3] *= -D; M[4] = A22;
        double b1 = -M[0] * M[2] - M[1] * M[5], b2 = -M[3] * M[2] - M[4] * M[5];
        M[2] = b1; M[5] = b2;
    }
    return warp_impl(src, sstep, sw, sh, dst, dstep, dw, dh, type, M, 0, flags & 7, border, bv, NULL);
}

PORT_API int port_warp_perspective(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type, const double* m,
                                   int flags, int border, const double* bv)
{
    double M[9];
    memcpy(M, m, sizeof(M));
    if (!(flags & 16)) {
        double det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
        if (det != 0.) {
            double d = 1. / det;
            M[0] = (m[4] * m[8] - m[5] * m[7]) * d; M[1] = (m[2] * m[7] - m[1] * m[8]) * d; M[2] = (m[1] * m[5] - m[2] * m[4]) * d;
            M[3] = (m[5] * m[6] - m[3] * m[8]) * d; M[4] = (m[0] * m[8] - m[2] * m[6]) * d; M[5] = (m[2] * m[3] - m[0] * m[5]) * d;
            M[6] = (m[3] * m[7] - m[4] * m[6]) * d; M[7] = (m[1] * m[6] - m[0] * m[7]) * d; M[8] = (m[0] * m[4] - m[1] * m[3]) * d;
        } else memset(M, 0, sizeof(M));
    }
    return warp_impl(src, sstep, sw, sh, dst, dstep, dw, dh, type, M, 1, flags & 7, border, bv, NULL);
}

/* cv::remap (imgwarp.cpp:1762-1900) */
PORT_API int port_remap(const void* src, size_t sstep, int sw, int sh, int type, void* dst, size_t dstep, int dw, int dh,
                        const void* m1, size_t m1step, int m1type, const void* m2, size_t m2step, int m2type, int interp, int border, const double* bv)
{
    PortMaps mp = {m1, m1step, m1type, m2, m2step, m2type};
    static const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (interp & 32) return 1;
    return warp_impl(src, sstep, sw, sh, dst, dstep, dw, dh, type, I, 0, interp & 7, border, bv, &mp);
}

/* cv::pyrDown (pyramids.cpp:884-1039), default destination size.  8-bit exact; float in the order of the reference's SSE bodies
   (:324-341 rows, :497-516 columns; its edge columns and vector remainders use the scalar order: <= 1 ulp there) */
PORT_API int port_pyr_down(const void* src, size_t sstep, int sw, int sh, int type, void* dst, size_t dstep, int border)
{
    int depth = P_DEPTH(type), cn = P_CN(type), dw = (sw + 1) / 2, dh = (sh + 1) / 2;
    if (depth != P_8U && depth != P_32F) return 1;
    border &= ~16;
    for (int y = 0; y < dh; y++)
        for (int x = 0; x < dw; x++)
            for (int c = 0; c < cn; c++) {
                int sx[5];
                for (int k = 0; k < 5; k++) sx[k] = port_border(2 * x + k - 2, sw, border) * cn + c;
                if (depth == P_8U) {
                    int r[5];
                    for (int j = 0; j < 5; j++) {
                        const uchar* s = (const uchar*)src + (size_t)port_border(2 * y + j - 2, sh, border) * sstep;
                        r[j] = s[sx[2]] * 6 + (s[sx[1]] + s[sx[3]]) * 4 + s[sx[0]] + s[sx[4]];
                    }
                    ((uchar*)dst + (size_t)y * dstep)[x * cn + c] = (uchar)((r[2] * 6 + (r[1] + r[3]) * 4 + r[0] + r[4] + 128) >> 8);
                } else {
                    volatile float r[5], t, u;
                    for (int j = 0; j < 5; j++) {
                        const float* s = (const float*)((const char*)src + (size_t)port_border(2 * y + j - 2, sh, border) * sstep);
                        t = s[sx[1]] + s[sx[3]]; t = t * 4.f; u = s[sx[0]] + s[sx[4]]; t = t + u; u = s[sx[2]] * 6.f; r[j] = u + t;
                    }
                    t = r[1] + r[3]; t = t + r[2]; t = t * 4.f; u = r[0] + r[4]; { volatile float d2 = r[2] + r[2]; u = u + d2; } t = t + u;
                    ((float*)((char*)dst + (size_t)y * dstep))[x * cn + c] = t * (1.f / 256);
                }
            }
    return 0;
}

static float pyr_up_hf(const float* s, int dx, int c, int cn, int sw)
{
    int x = dx >> 1, odd = dx & 1;
    volatile float a, b;
    if (sw == 1) return s[c] * 8.f;
    if (x == 0) { if (odd) { a = s[c] + s[cn + c]; return a * 4.f; } a = s[c] * 6.f; b = s[cn + c] * 2.f; return a + b; }
    if (x == sw - 1) { if (odd) return s[x * cn + c] * 8.f; a = s[x * cn + c] * 7.f; return s[(x - 1) * cn + c] + a; }
    if (odd) { a = s[x * cn + c] + s[(x + 1) * cn + c]; return a * 4.f; }
    a = s[x * cn + c] * 6.f; b = s[(x - 1) * cn + c] + a; return b + s[(x + 1) * cn + c];
}
static int pyr_up_hi(const uchar* s, int dx, int c, int cn, int sw)
{
    int x = dx >> 1, odd = dx & 1;
    if (sw == 1) return s[c] * 8;
    if (x == 0) return odd ? (s[c] + s[cn + c]) * 4 : s[c] * 6 + s[cn + c] * 2;
    if (x == sw - 1) return odd ? s[x * cn + c] * 8 : s[(x - 1) * cn + c] + s[x * cn + c] * 7;
    return odd ? (s[x * cn + c] + s[(x + 1) * cn + c]) * 4 : s[(x - 1) * cn + c] + s[x * cn + c] * 6 + s[(x + 1) * cn + c];
}

/* cv::pyrUp (pyramids.cpp:1041-1155), 2W x 2H.  Rows of the ring: y-1 -> 1 at the top (REFLECT_101 on the doubled grid), y+1 -> H-1 at the bottom */
PORT_API int port_pyr_up(const void* src, size_t sstep, int sw, int sh, int type, void* dst, size_t dstep)
{
    int depth = P_DEPTH(type), cn = P_CN(type), dw = sw * 2, dh = sh * 2;
    if (depth != P_8U && depth != P_32F) return 1;
    for (int dy = 0; dy < dh; dy++) {
        int y = dy >> 1, y0 = y - 1 < 0 ? (sh > 1 ? 1 : 0) : y - 1, y2 = y + 1 >= sh ? sh - 1 : y + 1;
        for (int dx = 0; dx < dw; dx++)
            for (int c = 0; c < cn; c++) {
                if (depth == P_8U) {
                    const uchar* b = (const uchar*)src;
                    int r0 = pyr_up_hi(b + (size_t)y0 * sstep, dx, c, cn, sw), r1 = pyr_up_hi(b + (size_t)y * sstep, dx, c, cn, sw), r2 = pyr_up_hi(b + (size_t)y2 * sstep, dx, c, cn, sw);
                    ((uchar*)dst + (size_t)dy * dstep)[dx * cn + c] = (uchar)((dy & 1) ? ((r1 + r2) * 4 + 32) >> 6 : (r0 + r1 * 6 + r2 + 32) >> 6);
                } else {
                    const char* b = (const char*)src;
                    volatile float r0 = pyr_up_hf((const float*)(b + (size_t)y0 * sstep), dx, c, cn, sw), r1 = pyr_up_hf((const float*)(b + (size_t)y * sstep), dx, c, cn, sw),
                                   r2 = pyr_up_hf((const float*)(b + (size_t)y2 * sstep), dx, c, cn, sw), t;
                    if (dy & 1) { t = r1 + r2; t = (1.f / 16) * t; }
                    else { t = 6.f * r1; t = t + r0; t = t + r2; t = (1.f / 64) * t; }
                    ((float*)((char*)dst + (size_t)dy * dstep))[dx * cn + c] = t;
                }
            }
    }
    return 0;
}
