/* port_distance.c -- plain-C restatement of cv::distanceTransform(src, dst, distanceType, maskSize, dstType) for 8UC1 sources
 * (imgproc/src/distransform.cpp, built with IPP off).  TEST INFRASTRUCTURE ONLY.
 *
 *   chamfer   3x3 / 5x5 masks in 16.16 fixed point: a forward raster pass (left / upper neighbours, clamped at DIST_MAX) and a
 *             backward pass (right / lower neighbours, only where the value exceeds the horizontal weight); (float)t * 2^-16
 *   precise   column pass (squared distance to the nearest zero in the column, as a float of the unsigned square) and the lower
 *             envelope of parabolas along each row, with the reference's float operations in its order
 *   8-bit L1  saturating city-block scans: forward from the left and upper neighbours, backward from the right and lower ones
 *
 * port_distance_transform has the signature of ref_distance_transform (tests/cpp/dist_ref_shim.cpp): it returns the destination depth
 * it wrote (0 = 8U, 5 = 32F) or -1 where the reference refuses the arguments.
 */
#include <limits.h>
#include "port_common.h"

enum { D_USER = -1, D_L1 = 1, D_L2 = 2, D_C = 3 };
#define SQ_LIMIT 65536

/* ---- chamfer ----------------------------------------------------------------------------------------------------------------------- */
typedef struct { unsigned* t; int w, h; unsigned dmax; } Grid;

static inline unsigned g_at(const Grid* g, int y, int x)
{
    return (y < 0 || y >= g->h || x < 0 || x >= g->w) ? g->dmax : g->t[(size_t)y * g->w + x];
}

static inline unsigned umin(unsigned a, unsigned b) { return a < b ? a : b; }

/* weights hv, dg (and lg for the 5x5 mask, 0 otherwise); fills t with the backward pass's values */
static void chamfer(const uchar* src, size_t sstep, int w, int h, unsigned hv, unsigned dg, unsigned lg, int five, Grid* g)
{
    g->w = w; g->h = h;
    g->dmax = UINT_MAX - (five ? lg : dg);
    g->t = (unsigned*)malloc((size_t)w * h * sizeof(unsigned));
    for (int y = 0; y < h; y++) {
        const uchar* s = src + (size_t)y * sstep;
        for (int x = 0; x < w; x++) {
            unsigned v = 0;
            if (s[x]) {
                v = umin(g_at(g, y - 1, x - 1) + dg, g_at(g, y - 1, x) + hv);
                v = umin(v, g_at(g, y - 1, x + 1) + dg);
                v = umin(v, g_at(g, y, x - 1) + hv);
                if (five) {
                    v = umin(v, g_at(g, y - 2, x - 1) + lg);
                    v = umin(v, g_at(g, y - 2, x + 1) + lg);
                    v = umin(v, g_at(g, y - 1, x - 2) + lg);
                    v = umin(v, g_at(g, y - 1, x + 2) + lg);
                }
                if (v > g->dmax) v = g->dmax;
            }
            g->t[(size_t)y * w + x] = v;
        }
    }
    for (int y = h - 1; y >= 0; y--) {
        for (int x = w - 1; x >= 0; x--) {
            unsigned v = g->t[(size_t)y * w + x];
            if (v > hv) {
                v = umin(v, g_at(g, y + 1, x + 1) + dg);
                v = umin(v, g_at(g, y + 1, x) + hv);
                v = umin(v, g_at(g, y + 1, x - 1) + dg);
                v = umin(v, g_at(g, y, x + 1) + hv);
                if (five) {
                    v = umin(v, g_at(g, y + 2, x + 1) + lg);
                    v = umin(v, g_at(g, y + 2, x - 1) + lg);
                    v = umin(v, g_at(g, y + 1, x + 2) + lg);
                    v = umin(v, g_at(g, y + 1, x - 2) + lg);
                }
            }
            g->t[(size_t)y * w + x] = v;
        }
    }
}

static unsigned fix16(float m) { return (unsigned)lrintf(m * 65536.f); }

/* ---- precise ----------------------------------------------------------------------------------------------------------------------- */
static inline unsigned sq_of(long i, long limit) { return (i < limit && i < SQ_LIMIT) ? (unsigned)i * (unsigned)i : UINT_MAX; }

static void column_pass(const uchar* src, size_t sstep, float* dst, size_t dstep, int w, int h)
{
    int* below = (int*)malloc((size_t)h * sizeof(int));
    for (int x = 0; x < w; x++) {
        int d = h - 1;                 /* no zero below: h - 1 + the rows to the bottom, >= h */
        for (int y = h - 1; y >= 0; y--) {
            d = src[(size_t)y * sstep + x] ? d + 1 : 0;
            below[y] = d;
        }
        d = h - 1;
        for (int y = 0; y < h; y++) {
            d = d + 1 < below[y] ? d + 1 : below[y];
            *(float*)((char*)dst + (size_t)y * dstep + (size_t)x * 4) = (float)sq_of(d, h);
        }
    }
    free(below);
}

typedef struct { int* v; float* z; float* f; } Env;

/* the lower envelope of row f[0..n-1]; returns the index of its last parabola */
static int envelope(const float* f, int n, Env* e)
{
    const float inf = 1e15f;
    int k = 0;
    e->v[0] = 0; e->z[0] = -inf; e->z[1] = inf;
    for (int q = 1; q < n; q++) {
        for (;; k--) {
            const int p = e->v[k];
            const float inv = (float)(0.5 / (q - p));
            float parab;
            if (q < SQ_LIMIT) parab = (float)((unsigned)q * (unsigned)q - (unsigned)p * (unsigned)p);
            else parab = (float)(q + p) * (float)(q - p);
            const float diff = f[q] - f[p];
            const float num = diff + parab;
            const float s = num * inv;
            if (s > e->z[k]) {
                k++;
                e->v[k] = q; e->z[k] = s; e->z[k + 1] = inf;
                break;
            }
        }
    }
    return k;
}

static float envelope_value(const float* f, int n, const Env* e, int k, int q)
{
    const int p = e->v[k];
    const int a = q > p ? q - p : p - q;
    return sqrtf((float)sq_of(a, n) + f[p]);
}

static void row_pass(float* dst, size_t dstep, int w, int h)
{
    float* f = (float*)malloc((size_t)w * sizeof(float));
    Env e = {(int*)malloc((size_t)w * sizeof(int)), (float*)malloc((size_t)(w + 1) * sizeof(float)), NULL};
    for (int y = 0; y < h; y++) {
        float* d = (float*)((char*)dst + (size_t)y * dstep);
        memcpy(f, d, (size_t)w * sizeof(float));
        envelope(f, w, &e);
        int k = 0;
        for (int q = 0; q < w; q++) {
            while (e.z[k + 1] < (float)q) k++;
            d[q] = envelope_value(f, w, &e, k, q);
        }
    }
    free(f); free(e.v); free(e.z);
}

/* ---- 8-bit L1 ---------------------------------------------------------------------------------------------------------------------- */
static inline uchar sat_next(int a) { return (uchar)(a >= 255 ? 255 : a + 1); }

static void l1_u8(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h)
{
    /* forward: a non-zero pixel is one more than the smaller of its left and upper neighbours (255 outside the image), saturated */
    for (int y = 0; y < h; y++) {
        const uchar* s = src + (size_t)y * sstep;
        uchar* d = dst + (size_t)y * dstep;
        const uchar* up = y > 0 ? d - dstep : NULL;
        for (int x = 0; x < w; x++) {
            const int left = x > 0 ? d[x - 1] : 255, above = up ? up[x] : 255;
            d[x] = s[x] ? sat_next(left < above ? left : above) : 0;
        }
    }
    /* backward: the same from the right and lower neighbours, kept only where smaller */
    for (int y = h - 1; y >= 0; y--) {
        uchar* d = dst + (size_t)y * dstep;
        const uchar* down = y < h - 1 ? d + dstep : NULL;
        for (int x = w - 1; x >= 0; x--) {
            const int right = x < w - 1 ? d[x + 1] : 255, below = down ? down[x] : 255;
            const uchar c = sat_next(right < below ? right : below);
            if (c < d[x]) d[x] = c;
        }
    }
}

/* ---- entry points ------------------------------------------------------------------------------------------------------------------ */
PORT_API int port_distance_transform(const uchar* src, size_t sstep, void* dst, size_t dstep, int w, int h, int dist_type, int mask_size,
                                     int dst_type)
{
    if (dist_type == D_L1 && dst_type == P_8U) {
        /* in place allowed: the scans read each source byte before they write it */
        if ((const void*)src != dst) {
            for (int y = 0; y < h; y++) memcpy((uchar*)dst + (size_t)y * dstep, src + (size_t)y * sstep, (size_t)w);
        }
        uchar* d = (uchar*)dst;
        uchar* copy = (uchar*)malloc((size_t)w * h);
        for (int y = 0; y < h; y++) memcpy(copy + (size_t)y * w, d + (size_t)y * dstep, (size_t)w);
        l1_u8(copy, (size_t)w, d, dstep, w, h);
        free(copy);
        return P_8U;
    }
    if (mask_size != 0 && mask_size != 3 && mask_size != 5) return -1;
    if (dist_type == D_C || dist_type == D_L1) mask_size = 3;
    if (mask_size == 0) {
        column_pass(src, sstep, (float*)dst, dstep, w, h);
        row_pass((float*)dst, dstep, w, h);
        return P_32F;
    }
    if (dist_type != D_C && dist_type != D_L1 && dist_type != D_L2) return -1;
    float m[3];
    if (dist_type == D_C) { m[0] = 1.f; m[1] = 1.f; m[2] = 2.f; }
    else if (dist_type == D_L1) { m[0] = 1.f; m[1] = 2.f; m[2] = 3.f; }
    else if (mask_size == 3) { m[0] = 0.955f; m[1] = 1.3693f; m[2] = 0.f; }
    else { m[0] = 1.f; m[1] = 1.4f; m[2] = 2.1969f; }
    Grid g;
    chamfer(src, sstep, w, h, fix16(m[0]), fix16(m[1]), mask_size == 5 ? fix16(m[2]) : 0u, mask_size == 5, &g);
    for (int y = 0; y < h; y++) {
        float* d = (float*)((char*)dst + (size_t)y * dstep);
        for (int x = 0; x < w; x++) d[x] = (float)g.t[(size_t)y * w + x] * (1.f / 65536.f);
    }
    free(g.t);
    return P_32F;
}

/* the 8-bit L1 call as the L1 3x3 chamfer (weights 1, 2) with the epilogue min(t >> 16, 255): the device's route, which
 * tests/test_dist_reference.py holds to the saturating scans above */
PORT_API int port_dist_l1_u8_chamfer(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h)
{
    Grid g;
    chamfer(src, sstep, w, h, 65536u, 131072u, 0u, 0, &g);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const unsigned t = g.t[(size_t)y * w + x] >> 16;
            dst[(size_t)y * dstep + x] = (uchar)(t < 255 ? t : 255);
        }
    free(g.t);
    return 0;
}

/* the precise transform's lookup two ways on every row: the linear walk `while (z[k+1] < q) k++` and the binary search for the
 * smallest k with z[k+1] >= q the device uses.  Returns the number of (row, column) where they pick different parabolas, or -1 where
 * z does not increase strictly along a stack. */
PORT_API long port_dist_lookup_mismatches(const uchar* src, size_t sstep, int w, int h)
{
    float* plane = (float*)malloc((size_t)w * h * sizeof(float));
    column_pass(src, sstep, plane, (size_t)w * 4, w, h);
    Env e = {(int*)malloc((size_t)w * sizeof(int)), (float*)malloc((size_t)(w + 1) * sizeof(float)), NULL};
    long bad = 0;
    for (int y = 0; y < h && bad >= 0; y++) {
        const float* f = plane + (size_t)y * w;
        const int K = envelope(f, w, &e);
        for (int k = 0; k <= K; k++)
            if (!(e.z[k] < e.z[k + 1])) { bad = -1; break; }
        int k = 0;
        for (int q = 0; q < w && bad >= 0; q++) {
            while (e.z[k + 1] < (float)q) k++;
            int lo = 0, hi = K;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (e.z[mid + 1] < (float)q) lo = mid + 1; else hi = mid;
            }
            bad += lo != k;
        }
    }
    free(plane); free(e.v); free(e.z);
    return bad;
}
