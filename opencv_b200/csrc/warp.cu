// warp.cu -- cv::warpAffine / cv::warpPerspective (INTER_NEAREST / LINEAR / CUBIC; 8-bit and float; 1/3/4 channels).
//
// One fused kernel per call (coordinate generation + gather + blend); the reference does the same per 64x64-ish block
// through cv::remap (WarpAffineInvoker imgwarp.cpp:2233-2298, WarpPerspectiveInvoker :3160-3226).
//
// Coordinates reproduce the reference's fixed-point pipeline exactly (explicit _rn fp64 intrinsics, no contraction):
//   affine       adelta=rint(M0*x*1024), bdelta=rint(M3*x*1024), X0=rint((M1*y+M2)*1024)+rd, Y0=rint((M4*y+M5)*1024)+rd,
//                rd = 512 (NEAREST) | 16 (others); NEAREST: (X0+adelta)>>10; others: X=(X0+adelta)>>5, sx=X>>5, fx=X&31
//                (hal::warpAffine :2673-2700, warpAffineBlockline[NN] :2702-2782)
//   perspective  block-relative fp64: x_b = x - x%bw0, X0=M0*x_b+M1*y+M2 (same for Y0,W0); W=W0+M6*x1; W = W ? 32/W : 0
//                (1/W for NEAREST); X=rint(clamp((X0+M0*x1)*W, INT_MIN, INT_MAX))  (:3199-3201, :3299-3365)
// Sampling follows remapNearest / remapBilinear / remapBicubic (:329-430, :675-904, :907-1010): 5-bit sub-pixel index into
// the 32x32 tap tables (initInterTab2D :213-287; built on the host with the same float code and uploaded once),
// u8: sat_u8((sum + 2^14) >> 15); f32: float sums in the reference's order; borders CONSTANT/REPLICATE/REFLECT/REFLECT_101/WRAP.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "common.cuh"
#include "host_tables.h"

namespace b200cv {

__device__ short g_bilin_i[1024 * 4];
__device__ float g_bilin_f[1024 * 4];
__device__ short g_bicub_i[1024 * 16];
__device__ float g_bicub_f[1024 * 16];
__device__ short g_lanc_i[1024 * 64];      // INTER_LANCZOS4: 8 x 8 taps per sub-pixel position (remapLanczos4, imgwarp.cpp:1012-1113)
__device__ float g_lanc_f[1024 * 64];

struct WarpParams {
    double M[9];
    float cval_f[4];
    int cval_i[4];
    int sw, sh, dw, dh;
    int border, persp, bw0;
};

enum { W_NN = 0, W_LIN = 1, W_CUB = 2, W_LAN = 3 };

template <typename T> struct TabOf;
template <> struct TabOf<uchar> { typedef short type; __device__ static const short* lin() { return g_bilin_i; } __device__ static const short* cub() { return g_bicub_i; } __device__ static const short* lan() { return g_lanc_i; } };
template <> struct TabOf<float> { typedef float type; __device__ static const float* lin() { return g_bilin_f; } __device__ static const float* cub() { return g_bicub_f; } __device__ static const float* lan() { return g_lanc_f; } };

__device__ __forceinline__ int clipi(int x, int a, int b) { return x >= a ? (x < b ? x : b - 1) : a; }

template <int INTERP>
__device__ __forceinline__ void warp_coords(const WarpParams& p, int x, int y, int& sx, int& sy, int& a)
{
    if (!p.persp) {
        const int rd = INTERP == W_NN ? 512 : 16;
        int adelta = __double2int_rn(__dmul_rn(__dmul_rn(p.M[0], (double)x), 1024.0));
        int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(p.M[3], (double)x), 1024.0));
        int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.M[1], (double)y), p.M[2]), 1024.0)) + rd;
        int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.M[4], (double)y), p.M[5]), 1024.0)) + rd;
        if (INTERP == W_NN) {
            sx = sat_s16((X0 + adelta) >> 10);
            sy = sat_s16((Y0 + bdelta) >> 10);
            a = 0;
        } else {
            int X = (X0 + adelta) >> 5, Y = (Y0 + bdelta) >> 5;
            sx = sat_s16(X >> 5);
            sy = sat_s16(Y >> 5);
            a = (Y & 31) * 32 + (X & 31);
        }
    } else {
        int xb = (x / p.bw0) * p.bw0, x1 = x - xb;
        double X0 = __dadd_rn(__dadd_rn(__dmul_rn(p.M[0], (double)xb), __dmul_rn(p.M[1], (double)y)), p.M[2]);
        double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(p.M[3], (double)xb), __dmul_rn(p.M[4], (double)y)), p.M[5]);
        double W0 = __dadd_rn(__dadd_rn(__dmul_rn(p.M[6], (double)xb), __dmul_rn(p.M[7], (double)y)), p.M[8]);
        double W = __dadd_rn(W0, __dmul_rn(p.M[6], (double)x1));
        W = W != 0.0 ? __ddiv_rn(INTERP == W_NN ? 1.0 : 32.0, W) : 0.0;
        double fX = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(__dadd_rn(X0, __dmul_rn(p.M[0], (double)x1)), W)));
        double fY = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(__dadd_rn(Y0, __dmul_rn(p.M[3], (double)x1)), W)));
        int X = __double2int_rn(fX), Y = __double2int_rn(fY);
        if (INTERP == W_NN) { sx = sat_s16(X); sy = sat_s16(Y); a = 0; }
        else { sx = sat_s16(X >> 5); sy = sat_s16(Y >> 5); a = (Y & 31) * 32 + (X & 31); }
    }
}

// one destination pixel gathered straight from global memory, all border modes.  Returns false when the pixel is to be left untouched
// (BORDER_TRANSPARENT: remapNearest imgwarp.cpp:373,408; remapBilinear :788-815 -- a point inside the image that lacks some of its four
// neighbours is blended from the ones that exist, re-normalised; remapBicubic :925,965-968 -- centre outside: untouched, else REFLECT_101 taps)
template <typename T, int CN, int INTERP>
__device__ __forceinline__ bool sample_direct(const Img& src, int f, const WarpParams& p, int sx, int sy, int a, T* d)
{
    const int sw = p.sw, sh = p.sh;
    const bool transparent = p.border == B200CV_BORDER_TRANSPARENT;
    const int border = (transparent && (INTERP == W_CUB || INTERP == W_LAN)) ? B200CV_BORDER_REFLECT_101 : p.border;
    T cval[4];
#pragma unroll
    for (int c = 0; c < 4; c++) { if constexpr (sizeof(T) == 1) cval[c] = (T)p.cval_i[c]; else cval[c] = p.cval_f[c]; }

    if constexpr (INTERP == W_NN) {
        const T* s;
        if ((unsigned)sx < (unsigned)sw && (unsigned)sy < (unsigned)sh) s = src.row<T>(f, sy) + (size_t)sx * CN;
        else if (transparent) return false;
        else if (border == B200CV_BORDER_REPLICATE) s = src.row<T>(f, clipi(sy, 0, sh)) + (size_t)clipi(sx, 0, sw) * CN;
        else if (border == B200CV_BORDER_CONSTANT) s = nullptr;
        else s = src.row<T>(f, border_interpolate(sy, sh, border)) + (size_t)border_interpolate(sx, sw, border) * CN;
#pragma unroll
        for (int c = 0; c < CN; c++) d[c] = s ? s[c] : cval[c];
        return true;
    } else if constexpr (INTERP == W_LIN) {
        typedef typename TabOf<T>::type AT;
        const AT* w = TabOf<T>::lin() + a * 4;
        if (border == B200CV_BORDER_CONSTANT && (sx >= sw || sx + 1 < 0 || sy >= sh || sy + 1 < 0)) {
#pragma unroll
            for (int c = 0; c < CN; c++) d[c] = cval[c];
            return true;
        }
        const bool inl = (unsigned)sx < (unsigned)max(sw - 1, 0) && (unsigned)sy < (unsigned)max(sh - 1, 0);
        if (transparent && !inl) {
            if (!(sx >= 0 && sx <= sw - 1 && sy >= 0 && sy <= sh - 1)) return false;
            const bool e1 = sx < sw - 1, e2 = sy < sh - 1;
            const T* S = src.row<T>(f, sy) + (size_t)sx * CN;
            const T* S1 = e2 ? src.row<T>(f, sy + 1) + (size_t)sx * CN : S;
            if constexpr (sizeof(T) == 1) {
                int w_tot = w[0]; if (e1) w_tot += w[1]; if (e2) w_tot += w[2]; if (e1 && e2) w_tot += w[3];
                if (w_tot == 0) return false;
                const int w_ini = (int)w[0] + w[1] + w[2] + w[3];
#pragma unroll
                for (int c = 0; c < CN; c++) {
                    int t0 = S[c] * w[0];
                    if (e1) t0 += S[c + CN] * w[1];
                    if (e2) t0 += S1[c] * w[2];
                    if (e1 && e2) t0 += S1[c + CN] * w[3];
                    t0 = (int)__fdiv_rn(__fmul_rn((float)t0, (float)w_ini), (float)w_tot);      // (WT)(t0 * (float)w_tot_ini / w_tot), WT = int: truncation
                    d[c] = sat_u8((t0 + (1 << 14)) >> 15);
                }
            } else {
                float w_tot = 0.f;
                w_tot = __fadd_rn(w_tot, w[0]); if (e1) w_tot = __fadd_rn(w_tot, w[1]); if (e2) w_tot = __fadd_rn(w_tot, w[2]); if (e1 && e2) w_tot = __fadd_rn(w_tot, w[3]);
                if (w_tot == 0.f) return false;
                const float w_ini = __fadd_rn(__fadd_rn(__fadd_rn(w[0], w[1]), w[2]), w[3]);
#pragma unroll
                for (int c = 0; c < CN; c++) {
                    float t0 = __fadd_rn(0.f, __fmul_rn(S[c], w[0]));
                    if (e1) t0 = __fadd_rn(t0, __fmul_rn(S[c + CN], w[1]));
                    if (e2) t0 = __fadd_rn(t0, __fmul_rn(S1[c], w[2]));
                    if (e1 && e2) t0 = __fadd_rn(t0, __fmul_rn(S1[c + CN], w[3]));
                    d[c] = __fdiv_rn(__fmul_rn(t0, w_ini), w_tot);
                }
            }
            return true;
        }
        int sx0, sx1, sy0, sy1;
        if (inl) { sx0 = sx; sx1 = sx + 1; sy0 = sy; sy1 = sy + 1; }
        else if (border == B200CV_BORDER_REPLICATE) { sx0 = clipi(sx, 0, sw); sx1 = clipi(sx + 1, 0, sw); sy0 = clipi(sy, 0, sh); sy1 = clipi(sy + 1, 0, sh); }
        else {
            sx0 = border_interpolate(sx, sw, border); sx1 = border_interpolate(sx + 1, sw, border);
            sy0 = border_interpolate(sy, sh, border); sy1 = border_interpolate(sy + 1, sh, border);
        }
        const T* r0 = sy0 >= 0 ? src.row<T>(f, sy0) : nullptr;
        const T* r1 = sy1 >= 0 ? src.row<T>(f, sy1) : nullptr;
#pragma unroll
        for (int c = 0; c < CN; c++) {
            T v0 = (r0 && sx0 >= 0) ? r0[sx0 * CN + c] : cval[c];
            T v1 = (r0 && sx1 >= 0) ? r0[sx1 * CN + c] : cval[c];
            T v2 = (r1 && sx0 >= 0) ? r1[sx0 * CN + c] : cval[c];
            T v3 = (r1 && sx1 >= 0) ? r1[sx1 * CN + c] : cval[c];
            if constexpr (sizeof(T) == 1) d[c] = sat_u8((v0 * w[0] + v1 * w[1] + v2 * w[2] + v3 * w[3] + (1 << 14)) >> 15);
            else d[c] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(v0, w[0]), __fmul_rn(v1, w[1])), __fmul_rn(v2, w[2])), __fmul_rn(v3, w[3]));
        }
        return true;
    } else {
        // INTER_CUBIC (4 x 4 taps, remapBicubic imgwarp.cpp:907-1010) and INTER_LANCZOS4 (8 x 8 taps, remapLanczos4 :1012-1113): the same structure
        typedef typename TabOf<T>::type AT;
        constexpr int NT = INTERP == W_CUB ? 4 : 8, OFS = NT / 2 - 1;
        const AT* w = (INTERP == W_CUB ? TabOf<T>::cub() : TabOf<T>::lan()) + a * (NT * NT);
        sx -= OFS; sy -= OFS;
        const bool inlier = (unsigned)sx < (unsigned)max(sw - (NT - 1), 0) && (unsigned)sy < (unsigned)max(sh - (NT - 1), 0);
        if (!inlier && transparent && ((unsigned)(sx + OFS) >= (unsigned)sw || (unsigned)(sy + OFS) >= (unsigned)sh)) return false;
        if (!inlier && border == B200CV_BORDER_CONSTANT && (sx >= sw || sx + NT <= 0 || sy >= sh || sy + NT <= 0)) {
#pragma unroll
            for (int c = 0; c < CN; c++) d[c] = cval[c];
            return true;
        }
        int xs[NT], ys[NT];
#pragma unroll
        for (int i = 0; i < NT; i++) {
            xs[i] = inlier ? sx + i : border_interpolate(sx + i, sw, border);
            ys[i] = inlier ? sy + i : border_interpolate(sy + i, sh, border);
        }
#pragma unroll
        for (int c = 0; c < CN; c++) {
            if constexpr (sizeof(T) == 1) {
                int sum = 0;
#pragma unroll
                for (int i = 0; i < NT; i++) {
                    const uchar* r = ys[i] >= 0 ? src.row<uchar>(f, ys[i]) : nullptr;
#pragma unroll
                    for (int j = 0; j < NT; j++) {
                        int v = (r && xs[j] >= 0) ? r[xs[j] * CN + c] : cval[c];
                        sum += v * w[i * NT + j];
                    }
                }
                d[c] = sat_u8((sum + (1 << 14)) >> 15);
            } else {
                if (inlier) {
                    // rows left to right; cubic: sum = row0, then += row_i; lanczos: sum = 0, then += row_i for every row
                    float sum = 0.f;
#pragma unroll
                    for (int i = 0; i < NT; i++) {
                        const float* r = src.row<float>(f, ys[i]) + (size_t)xs[0] * CN + c;
                        float rs = __fmul_rn(r[0], w[i * NT]);
#pragma unroll
                        for (int j = 1; j < NT; j++) rs = __fadd_rn(rs, __fmul_rn(r[j * CN], w[i * NT + j]));
                        sum = (i == 0 && INTERP == W_CUB) ? rs : __fadd_rn(sum, rs);
                    }
                    d[c] = sum;
                } else {
                    float cv = cval[c], sum = cv;
#pragma unroll
                    for (int i = 0; i < NT; i++) {
                        if (ys[i] < 0) continue;
                        const float* r = src.row<float>(f, ys[i]);
#pragma unroll
                        for (int j = 0; j < NT; j++)
                            if (xs[j] >= 0) sum = __fadd_rn(sum, __fmul_rn(__fsub_rn(r[xs[j] * CN + c], cv), w[i * NT + j]));
                    }
                    d[c] = sum;
                }
            }
        }
    }
    return true;
}

template <typename T, int CN, int INTERP>
__global__ void __launch_bounds__(256) warp_kernel(Img src, Img dst, const __grid_constant__ WarpParams p)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x >= p.dw) return;
    int sx, sy, a;
    warp_coords<INTERP>(p, x, y, sx, sy, a);
    T v[4];
    if (sample_direct<T, CN, INTERP>(src, f, p, sx, sy, a, v)) {        // false: BORDER_TRANSPARENT leaves the destination pixel as it is
        T* d = dst.row<T>(f, y) + (size_t)x * CN;
#pragma unroll
        for (int c = 0; c < CN; c++) d[c] = v[c];
    }
}


// ---- 8-bit sampling from the staged footprint with word loads -----------------------------------------------------------------
// A tap row is TAPS*CN consecutive bytes at an arbitrary byte address: read the aligned words that cover it, realign with funnel
// shifts, gather the TAPS bytes of one channel into a word with PRMT (all selectors are compile-time) and let IDP2A multiply them by
// the 16-bit table weights: dp2a.lo(a = two s16 weights, b = bytes 0,1).  Exact 32-bit integer sums, as remapBilinear /
// remapBicubic compute them (imgwarp.cpp:675-904, :907-1010).
__device__ __forceinline__ int dp2a_lo_su(int a, unsigned b, int c)
{
    int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}
// (tap j0, tap j0+1) of channel c as bytes 0,1 of a word: bytes c + j0*CN and c + (j0+1)*CN of the 16-byte string in w[0..3].
// One PRMT: its two source words are the ones holding the two bytes (positions are compile-time after unrolling).
template <int CN> __device__ __forceinline__ unsigned tap_pair(const unsigned* w, int c, int j0)
{
    const int p0 = c + j0 * CN, p1 = p0 + CN;
    return __byte_perm(w[p0 >> 2], w[p1 >> 2], (unsigned)((p0 & 3) | ((4 + (p1 & 3)) << 4)));
}

// ---- tiled kernel: the source footprint of a 64x16 destination tile is staged in shared memory ---------------------------
// The footprint is the bounding box of the tile's four corner coordinates (exact for the affine fixed-point map, which is
// monotone in x and in y; for a projective map every pixel re-checks containment and falls back to the direct gather).
// Staging is coalesced 16-byte traffic and applies the border rule once per staged element, so the gather itself is
// branch-free shared-memory reads: the global-memory gather costs one L1 wavefront per touched line per tap, this costs one
// per warp per tap.
constexpr int WT_W = 64, WT_H = 16;
constexpr int WT_SMEM_MAX = 96 * 1024;

template <typename T, int CN, int INTERP>
__global__ void __launch_bounds__(256) warp_tile_kernel(Img src, Img dst, const __grid_constant__ WarpParams p, int smem_cap)
{
    extern __shared__ __align__(16) unsigned char s_src[];
    __shared__ int s_box[4];
    __shared__ int s_ad[WT_W], s_bd[WT_W], s_X0[WT_H], s_Y0[WT_H];     // affine: the reference's adelta/bdelta and per-row X0/Y0 tables
    constexpr int ES = CN * (int)sizeof(T);                  // bytes per pixel
    constexpr int K0 = INTERP == W_CUB ? -1 : 0, K1 = INTERP == W_NN ? 0 : INTERP == W_LIN ? 1 : 2;
    const int f = blockIdx.z, x0 = blockIdx.x * WT_W, y0 = blockIdx.y * WT_H;
    const int tid = threadIdx.x;
    if (tid < 32) {
        const int cx = (tid & 1) ? min(x0 + WT_W, p.dw) - 1 : x0, cy = (tid & 2) ? min(y0 + WT_H, p.dh) - 1 : y0;
        int sx, sy, a;
        warp_coords<INTERP>(p, cx, cy, sx, sy, a);
        int mnx = sx, mxx = sx, mny = sy, mxy = sy;
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            mnx = min(mnx, __shfl_xor_sync(0xffffffffu, mnx, o)); mxx = max(mxx, __shfl_xor_sync(0xffffffffu, mxx, o));
            mny = min(mny, __shfl_xor_sync(0xffffffffu, mny, o)); mxy = max(mxy, __shfl_xor_sync(0xffffffffu, mxy, o));
        }
        if (tid == 0) { s_box[0] = (mnx + K0) & ~15; s_box[1] = mny + K0; s_box[2] = mxx + K1; s_box[3] = mxy + K1; }
    } else if (!p.persp) {
        // fp64 once per tile column / row instead of once per pixel (hal::warpAffine builds the same tables on the host, imgwarp.cpp:2673-2700)
        const int t = tid - 32;
        if (t < WT_W) {
            const double x = (double)(x0 + t);
            s_ad[t] = __double2int_rn(__dmul_rn(__dmul_rn(p.M[0], x), 1024.0));
            s_bd[t] = __double2int_rn(__dmul_rn(__dmul_rn(p.M[3], x), 1024.0));
        } else if (t < WT_W + WT_H) {
            const double y = (double)(y0 + t - WT_W);
            const int rd = INTERP == W_NN ? 512 : 16;
            s_X0[t - WT_W] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.M[1], y), p.M[2]), 1024.0)) + rd;
            s_Y0[t - WT_W] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.M[4], y), p.M[5]), 1024.0)) + rd;
        }
    }
    __syncthreads();
    const int bx0 = s_box[0], by0 = s_box[1];
    const int bw = (s_box[2] - bx0 + 16) & ~15, bh = s_box[3] - by0 + 1;        // staged pixels per row (multiple of 16), rows
    int nvec = bw * ES / 16;                                                    // 16-byte vectors per staged row
    const int pitch = (nvec | 1) * 16;                                          // odd number of vectors: rows start on different banks
    const bool staged = (long long)pitch * bh <= smem_cap;
    const int sw = p.sw, sh = p.sh, border = p.border;

    if (staged) {
        // one warp per staged row (row-uniform work hoisted), lanes over its 16-byte vectors
        const bool aligned = (((uintptr_t)src.data | src.step | src.fstep) & 15) == 0;
        const int gb0 = bx0 * ES;                                               // byte offset of the staged row start inside a source row
        const int row_bytes = sw * ES;
        // tiles that look outside the image (a rotation about the centre leaves ~20 % of the destination there): whole vectors of border value
        bool cfill = border == B200CV_BORDER_CONSTANT;
        unsigned cword;
        if constexpr (sizeof(T) == 1) { cfill = cfill && p.cval_i[0] == p.cval_i[1] && p.cval_i[1] == p.cval_i[2] && p.cval_i[2] == p.cval_i[3]; cword = (unsigned)(p.cval_i[0] & 255) * 0x01010101u; }
        else { cfill = cfill && p.cval_f[0] == p.cval_f[1] && p.cval_f[1] == p.cval_f[2] && p.cval_f[2] == p.cval_f[3]; cword = __float_as_uint(p.cval_f[0]); }
        for (int r = tid >> 5; r < bh; r += 8) {
            int sy = by0 + r;
            if ((unsigned)sy >= (unsigned)sh) sy = border == B200CV_BORDER_REPLICATE ? clipi(sy, 0, sh) : border_interpolate(sy, sh, border);
            const unsigned char* srow = sy >= 0 ? (const unsigned char*)src.row<T>(f, sy) : nullptr;
            unsigned char* drow = s_src + r * pitch;
            for (int j = tid & 31; j < nvec; j += 32) {
                const int gb = gb0 + j * 16;                                    // first byte of this vector within the source row
                uint4 val;
                if (srow && aligned && gb >= 0 && gb + 16 <= row_bytes) {
                    val = *(const uint4*)(srow + gb);
                } else if (cfill && (!srow || gb + 16 <= 0 || gb >= row_bytes)) {
                    val = make_uint4(cword, cword, cword, cword);        // wholly outside the image under BORDER_CONSTANT with one value for all channels
                } else {
                    T e[16 / sizeof(T)];
#pragma unroll
                    for (int i = 0; i < (int)(16 / sizeof(T)); i++) {
                        const int ge = gb / (int)sizeof(T) + i;                 // element index in the row (may be negative; gb is a multiple of 16)
                        const int px = ge >= 0 ? ge / CN : -((-ge + CN - 1) / CN);
                        const int c = ge - px * CN;
                        int sx = px;
                        if ((unsigned)sx >= (unsigned)sw) sx = border == B200CV_BORDER_REPLICATE ? clipi(sx, 0, sw) : border_interpolate(sx, sw, border);
                        if (srow && sx >= 0) e[i] = ((const T*)srow)[sx * CN + c];
                        else { if constexpr (sizeof(T) == 1) e[i] = (T)p.cval_i[c]; else e[i] = p.cval_f[c]; }
                    }
                    val = *(const uint4*)e;
                }
                *(uint4*)(drow + j * 16) = val;
            }
        }
    }
    __syncthreads();

    const int x = x0 + (tid & (WT_W - 1));
    if (x >= p.dw) return;
#pragma unroll 1
    for (int yy = tid / WT_W; yy < WT_H; yy += 256 / WT_W) {
        const int y = y0 + yy;
        if (y >= p.dh) break;
        int sx, sy, a;
        if (p.persp) warp_coords<INTERP>(p, x, y, sx, sy, a);
        else {
            const int XX = s_X0[yy] + s_ad[tid & (WT_W - 1)], YY = s_Y0[yy] + s_bd[tid & (WT_W - 1)];
            if (INTERP == W_NN) { sx = sat_s16(XX >> 10); sy = sat_s16(YY >> 10); a = 0; }
            else { sx = sat_s16(XX >> 10); sy = sat_s16(YY >> 10); a = ((YY >> 5) & 31) * 32 + ((XX >> 5) & 31); }
        }
        T* d = dst.row<T>(f, y) + (size_t)x * CN;
        const int lx = sx + K0 - bx0, ly = sy + K0 - by0;            // first tap, staged coordinates
        if (!staged || lx < 0 || ly < 0 || lx + (K1 - K0) >= bw || ly + (K1 - K0) >= bh) {
            sample_direct<T, CN, INTERP>(src, f, p, sx, sy, a, d);
            continue;
        }
        const T* s = (const T*)(s_src + ly * pitch) + lx * CN;
        const int rp = pitch / (int)sizeof(T);                       // row pitch in elements
        if constexpr (INTERP == W_NN) {
#pragma unroll
            for (int c = 0; c < CN; c++) d[c] = s[c];
        } else if constexpr (INTERP == W_LIN) {
            if constexpr (sizeof(T) == 1) {
                const int2 w = *(const int2*)(g_bilin_i + a * 4);              // (w0, w1), (w2, w3) as s16 pairs
                const unsigned A = (unsigned)(ly * pitch + lx * CN), sh8 = 8 * (A & 3);
                constexpr int NW = (2 * CN + 3) / 4;                           // words that hold one realigned tap row
                unsigned r0[4], r1[4];
                const unsigned* q0 = (const unsigned*)(s_src + (A & ~3u));
                const unsigned* q1 = (const unsigned*)(s_src + (A & ~3u) + pitch);
#pragma unroll
                for (int i = 0; i < NW; i++) { r0[i] = __funnelshift_r(q0[i], q0[i + 1], sh8); r1[i] = __funnelshift_r(q1[i], q1[i + 1], sh8); }
#pragma unroll
                for (int c = 0; c < CN; c++) {
                    int sum = dp2a_lo_su(w.x, tap_pair<CN>(r0, c, 0), 1 << 14);
                    sum = dp2a_lo_su(w.y, tap_pair<CN>(r1, c, 0), sum);
                    d[c] = sat_u8(sum >> 15);
                }
            } else {
                const float4 w = *(const float4*)(g_bilin_f + a * 4);
#pragma unroll
                for (int c = 0; c < CN; c++)
                    d[c] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s[c], w.x), __fmul_rn(s[CN + c], w.y)), __fmul_rn(s[rp + c], w.z)),
                                     __fmul_rn(s[rp + CN + c], w.w));
            }
        } else {
            if constexpr (sizeof(T) == 1) {
                int w[8];                                                        // 16 s16 weights: row i = (w[2i], w[2i+1])
                *(uint4*)w = *(const uint4*)(g_bicub_i + a * 16);
                *(uint4*)(w + 4) = *(const uint4*)(g_bicub_i + a * 16 + 8);
                const unsigned A = (unsigned)(ly * pitch + lx * CN), sh8 = 8 * (A & 3);
                constexpr int NW = (4 * CN + 3) / 4;
                int sum[CN];
#pragma unroll
                for (int c = 0; c < CN; c++) sum[c] = 1 << 14;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const unsigned* q = (const unsigned*)(s_src + (A & ~3u) + i * pitch);
                    unsigned r[4];
#pragma unroll
                    for (int k = 0; k < NW; k++) r[k] = __funnelshift_r(q[k], q[k + 1], sh8);
#pragma unroll
                    for (int c = 0; c < CN; c++) {
                        sum[c] = dp2a_lo_su(w[2 * i + 1], tap_pair<CN>(r, c, 2), dp2a_lo_su(w[2 * i], tap_pair<CN>(r, c, 0), sum[c]));
                    }
                }
#pragma unroll
                for (int c = 0; c < CN; c++) d[c] = sat_u8(sum[c] >> 15);
            } else {
                float w[16];
#pragma unroll
                for (int i = 0; i < 4; i++) *(float4*)(w + 4 * i) = *(const float4*)(g_bicub_f + a * 16 + 4 * i);
                // the reference uses two different summation orders (remapBicubic, imgwarp.cpp:944-1003)
                const bool inlier = (unsigned)(sx - 1) < (unsigned)max(sw - 3, 0) && (unsigned)(sy - 1) < (unsigned)max(sh - 3, 0);
#pragma unroll
                for (int c = 0; c < CN; c++) {
                    if (inlier) {
                        float sum = 0.f;
#pragma unroll
                        for (int i = 0; i < 4; i++) {
                            const float* r = s + i * rp + c;
                            float rs = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], w[i * 4]), __fmul_rn(r[CN], w[i * 4 + 1])),
                                                           __fmul_rn(r[2 * CN], w[i * 4 + 2])), __fmul_rn(r[3 * CN], w[i * 4 + 3]));
                            sum = i == 0 ? rs : __fadd_rn(sum, rs);
                        }
                        d[c] = sum;
                    } else {
                        sample_direct<T, CN, INTERP>(src, f, p, sx, sy, a, d);   // border pixels: the skip-outside-taps formula
                        break;
                    }
                }
            }
        }
    }
}

// ---- 8-bit LINEAR / CUBIC, second version of the tiled kernel -------------------------------------------------------------------------------
// Same staging and the same sampling arithmetic as warp_tile_kernel; what changes is how the work is cut (the first
// version was instruction-issue bound, most of its instructions not sampling):
//   * tile 128 x 32 instead of 64 x 16: the per-thread fixed costs (corner coordinates, tables, staged-row pointers and border tests) are
//     spread over 16 pixels per thread instead of 4; the footprint of an 8UC3 tile is still only ~25 KB
//   * a thread produces 4 consecutive pixels of a row: their bytes leave as CN aligned 32-bit stores (12 bytes of an 8UC3 row per thread, a
//     warp writes 384 contiguous bytes) instead of 4 CN byte stores
//   * projective maps: X0, Y0, W0 = M * (x_block, y, 1) are per (row, 64-column block) values (the reference evaluates them once per block
//     line, imgwarp.cpp:3182-3206): built once per tile in shared memory; per pixel remain the divide and two multiply-adds in fp64
constexpr int WQ_W = 128, WQ_H = 32, WQ_NB = 4;      // WQ_NB: 64-column blocks a tile row can touch (+1 for maps with other block widths)

template <int CN, int INTERP>
__device__ __forceinline__ void sample_staged_u8(const unsigned char* s_src, int pitch, int lx, int ly, int a, unsigned char* d)
{
    if constexpr (INTERP == W_LIN) {
        const int2 w = __ldg((const int2*)(g_bilin_i + a * 4));           // (w0, w1), (w2, w3) as s16 pairs
        const unsigned A = (unsigned)(ly * pitch + lx * CN), sh8 = 8 * (A & 3);
        constexpr int NW = (2 * CN + 3) / 4;                              // words that hold one realigned tap row
        unsigned r0[4], r1[4];
        const unsigned* q0 = (const unsigned*)(s_src + (A & ~3u));
        const unsigned* q1 = (const unsigned*)(s_src + (A & ~3u) + pitch);
#pragma unroll
        for (int i = 0; i < NW; i++) { r0[i] = __funnelshift_r(q0[i], q0[i + 1], sh8); r1[i] = __funnelshift_r(q1[i], q1[i + 1], sh8); }
#pragma unroll
        for (int c = 0; c < CN; c++) {
            int sum = dp2a_lo_su(w.x, tap_pair<CN>(r0, c, 0), 1 << 14);
            sum = dp2a_lo_su(w.y, tap_pair<CN>(r1, c, 0), sum);
            d[c] = (unsigned char)(sum >> 15);           // bilinear table weights are >= 0 and add up to 2^15 (initInterTab2D): the blend of bytes is a byte
        }
    } else {
        int w[8];                                                          // 16 s16 weights: row i = (w[2i], w[2i+1])
        *(uint4*)w = __ldg((const uint4*)(g_bicub_i + a * 16));
        *(uint4*)(w + 4) = __ldg((const uint4*)(g_bicub_i + a * 16 + 8));
        const unsigned A = (unsigned)(ly * pitch + lx * CN), sh8 = 8 * (A & 3);
        constexpr int NW = (4 * CN + 3) / 4;
        int sum[CN];
#pragma unroll
        for (int c = 0; c < CN; c++) sum[c] = 1 << 14;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const unsigned* q = (const unsigned*)(s_src + (A & ~3u) + i * pitch);
            unsigned r[4];
#pragma unroll
            for (int k = 0; k < NW; k++) r[k] = __funnelshift_r(q[k], q[k + 1], sh8);
#pragma unroll
            for (int c = 0; c < CN; c++) sum[c] = dp2a_lo_su(w[2 * i + 1], tap_pair<CN>(r, c, 2), dp2a_lo_su(w[2 * i], tap_pair<CN>(r, c, 0), sum[c]));
        }
#pragma unroll
        for (int c = 0; c < CN; c++) d[c] = sat_u8(sum[c] >> 15);
    }
}

template <int CN, int INTERP>
__global__ void __launch_bounds__(256) warp_tile4_kernel(Img src, Img dst, const __grid_constant__ WarpParams p, int smem_cap)
{
    typedef unsigned char T;
    extern __shared__ __align__(16) unsigned char s_src[];
    __shared__ int s_box[4];
    __shared__ __align__(16) int s_ad[WQ_W], s_bd[WQ_W];
    __shared__ int s_X0[WQ_H], s_Y0[WQ_H];                               // affine: the reference's adelta / bdelta and per-row X0 / Y0 tables
    __shared__ double s_pX[WQ_H][WQ_NB], s_pY[WQ_H][WQ_NB], s_pW[WQ_H][WQ_NB];   // projective: M * (x_block, y, 1) per row and column block
    constexpr int ES = CN;
    constexpr int K0 = INTERP == W_CUB ? -1 : 0, K1 = INTERP == W_LIN ? 1 : 2;
    const int f = blockIdx.z, x0 = blockIdx.x * WQ_W, y0 = blockIdx.y * WQ_H;
    const int tid = threadIdx.x;
    const int blk0 = x0 / p.bw0;
    if (tid < 32) {
        const int cx = (tid & 1) ? min(x0 + WQ_W, p.dw) - 1 : x0, cy = (tid & 2) ? min(y0 + WQ_H, p.dh) - 1 : y0;
        int sx, sy, a;
        warp_coords<INTERP>(p, cx, cy, sx, sy, a);
        int mnx = sx, mxx = sx, mny = sy, mxy = sy;
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            mnx = min(mnx, __shfl_xor_sync(0xffffffffu, mnx, o)); mxx = max(mxx, __shfl_xor_sync(0xffffffffu, mxx, o));
            mny = min(mny, __shfl_xor_sync(0xffffffffu, mny, o)); mxy = max(mxy, __shfl_xor_sync(0xffffffffu, mxy, o));
        }
        if (tid == 0) { s_box[0] = (mnx + K0) & ~15; s_box[1] = mny + K0; s_box[2] = mxx + K1; s_box[3] = mxy + K1; }
    } else if (!p.persp) {
        // fp64 once per tile column / row instead of once per pixel (hal::warpAffine builds the same tables on the host, imgwarp.cpp:2673-2700)
        const int t = tid - 32;
        if (t < WQ_W) {
            const double x = (double)(x0 + t);
            s_ad[t] = __double2int_rn(__dmul_rn(__dmul_rn(p.M[0], x), 1024.0));
            s_bd[t] = __double2int_rn(__dmul_rn(__dmul_rn(p.M[3], x), 1024.0));
        } else if (t < WQ_W + WQ_H) {
            const double y = (double)(y0 + t - WQ_W);
            s_X0[t - WQ_W] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.M[1], y), p.M[2]), 1024.0)) + 16;
            s_Y0[t - WQ_W] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.M[4], y), p.M[5]), 1024.0)) + 16;
        }
    } else {
        const int t = tid - 32;
        if (t < WQ_H * WQ_NB) {
            const int yy = t / WQ_NB, b = t - yy * WQ_NB;
            const double xb = (double)((blk0 + b) * p.bw0), y = (double)(y0 + yy);
            s_pX[yy][b] = __dadd_rn(__dadd_rn(__dmul_rn(p.M[0], xb), __dmul_rn(p.M[1], y)), p.M[2]);
            s_pY[yy][b] = __dadd_rn(__dadd_rn(__dmul_rn(p.M[3], xb), __dmul_rn(p.M[4], y)), p.M[5]);
            s_pW[yy][b] = __dadd_rn(__dadd_rn(__dmul_rn(p.M[6], xb), __dmul_rn(p.M[7], y)), p.M[8]);
        }
    }
    __syncthreads();
    const int bx0 = s_box[0], by0 = s_box[1];
    const int bw = (s_box[2] - bx0 + 16) & ~15, bh = s_box[3] - by0 + 1;        // staged pixels per row (multiple of 16), rows
    const int nvec = bw * ES / 16;                                              // 16-byte vectors per staged row
    const int pitch = (nvec | 1) * 16;                                          // odd number of vectors: rows start on different banks
    const bool staged = (long long)pitch * bh <= smem_cap;
    const int sw = p.sw, sh = p.sh, border = p.border;

    if (staged) {
        // one warp per staged row (row-uniform work hoisted), lanes over its 16-byte vectors
        const bool aligned = (((uintptr_t)src.data | src.step | src.fstep) & 15) == 0;
        const int gb0 = bx0 * ES;                                               // byte offset of the staged row start inside a source row
        const int row_bytes = sw * ES;
        const bool cfill = border == B200CV_BORDER_CONSTANT && p.cval_i[0] == p.cval_i[1] && p.cval_i[1] == p.cval_i[2] && p.cval_i[2] == p.cval_i[3];
        const unsigned cword = (unsigned)(p.cval_i[0] & 255) * 0x01010101u;
        for (int r = tid >> 5; r < bh; r += 8) {
            int sy = by0 + r;
            if ((unsigned)sy >= (unsigned)sh) sy = border == B200CV_BORDER_REPLICATE ? clipi(sy, 0, sh) : border_interpolate(sy, sh, border);
            const unsigned char* srow = sy >= 0 ? (const unsigned char*)src.row<T>(f, sy) : nullptr;
            unsigned char* drow = s_src + r * pitch;
            for (int j = tid & 31; j < nvec; j += 32) {
                const int gb = gb0 + j * 16;                                    // first byte of this vector within the source row
                uint4 val;
                if (srow && aligned && gb >= 0 && gb + 16 <= row_bytes) {
                    val = *(const uint4*)(srow + gb);
                } else if (cfill && (!srow || gb + 16 <= 0 || gb >= row_bytes)) {
                    val = make_uint4(cword, cword, cword, cword);
                } else {
                    T e[16];
#pragma unroll
                    for (int i = 0; i < 16; i++) {
                        const int ge = gb + i;                                  // element index in the row (may be negative; gb is a multiple of 16)
                        const int px = ge >= 0 ? ge / CN : -((-ge + CN - 1) / CN);
                        const int c = ge - px * CN;
                        int sx = px;
                        if ((unsigned)sx >= (unsigned)sw) sx = border == B200CV_BORDER_REPLICATE ? clipi(sx, 0, sw) : border_interpolate(sx, sw, border);
                        e[i] = (srow && sx >= 0) ? srow[sx * CN + c] : (T)p.cval_i[c];
                    }
                    val = *(const uint4*)e;
                }
                *(uint4*)(drow + j * 16) = val;
            }
        }
    }
    __syncthreads();

    const bool dvec = (((uintptr_t)dst.data | dst.step | dst.fstep) & 3) == 0;
#pragma unroll 1
    for (int g = tid; g < (WQ_W / 4) * WQ_H; g += 256) {
        const int yy = g / (WQ_W / 4), xq = (g - yy * (WQ_W / 4)) * 4;
        const int y = y0 + yy, x = x0 + xq;
        if (y >= p.dh || x >= p.dw) continue;
        int4 ad = make_int4(0, 0, 0, 0), bd = ad;
        int X0r = 0, Y0r = 0;
        if (!p.persp) { ad = *(const int4*)(s_ad + xq); bd = *(const int4*)(s_bd + xq); X0r = s_X0[yy]; Y0r = s_Y0[yy]; }
        const int adv[4] = {ad.x, ad.y, ad.z, ad.w}, bdv[4] = {bd.x, bd.y, bd.z, bd.w};
        unsigned char ob[4 * CN];
        int pb = 0, px1 = 0;                                   // projective: column block (relative to the tile's first) and offset inside it
        if (p.persp) { pb = x / p.bw0 - blk0; px1 = x - (blk0 + pb) * p.bw0; }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int sx, sy, a;
            if (p.persp) {
                const int b = pb, x1 = px1;
                if (++px1 == p.bw0) { px1 = 0; pb++; }
                double W = __dadd_rn(s_pW[yy][b], __dmul_rn(p.M[6], (double)x1));
                W = W != 0.0 ? __ddiv_rn(32.0, W) : 0.0;
                const double fX = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(__dadd_rn(s_pX[yy][b], __dmul_rn(p.M[0], (double)x1)), W)));
                const double fY = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(__dadd_rn(s_pY[yy][b], __dmul_rn(p.M[3], (double)x1)), W)));
                const int X = __double2int_rn(fX), Y = __double2int_rn(fY);
                sx = sat_s16(X >> 5); sy = sat_s16(Y >> 5); a = (Y & 31) * 32 + (X & 31);
            } else {
                const int XX = X0r + adv[k], YY = Y0r + bdv[k];
                sx = sat_s16(XX >> 10); sy = sat_s16(YY >> 10); a = ((YY >> 5) & 31) * 32 + ((XX >> 5) & 31);
            }
            const int lx = sx + K0 - bx0, ly = sy + K0 - by0;            // first tap, staged coordinates
            unsigned char px[4] = {0, 0, 0, 0};
            if (x + k < p.dw) {
                if (!staged || lx < 0 || ly < 0 || lx + (K1 - K0) >= bw || ly + (K1 - K0) >= bh) sample_direct<T, CN, INTERP>(src, f, p, sx, sy, a, px);
                else sample_staged_u8<CN, INTERP>(s_src, pitch, lx, ly, a, px);
            }
#pragma unroll
            for (int c = 0; c < CN; c++) ob[k * CN + c] = px[c];
        }
        unsigned char* dp = dst.row<T>(f, y) + (size_t)x * CN;
        if (dvec && x + 4 <= p.dw) {
#pragma unroll
            for (int i = 0; i < CN; i++)
                ((unsigned*)dp)[i] = (unsigned)ob[4 * i] | ((unsigned)ob[4 * i + 1] << 8) | ((unsigned)ob[4 * i + 2] << 16) | ((unsigned)ob[4 * i + 3] << 24);
        } else {
            const int n = min(4, p.dw - x);
            for (int i = 0; i < n * CN; i++) dp[i] = ob[i];
        }
    }
}

// ---- NEAREST, 8-bit: the coordinate tables of warp_tile4_kernel without the staging pass ---------------------------------------------------
// The direct kernel evaluates the fp64 coordinate pipeline per pixel per pixel: here the affine adelta / bdelta / X0 / Y0 tables and the projective per-(row, column block)
// terms are built once per 128 x 32 tile, a thread gathers 4 consecutive pixels and stores them as CN 32-bit words.
template <int CN>
__global__ void __launch_bounds__(256) warp_nn4_kernel(Img src, Img dst, const __grid_constant__ WarpParams p)
{
    typedef unsigned char T;
    __shared__ __align__(16) int s_ad[WQ_W], s_bd[WQ_W];
    __shared__ int s_X0[WQ_H], s_Y0[WQ_H];
    __shared__ double s_pX[WQ_H][WQ_NB], s_pY[WQ_H][WQ_NB], s_pW[WQ_H][WQ_NB];
    const int f = blockIdx.z, x0 = blockIdx.x * WQ_W, y0 = blockIdx.y * WQ_H;
    const int tid = threadIdx.x;
    const int blk0 = x0 / p.bw0;
    if (!p.persp) {
        if (tid < WQ_W) {
            const double x = (double)(x0 + tid);
            s_ad[tid] = __double2int_rn(__dmul_rn(__dmul_rn(p.M[0], x), 1024.0));
            s_bd[tid] = __double2int_rn(__dmul_rn(__dmul_rn(p.M[3], x), 1024.0));
        } else if (tid < WQ_W + WQ_H) {
            const double y = (double)(y0 + tid - WQ_W);
            s_X0[tid - WQ_W] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.M[1], y), p.M[2]), 1024.0)) + 512;
            s_Y0[tid - WQ_W] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.M[4], y), p.M[5]), 1024.0)) + 512;
        }
    } else if (tid < WQ_H * WQ_NB) {
        const int yy = tid / WQ_NB, b = tid - yy * WQ_NB;
        const double xb = (double)((blk0 + b) * p.bw0), y = (double)(y0 + yy);
        s_pX[yy][b] = __dadd_rn(__dadd_rn(__dmul_rn(p.M[0], xb), __dmul_rn(p.M[1], y)), p.M[2]);
        s_pY[yy][b] = __dadd_rn(__dadd_rn(__dmul_rn(p.M[3], xb), __dmul_rn(p.M[4], y)), p.M[5]);
        s_pW[yy][b] = __dadd_rn(__dadd_rn(__dmul_rn(p.M[6], xb), __dmul_rn(p.M[7], y)), p.M[8]);
    }
    __syncthreads();
    const bool dvec = (((uintptr_t)dst.data | dst.step | dst.fstep) & 3) == 0;
#pragma unroll 1
    for (int g = tid; g < (WQ_W / 4) * WQ_H; g += 256) {
        const int yy = g / (WQ_W / 4), xq = (g - yy * (WQ_W / 4)) * 4;
        const int y = y0 + yy, x = x0 + xq;
        if (y >= p.dh || x >= p.dw) continue;
        int4 ad = make_int4(0, 0, 0, 0), bd = ad;
        int X0r = 0, Y0r = 0;
        if (!p.persp) { ad = *(const int4*)(s_ad + xq); bd = *(const int4*)(s_bd + xq); X0r = s_X0[yy]; Y0r = s_Y0[yy]; }
        const int adv[4] = {ad.x, ad.y, ad.z, ad.w}, bdv[4] = {bd.x, bd.y, bd.z, bd.w};
        int pb = 0, px1 = 0;
        if (p.persp) { pb = x / p.bw0 - blk0; px1 = x - (blk0 + pb) * p.bw0; }
        unsigned char ob[4 * CN];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int sx, sy;
            if (p.persp) {
                const int b = pb, x1 = px1;
                if (++px1 == p.bw0) { px1 = 0; pb++; }
                double W = __dadd_rn(s_pW[yy][b], __dmul_rn(p.M[6], (double)x1));
                W = W != 0.0 ? __ddiv_rn(1.0, W) : 0.0;
                const double fX = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(__dadd_rn(s_pX[yy][b], __dmul_rn(p.M[0], (double)x1)), W)));
                const double fY = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(__dadd_rn(s_pY[yy][b], __dmul_rn(p.M[3], (double)x1)), W)));
                sx = sat_s16(__double2int_rn(fX)); sy = sat_s16(__double2int_rn(fY));
            } else {
                sx = sat_s16((X0r + adv[k]) >> 10); sy = sat_s16((Y0r + bdv[k]) >> 10);
            }
            unsigned char px[4] = {0, 0, 0, 0};
            if (x + k < p.dw) sample_direct<T, CN, W_NN>(src, f, p, sx, sy, 0, px);
#pragma unroll
            for (int c = 0; c < CN; c++) ob[k * CN + c] = px[c];
        }
        unsigned char* dp = dst.row<T>(f, y) + (size_t)x * CN;
        if (dvec && x + 4 <= p.dw) {
#pragma unroll
            for (int i = 0; i < CN; i++)
                ((unsigned*)dp)[i] = (unsigned)ob[4 * i] | ((unsigned)ob[4 * i + 1] << 8) | ((unsigned)ob[4 * i + 2] << 16) | ((unsigned)ob[4 * i + 3] << 24);
        } else {
            const int n = min(4, p.dw - x);
            for (int i = 0; i < n * CN; i++) dp[i] = ob[i];
        }
    }
}

static int ensure_warp_tables()
{
    static PerDeviceFlag done_pd; bool& done = done_pd.cur();
    if (done) return B200CV_OK;
    std::vector<float> f; std::vector<short> q;
    bilinear_tab(f, q);
    B200_CUDA(cudaMemcpyToSymbol(g_bilin_f, f.data(), f.size() * sizeof(float)));
    B200_CUDA(cudaMemcpyToSymbol(g_bilin_i, q.data(), q.size() * sizeof(short)));
    bicubic_tab(f, q);
    B200_CUDA(cudaMemcpyToSymbol(g_bicub_f, f.data(), f.size() * sizeof(float)));
    B200_CUDA(cudaMemcpyToSymbol(g_bicub_i, q.data(), q.size() * sizeof(short)));
    lanczos4_tab(f, q);
    B200_CUDA(cudaMemcpyToSymbol(g_lanc_f, f.data(), f.size() * sizeof(float)));
    B200_CUDA(cudaMemcpyToSymbol(g_lanc_i, q.data(), q.size() * sizeof(short)));
    done = true;
    return B200CV_OK;
}

// host estimate of the staged footprint (bytes) of one 64x16 tile whose first pixel is (x0, y0); < 0: do not stage
static long long tile_footprint(const WarpParams& p, int x0, int y0, int es, int taps, int TW = WT_W, int TH = WT_H)
{
    double mnx = 1e300, mxx = -1e300, mny = 1e300, mxy = -1e300;
    for (int k = 0; k < 4; k++) {
        double x = (k & 1) ? std::min(x0 + TW, p.dw) - 1 : x0, y = (k & 2) ? std::min(y0 + TH, p.dh) - 1 : y0;
        double X = p.M[0] * x + p.M[1] * y + p.M[2], Y = p.M[3] * x + p.M[4] * y + p.M[5], W = p.persp ? p.M[6] * x + p.M[7] * y + p.M[8] : 1.0;
        if (!(fabs(W) > 1e-12)) return -1;
        X /= W; Y /= W;
        if (!(fabs(X) < 1e6 && fabs(Y) < 1e6)) return -1;
        mnx = std::min(mnx, X); mxx = std::max(mxx, X); mny = std::min(mny, Y); mxy = std::max(mxy, Y);
    }
    long long bw = ((long long)(mxx - mnx) + taps + 3 + 15 + 15) & ~15LL, bh = (long long)(mxy - mny) + taps + 3;
    long long nvec = bw * es / 16;
    return (nvec | 1) * 16 * bh;
}

template <typename T, int CN, int INTERP>
static int launch_warp_i(const Img& s, const Img& d, const WarpParams& p, cudaStream_t st)
{
    if constexpr (INTERP == W_LAN) {          // 8 x 8 taps: the direct gather (no staged variant)
        dim3 grid(div_up((unsigned)p.dw, 256), (unsigned)p.dh, (unsigned)s.frames);
        warp_kernel<T, CN, INTERP><<<grid, 256, 0, st>>>(s, d, p);
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    } else {
    const int es = CN * (int)sizeof(T), taps = INTERP == W_NN ? 1 : INTERP == W_LIN ? 2 : 4;
    // shared memory to request: the largest footprint over a coarse sample of tiles (an affine map has the same footprint everywhere)
    long long need = 0;
    const int tx = (int)div_up((unsigned)p.dw, WT_W), ty = (int)div_up((unsigned)p.dh, WT_H);
    const int nsx = p.persp ? std::min(tx, 9) : 1, nsy = p.persp ? std::min(ty, 9) : 1;
    for (int j = 0; j < nsy && need >= 0; j++)
        for (int i = 0; i < nsx; i++) {
            int bx = nsx > 1 ? (int)((long long)i * (tx - 1) / (nsx - 1)) : 0, by = nsy > 1 ? (int)((long long)j * (ty - 1) / (nsy - 1)) : 0;
            long long fp = tile_footprint(p, bx * WT_W, by * WT_H, es, taps);
            if (fp < 0) { need = -1; break; }
            need = std::max(need, fp);
        }
    const char* path = getenv("B200CV_WARP_PATH");
    if constexpr (sizeof(T) == 1 && INTERP == W_NN) {
        // 8-bit NEAREST: table-driven coordinates, 4 pixels per thread (BORDER_TRANSPARENT needs the per-pixel keep decision: direct kernel)
        const bool blocks_ok = !p.persp || (p.bw0 > 0 && (WQ_W + p.bw0 - 1) / p.bw0 + 1 <= WQ_NB);
        if (blocks_ok && p.border != B200CV_BORDER_TRANSPARENT && !(path && !strcmp(path, "direct"))) {
            dim3 grid(div_up((unsigned)p.dw, WQ_W), div_up((unsigned)p.dh, WQ_H), (unsigned)s.frames);
            warp_nn4_kernel<CN><<<grid, 256, 0, st>>>(s, d, p);
            B200_LAUNCH_CHECK();
            return B200CV_OK;
        }
    }
    // one tap per pixel (NEAREST) does not repay the staging pass
    // BORDER_TRANSPARENT: per-pixel keep / blend decisions, the direct kernel only
    if (INTERP == W_NN || need < 0 || need > WT_SMEM_MAX || p.border == B200CV_BORDER_TRANSPARENT || (path && !strcmp(path, "direct"))) {          // heavy minification / degenerate map: direct gather
        dim3 grid(div_up((unsigned)p.dw, 256), (unsigned)p.dh, (unsigned)s.frames);
        warp_kernel<T, CN, INTERP><<<grid, 256, 0, st>>>(s, d, p);
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }
    if constexpr (sizeof(T) == 1 && INTERP != W_NN) {
        // 8-bit LINEAR / CUBIC: the 128 x 32 tile kernel when its footprint fits and a tile row touches at most WQ_NB column blocks
        const int qx = (int)div_up((unsigned)p.dw, WQ_W), qy = (int)div_up((unsigned)p.dh, WQ_H);
        long long need4 = 0;
        const int msx = p.persp ? std::min(qx, 9) : 1, msy = p.persp ? std::min(qy, 9) : 1;
        for (int j = 0; j < msy && need4 >= 0; j++)
            for (int i = 0; i < msx; i++) {
                int bx = msx > 1 ? (int)((long long)i * (qx - 1) / (msx - 1)) : 0, by = msy > 1 ? (int)((long long)j * (qy - 1) / (msy - 1)) : 0;
                long long fp = tile_footprint(p, bx * WQ_W, by * WQ_H, es, taps, WQ_W, WQ_H);
                if (fp < 0) { need4 = -1; break; }
                need4 = std::max(need4, fp);
            }
        const bool blocks_ok = !p.persp || (p.bw0 > 0 && (WQ_W + p.bw0 - 1) / p.bw0 + 1 <= WQ_NB);
        if (need4 > 0 && need4 <= WT_SMEM_MAX && blocks_ok && !(path && !strcmp(path, "tile64"))) {
            int smem4 = (int)std::min<long long>(WT_SMEM_MAX, std::max<long long>(need4 + need4 / 8, 8 * 1024));
            auto kern4 = warp_tile4_kernel<CN, INTERP>;
            static PerDeviceFlag attr4_pd; bool& attr4 = attr4_pd.cur();
            if (!attr4) { B200_CUDA(cudaFuncSetAttribute(kern4, cudaFuncAttributeMaxDynamicSharedMemorySize, WT_SMEM_MAX)); attr4 = true; }
            kern4<<<dim3((unsigned)qx, (unsigned)qy, (unsigned)s.frames), 256, smem4, st>>>(s, d, p, smem4);
            B200_LAUNCH_CHECK();
            return B200CV_OK;
        }
    }
    int smem = (int)std::min<long long>(WT_SMEM_MAX, std::max<long long>(need + need / 8, 8 * 1024));
    auto kern = warp_tile_kernel<T, CN, INTERP>;
    static PerDeviceFlag attr_pd; bool& attr = attr_pd.cur();
    if (!attr) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, WT_SMEM_MAX)); attr = true; }
    dim3 grid((unsigned)tx, (unsigned)ty, (unsigned)s.frames);
    kern<<<grid, 256, smem, st>>>(s, d, p, smem);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
    }
}

template <typename T, int CN>
static int launch_warp(int interp, const Img& s, const Img& d, const WarpParams& p, cudaStream_t st)
{
    if (interp == W_NN) return launch_warp_i<T, CN, W_NN>(s, d, p, st);
    if (interp == W_LIN) return launch_warp_i<T, CN, W_LIN>(s, d, p, st);
    if (interp == W_LAN) return launch_warp_i<T, CN, W_LAN>(s, d, p, st);
    return launch_warp_i<T, CN, W_CUB>(s, d, p, st);
}


// ---- cv::remap: coordinates come from maps instead of a matrix; sampling is the warps' (RemapInvoker, imgwarp.cpp:1096-1330) -----------
enum { MAP_PLANAR_F32 = 0, MAP_PACKED_F32 = 1, MAP_FIXED = 2 };

// cvRound / v_round on x86: round-to-nearest-even, the "integer indefinite" 0x80000000 for NaN and values outside int32
__device__ __forceinline__ int x86_round(float v) { return fabsf(v) < 2147483648.f ? __float2int_rn(v) : (int)0x80000000; }

template <typename T, int CN, int INTERP>
__global__ void __launch_bounds__(256) remap_kernel(Img src, Img dst, Img m1, Img m2, const __grid_constant__ WarpParams p, int kind)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x >= p.dw) return;
    int sx, sy, a = 0;
    if (kind == MAP_FIXED) {
        const short* xy = m1.row<short>(0, y) + 2 * x;
        const int fr = m2.data ? (m2.row<unsigned short>(0, y)[x] & 1023) : 0;
        if (INTERP == W_NN && m2.data) {       // NNDeltaTab_i as the reference fills it: +1 where the 5-bit fraction is BELOW 1/2 (:237-238, :1176-1181)
            sx = (short)(xy[0] + ((fr & 31) < 16)); sy = (short)(xy[1] + ((fr >> 5) < 16));
        } else { sx = xy[0]; sy = xy[1]; a = fr; }      // NEAREST without a fraction map: the coordinates as they are (:1166)
    } else {
        float mx, my;
        if (kind == MAP_PLANAR_F32) { mx = m1.row<float>(0, y)[x]; my = m2.row<float>(0, y)[x]; }
        else { const float2 q = ((const float2*)m1.row<float>(0, y))[x]; mx = q.x; my = q.y; }
        if (INTERP == W_NN) { sx = sat_s16(x86_round(mx)); sy = sat_s16(x86_round(my)); }       // saturate_cast<short>(float), :1195-1216
        else {                                                                                   // :1253-1283
            const int ix = x86_round(__fmul_rn(mx, 32.f)), iy = x86_round(__fmul_rn(my, 32.f));
            sx = sat_s16(ix >> 5); sy = sat_s16(iy >> 5);
            a = (iy & 31) * 32 + (ix & 31);
        }
    }
    T v[4];
    if (sample_direct<T, CN, INTERP>(src, f, p, sx, sy, a, v)) {
        T* d = dst.row<T>(f, y) + (size_t)x * CN;
#pragma unroll
        for (int c = 0; c < CN; c++) d[c] = v[c];
    }
}

template <typename T, int CN>
static int launch_remap(int interp, const Img& s, const Img& d, const Img& m1, const Img& m2, const WarpParams& p, int kind, cudaStream_t st)
{
    dim3 grid(div_up((unsigned)p.dw, 256), (unsigned)p.dh, (unsigned)s.frames);
    if (interp == W_NN) remap_kernel<T, CN, W_NN><<<grid, 256, 0, st>>>(s, d, m1, m2, p, kind);
    else if (interp == W_LIN) remap_kernel<T, CN, W_LIN><<<grid, 256, 0, st>>>(s, d, m1, m2, p, kind);
    else if (interp == W_LAN) remap_kernel<T, CN, W_LAN><<<grid, 256, 0, st>>>(s, d, m1, m2, p, kind);
    else remap_kernel<T, CN, W_CUB><<<grid, 256, 0, st>>>(s, d, m1, m2, p, kind);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

static int warp_common(const b200cvMat* src, const b200cvMat* dst, const double* Minv, int persp, int flags, int border,
                       const double* bv, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->type == dst->type, "warp: dst type must equal src type");
    B200_REQUIRE(src->data != dst->data, "warp: in-place is not supported");
    const int depth = B200CV_DEPTH(src->type), cn = B200CV_CN(src->type);
    if ((depth != B200CV_8U && depth != B200CV_32F) || (cn != 1 && cn != 3 && cn != 4)) return B200CV_NOT_IMPLEMENTED;
    int interp = flags & 7;
    if (interp == B200CV_INTER_AREA) interp = B200CV_INTER_LINEAR;            // imgwarp.cpp:2816, :3393
    if (interp > B200CV_INTER_CUBIC && interp != B200CV_INTER_LANCZOS4) return B200CV_NOT_IMPLEMENTED;
    if (interp == B200CV_INTER_LANCZOS4) interp = W_LAN;
    border &= ~B200CV_BORDER_ISOLATED;
    if (border < 0 || border > B200CV_BORDER_TRANSPARENT) return B200CV_NOT_IMPLEMENTED;
    if (src->cols >= 32767 || src->rows >= 32767 || dst->rows >= 65536) return B200CV_NOT_IMPLEMENTED;   // CV_Assert(cols,rows < SHRT_MAX) imgwarp.cpp:1813
    if ((rc = ensure_warp_tables())) return rc;
    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    WarpParams p;
    for (int i = 0; i < 9; i++) p.M[i] = Minv[i];
    for (int c = 0; c < 4; c++) {
        double v = bv ? bv[c] : 0.0;
        long r = lrint(v);
        p.cval_i[c] = (int)(r < 0 ? 0 : r > 255 ? 255 : r);
        p.cval_f[c] = (float)v;
    }
    p.sw = src->cols; p.sh = src->rows; p.dw = dst->cols; p.dh = dst->rows; p.border = border; p.persp = persp;
    {   // WarpPerspectiveInvoker block width (imgwarp.cpp:3182-3184)
        int bh0 = p.dh < 16 ? p.dh : 16;
        int bw0 = 1024 / bh0; if (bw0 > p.dw) bw0 = p.dw;
        p.bw0 = bw0;
    }
    cudaStream_t st = as_stream(stream);
    if (depth == B200CV_8U) {
        if (cn == 1) return launch_warp<uchar, 1>(interp, s, d, p, st);
        if (cn == 3) return launch_warp<uchar, 3>(interp, s, d, p, st);
        return launch_warp<uchar, 4>(interp, s, d, p, st);
    }
    if (cn == 1) return launch_warp<float, 1>(interp, s, d, p, st);
    if (cn == 3) return launch_warp<float, 3>(interp, s, d, p, st);
    return launch_warp<float, 4>(interp, s, d, p, st);
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_warp_affine(const b200cvMat* src, const b200cvMat* dst, const double* M0, int flags, int border,
                                  const double* border_value, void* stream)
{
    B200_REQUIRE(M0, "null matrix");
    double M[9] = {M0[0], M0[1], M0[2], M0[3], M0[4], M0[5], 0, 0, 1};
    if (!(flags & B200CV_WARP_INVERSE_MAP)) {      // cv::warpAffine, imgwarp.cpp:2824-2834
        double D = M[0] * M[4] - M[1] * M[3];
        D = D != 0 ? 1. / D : 0;
        double A11 = M[4] * D, A22 = M[0] * D;
        M[0] = A11; M[1] *= -D;
        M[3] *= -D; M[4] = A22;
        double b1 = -M[0] * M[2] - M[1] * M[5];
        double b2 = -M[3] * M[2] - M[4] * M[5];
        M[2] = b1; M[5] = b2;
    }
    return warp_common(src, dst, M, 0, flags, border, border_value, stream);
}

extern "C" int b200cv_warp_perspective(const b200cvMat* src, const b200cvMat* dst, const double* M0, int flags, int border,
                                       const double* border_value, void* stream)
{
    B200_REQUIRE(M0, "null matrix");
    double M[9];
    for (int i = 0; i < 9; i++) M[i] = M0[i];
    if (!(flags & B200CV_WARP_INVERSE_MAP)) {      // cv::invert of a 3x3 CV_64F matrix: adjugate / determinant (core/src/lapack.cpp:944-970)
        const double* m = M0;
        double det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
        if (det != 0.) {
            double d = 1. / det;
            M[0] = (m[4] * m[8] - m[5] * m[7]) * d; M[1] = (m[2] * m[7] - m[1] * m[8]) * d; M[2] = (m[1] * m[5] - m[2] * m[4]) * d;
            M[3] = (m[5] * m[6] - m[3] * m[8]) * d; M[4] = (m[0] * m[8] - m[2] * m[6]) * d; M[5] = (m[2] * m[3] - m[0] * m[5]) * d;
            M[6] = (m[3] * m[7] - m[4] * m[6]) * d; M[7] = (m[1] * m[6] - m[0] * m[7]) * d; M[8] = (m[0] * m[4] - m[1] * m[3]) * d;
        } else {
            for (int i = 0; i < 9; i++) M[i] = 0;   // cv::invert leaves dst = 0 for a singular matrix
        }
    }
    return warp_common(src, dst, M, 1, flags, border, border_value, stream);
}

extern "C" int b200cv_remap(const b200cvMat* src, const b200cvMat* dst, const b200cvMat* map1, const b200cvMat* map2, int interpolation,
                            int border, const double* bv, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst")) || (rc = check_mat(map1, "map1"))) return rc;
    if (map2 && map2->data && (rc = check_mat(map2, "map2"))) return rc;
    B200_REQUIRE(src->type == dst->type, "remap: dst type must equal src type");
    B200_REQUIRE(src->data != dst->data, "remap: in-place is not supported");
    B200_REQUIRE(dst->cols == map1->cols && dst->rows == map1->rows, "remap: dst must have the size of the maps");
    if (interpolation & B200CV_WARP_RELATIVE_MAP) return B200CV_NOT_IMPLEMENTED;
    const bool has2 = map2 && map2->data;
    if (has2) B200_REQUIRE(map2->cols == map1->cols && map2->rows == map1->rows, "remap: map sizes differ");
    int kind;
    const int t1 = map1->type, t2 = has2 ? map2->type : -1;
    if (t1 == B200CV_MAKETYPE(B200CV_32F, 1) && t2 == B200CV_MAKETYPE(B200CV_32F, 1)) kind = MAP_PLANAR_F32;
    else if (t1 == B200CV_MAKETYPE(B200CV_32F, 2) && !has2) kind = MAP_PACKED_F32;
    else if (t1 == B200CV_MAKETYPE(B200CV_16S, 2) && (t2 == B200CV_MAKETYPE(B200CV_16U, 1) || t2 == B200CV_MAKETYPE(B200CV_16S, 1) || !has2)) kind = MAP_FIXED;
    else return B200CV_NOT_IMPLEMENTED;
    const int depth = B200CV_DEPTH(src->type), cn = B200CV_CN(src->type);
    if ((depth != B200CV_8U && depth != B200CV_32F) || (cn != 1 && cn != 3 && cn != 4)) return B200CV_NOT_IMPLEMENTED;
    int interp = interpolation & 7;
    if (interp == B200CV_INTER_AREA) interp = B200CV_INTER_LINEAR;            // imgwarp.cpp:1826
    if (interp > B200CV_INTER_CUBIC && interp != B200CV_INTER_LANCZOS4) return B200CV_NOT_IMPLEMENTED;
    if (interp == B200CV_INTER_LANCZOS4) interp = W_LAN;
    if (kind == MAP_FIXED && !has2 && interp != B200CV_INTER_NEAREST) return B200CV_ERR_BAD_ARG;
    border &= ~B200CV_BORDER_ISOLATED;
    if (border < 0 || border > B200CV_BORDER_TRANSPARENT) return B200CV_NOT_IMPLEMENTED;
    if (src->cols >= 32767 || src->rows >= 32767 || dst->cols >= 32767 || dst->rows >= 32767) return B200CV_NOT_IMPLEMENTED;   // CV_Assert(... < SHRT_MAX), :1810
    if ((rc = ensure_warp_tables())) return rc;
    Img s = make_img(src), d = make_img(dst), m1 = make_img(map1), m2;
    memset(&m2, 0, sizeof(m2));
    if (has2) m2 = make_img(map2);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    WarpParams p;
    memset(&p, 0, sizeof(p));
    for (int c = 0; c < 4; c++) {
        double v = bv ? bv[c] : 0.0;
        long r = lrint(v);
        p.cval_i[c] = (int)(r < 0 ? 0 : r > 255 ? 255 : r);
        p.cval_f[c] = (float)v;
    }
    p.sw = src->cols; p.sh = src->rows; p.dw = dst->cols; p.dh = dst->rows; p.border = border; p.bw0 = 1;
    cudaStream_t st = as_stream(stream);
    if (depth == B200CV_8U) {
        if (cn == 1) return launch_remap<uchar, 1>(interp, s, d, m1, m2, p, kind, st);
        if (cn == 3) return launch_remap<uchar, 3>(interp, s, d, m1, m2, p, kind, st);
        return launch_remap<uchar, 4>(interp, s, d, m1, m2, p, kind, st);
    }
    if (cn == 1) return launch_remap<float, 1>(interp, s, d, m1, m2, p, kind, st);
    if (cn == 3) return launch_remap<float, 3>(interp, s, d, m1, m2, p, kind, st);
    return launch_remap<float, 4>(interp, s, d, m1, m2, p, kind, st);
}
