// resize.cu -- cv::resize: INTER_NEAREST, INTER_LINEAR (incl. the exact-1/2 case the reference rewrites to
// INTER_AREA), INTER_AREA with an exact 2x2 box, INTER_CUBIC; 8-bit and float, 1/3/4 channels.
//
// Everything the reference tabulates on the host (source offsets and fixed-point / float taps per destination
// column and row, resize.cpp:4097-4190) is recomputed per thread here with the same IEEE operations in the same
// order (explicit _rn intrinsics: no FMA contraction), so no tables travel through HBM:
//   NEAREST   sx = min(floor(x * (1/fx)), sw-1) in fp64                               (resizeNN, resize.cpp:1121-1172)
//   LINEAR    fx = (float)((dx+0.5)*scale - 0.5); sx = floor(fx); fx -= sx; edge clamps (:4099-4124);
//             u8: taps = sat_s16(round(c*2048)), H pass int, V pass ((b0*(T0>>4))>>16)+((b1*(T1>>4))>>16)+2)>>2
//             (HResizeLinear :1877-1928, VResizeLinear<uchar> :1963-1989);  f32: T = S0*a0 + S1*a1 (mul, mul, add)
//   AREA 2x2  u8 (a+b+c+d+2)>>2 ; f32 ((a+b)+(c+d))*0.25 (1/4 ch) or (((a+b)+c)+d)*0.25   (:2919-3068, :2857-2900)
//   CUBIC     A=-0.75 taps (interpolateCubic :964-972), per-tap index clamping at the edges (HResizeCubic :1993-2041);
//             u8 V pass: the reference's SSE body evaluates S0*b0+(S1*b1+(S2*b2+S3*b3)) in float with b=beta/2^22 and
//             rounds half-even for the first floor8(width*cn) elements of a row, and uses (sum+2^21)>>22 for the tail
//             (VResizeCubicVec_32s8u :1408-1444, FixedPtCast :2059-2060) -- both are reproduced, so u8 CUBIC is bit-exact.
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include "common.cuh"
#include "resize.cuh"

namespace b200cv {

// ---- NEAREST ------------------------------------------------------------------------------------------------------
// Each thread produces 4 consecutive destination pixels: the 4 gathers are independent (memory-level parallelism) and the
// 4*PIX output bytes leave as 32-bit stores when the destination row allows it.
template <int PIX>   // pixel size in bytes
__global__ void __launch_bounds__(256) resize_nn_kernel(Img src, Img dst, ResizeParams p, int vec_ok)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y;
    const int f = blockIdx.z;
    if (x0 >= p.dw) return;
    const int sy = min((int)floor(__dmul_rn((double)y, p.ify)), p.sh - 1);
    const uchar* srow = src.row<uchar>(f, sy);
    uchar* d = dst.row<uchar>(f, y) + (size_t)x0 * PIX;
    const int n = min(4, p.dw - x0);
    if (vec_ok && n == 4) {
        uint32_t out[PIX];                       // 4 pixels = 4*PIX bytes = PIX words
        uchar* ob = (uchar*)out;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int sx = min((int)floor(__dmul_rn((double)(x0 + k), p.ifx)), p.sw - 1);
            const uchar* sp = srow + (size_t)sx * PIX;
            if constexpr (PIX % 4 == 0) {
#pragma unroll
                for (int i = 0; i < PIX / 4; i++) out[k * (PIX / 4) + i] = ((const uint32_t*)sp)[i];
            } else {
#pragma unroll
                for (int i = 0; i < PIX; i++) ob[k * PIX + i] = sp[i];
            }
        }
#pragma unroll
        for (int i = 0; i < PIX; i++) ((uint32_t*)d)[i] = out[i];
    } else {
        for (int k = 0; k < n; k++) {
            const int sx = min((int)floor(__dmul_rn((double)(x0 + k), p.ifx)), p.sw - 1);
            const uchar* sp = srow + (size_t)sx * PIX;
            for (int i = 0; i < PIX; i++) d[k * PIX + i] = sp[i];
        }
    }
}

// Second version for byte pixels (1, 3, 4 channels): a thread keeps the source offsets of its 4 destination columns and walks down NN_ROWS
// destination rows -- the fp64 column index is computed once per 32 rows instead of once per pixel, and a destination row that maps to the
// same source row as the previous one (every other row when enlarging 2x) stores the registers again without gathering.
constexpr int NN_ROWS = 32;
template <int PIX>
__global__ void __launch_bounds__(128) resize_nn_walk_kernel(Img src, Img dst, ResizeParams p)
{
    const int x0 = (blockIdx.x * 128 + threadIdx.x) * 4;
    const int f = blockIdx.z, y0 = blockIdx.y * NN_ROWS, y1 = min(y0 + NN_ROWS, p.dh);
    if (x0 >= p.dw) return;
    const int n = min(4, p.dw - x0);
    int so[4];
#pragma unroll
    for (int k = 0; k < 4; k++) so[k] = min((int)floor(__dmul_rn((double)min(x0 + k, p.dw - 1), p.ifx)), p.sw - 1) * PIX;
    uint32_t out[PIX];
#pragma unroll
    for (int i = 0; i < PIX; i++) out[i] = 0;
    int prev = -1;
    uchar* d = dst.row<uchar>(f, y0) + (size_t)x0 * PIX;
    for (int y = y0; y < y1; y++, d += dst.step) {
        const int sy = min((int)floor(__dmul_rn((double)y, p.ify)), p.sh - 1);
        if (sy != prev) {
            prev = sy;
            const uchar* srow = src.row<uchar>(f, sy);
            uchar b[4 * PIX];
#pragma unroll
            for (int k = 0; k < 4; k++)
#pragma unroll
                for (int i = 0; i < PIX; i++) b[k * PIX + i] = __ldg(srow + so[k] + i);
#pragma unroll
            for (int i = 0; i < PIX; i++) out[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
        }
        if (n == 4) {
#pragma unroll
            for (int i = 0; i < PIX; i++) ((uint32_t*)d)[i] = out[i];
        } else {
            for (int i = 0; i < n * PIX; i++) d[i] = (uchar)(out[i >> 2] >> (8 * (i & 3)));
        }
    }
}

// ---- coefficient tables ----------------------------------------------------------------------------------------------
// The reference tabulates per destination column / row the source index and the taps once per call on the host
// (resize.cpp:4097-4190).  Same here, on the device: one tiny kernel fills the tables (identical arithmetic to the helpers
// above), the main kernels only read them -- no fp64 in the per-pixel loop.
template <bool CUBIC, bool FIXPT>
__global__ void resize_tab_kernel(ResTab* xt, ResTab* yt, ResizeParams p)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool is_y = i >= p.dw;
    const int d = is_y ? i - p.dw : i;
    if (is_y && d >= p.dh) return;
    (is_y ? yt : xt)[d] = res_tab_entry<CUBIC, FIXPT>(d, is_y, p);
}


// ---- 8-bit taps with word loads ---------------------------------------------------------------------------------------
// The TAPS*CN bytes of one source row that a destination pixel needs are contiguous (away from the clamped image edges): read the
// aligned 32-bit words covering them (one L1 wavefront each instead of one per byte), realign with funnel shifts, gather the two
// bytes of a tap pair with one PRMT and multiply by the s16 coefficient pair with IDP2A (exact: |coef| <= 2^15, bytes <= 255).
template <int NW>      // loads NW + 1 words starting at the word that holds byte A, returns the NW words starting AT byte A
__device__ __forceinline__ void load_realigned(const uchar* row, unsigned A, unsigned* w)
{
    const unsigned* q = (const unsigned*)(row + (A & ~3u));
    const unsigned sh8 = 8 * (A & 3u);
    unsigned t[NW + 1];
#pragma unroll
    for (int i = 0; i <= NW; i++) t[i] = q[i];
#pragma unroll
    for (int i = 0; i < NW; i++) w[i] = __funnelshift_r(t[i], t[i + 1], sh8);
}
template <int CN> __device__ __forceinline__ unsigned rs_tap_pair(const unsigned* w, int c, int j0)
{
    const int p0 = c + j0 * CN, p1 = p0 + CN;
    return __byte_perm(w[p0 >> 2], w[p1 >> 2], (unsigned)((p0 & 3) | ((4 + (p1 & 3)) << 4)));
}
__device__ __forceinline__ int rs_dp2a(int a, unsigned b, int c)
{
    int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}

constexpr int RS_ROWS = 8;   // destination rows per thread
// (Two shared-memory tiled variants were measured and dropped: staging the footprint and filtering every source row once, with
//  the intermediate rows in shared memory or in a per-thread register ring, ran at 12-24 resident warps per SM and were latency
//  bound, slower than the kernels below on the 8K->5K and 4K->8K cases.)

// ---- LINEAR ----------------------------------------------------------------------------------------------------------
template <typename T, int CN>
__global__ void __launch_bounds__(256) resize_linear_kernel(Img src, Img dst, ResizeParams p, const ResTab* __restrict__ xt, const ResTab* __restrict__ yt)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int yb = blockIdx.y * RS_ROWS;
    const int f = blockIdx.z;
    if (x >= p.dw) return;
    const ResTab tx = xt[x];
    const bool last_col = tx.last != 0;                    // dx >= xmax: D = S[sx] * ONE
    const size_t xo = (size_t)tx.s * CN;
    const bool words_ok = sizeof(T) == 1 && (((uintptr_t)src.data | src.step | src.fstep) & 3) == 0;
    const int row_bytes = p.sw * CN * (int)sizeof(T);
#pragma unroll 2
    for (int r = 0; r < RS_ROWS; r++) {
        const int y = yb + r;
        if (y >= p.dh) break;
        const ResTab ty = yt[y];                            // uniform across the CTA: one broadcast load
        const int sy0 = clip_i(ty.s, 0, p.sh), sy1 = clip_i(ty.s + 1, 0, p.sh);   // rows are clipped when fetched, the taps keep fy (:2211)
        const T* r0 = src.row<T>(f, sy0) + xo;
        const T* r1 = src.row<T>(f, sy1) + xo;
        T* d = dst.row<T>(f, y) + (size_t)x * CN;
        if constexpr (sizeof(T) == 1) {
            const int a0 = tx.ic[0], a1 = tx.ic[1], b0 = ty.ic[0], b1 = ty.ic[1];
            constexpr int NW = (2 * CN + 3) / 4;
            if (words_ok && !last_col && (int)xo + 2 * CN + 7 <= row_bytes) {          // the NW+1 words stay inside the row
                const int a01 = (a0 & 0xffff) | (a1 << 16);
                unsigned w0[NW], w1[NW];
                load_realigned<NW>(src.row<uchar>(f, sy0), (unsigned)xo, w0);
                load_realigned<NW>(src.row<uchar>(f, sy1), (unsigned)xo, w1);
#pragma unroll
                for (int c = 0; c < CN; c++) {
                    const int t0 = rs_dp2a(a01, rs_tap_pair<CN>(w0, c, 0), 0), t1 = rs_dp2a(a01, rs_tap_pair<CN>(w1, c, 0), 0);
                    d[c] = (uchar)((((b0 * (t0 >> 4)) >> 16) + ((b1 * (t1 >> 4)) >> 16) + 2) >> 2);
                }
            } else {
#pragma unroll
                for (int c = 0; c < CN; c++) {
                    int t0 = last_col ? r0[c] * 2048 : r0[c] * a0 + r0[c + CN] * a1;
                    int t1 = last_col ? r1[c] * 2048 : r1[c] * a0 + r1[c + CN] * a1;
                    d[c] = (uchar)((((b0 * (t0 >> 4)) >> 16) + ((b1 * (t1 >> 4)) >> 16) + 2) >> 2);
                }
            }
        } else {
            const float a0 = tx.fc[0], a1 = tx.fc[1], b0 = ty.fc[0], b1 = ty.fc[1];
#pragma unroll
            for (int c = 0; c < CN; c++) {
                float t0 = last_col ? r0[c] : __fadd_rn(__fmul_rn(r0[c], a0), __fmul_rn(r0[c + CN], a1));
                float t1 = last_col ? r1[c] : __fadd_rn(__fmul_rn(r1[c], a0), __fmul_rn(r1[c + CN], a1));
                d[c] = __fadd_rn(__fmul_rn(t0, b0), __fmul_rn(t1, b1));
            }
        }
    }
}

// ---- AREA, exact 2x2 ---------------------------------------------------------------------------------------------
// u8: each thread produces 4 destination pixels from 2 rows x 8 source pixels (contiguous 8*CN bytes per row)
template <int CN>
__global__ void __launch_bounds__(256) resize_area2_u8_kernel(Img src, Img dst, int dw, int vec_ok)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x0 >= dw) return;
    const uchar* s0 = src.row<uchar>(f, 2 * y) + (size_t)x0 * 2 * CN;
    const uchar* s1 = src.row<uchar>(f, 2 * y + 1) + (size_t)x0 * 2 * CN;
    uchar* d = dst.row<uchar>(f, y) + (size_t)x0 * CN;
    const int n = min(4, dw - x0);
    if (vec_ok && n == 4) {
        constexpr int NB = 8 * CN;                 // source bytes per row: 8 / 24 / 32
        uint32_t a[NB / 4], b[NB / 4], o[CN];
#pragma unroll
        for (int i = 0; i < NB / 4; i++) { a[i] = __ldg((const uint32_t*)s0 + i); b[i] = __ldg((const uint32_t*)s1 + i); }
        const uchar* pa = (const uchar*)a; const uchar* pb = (const uchar*)b; uchar* po = (uchar*)o;
#pragma unroll
        for (int px = 0; px < 4; px++)
#pragma unroll
            for (int c = 0; c < CN; c++)
                po[px * CN + c] = (uchar)((pa[px * 2 * CN + c] + pa[px * 2 * CN + CN + c] + pb[px * 2 * CN + c] + pb[px * 2 * CN + CN + c] + 2) >> 2);
#pragma unroll
        for (int i = 0; i < CN; i++) ((uint32_t*)d)[i] = o[i];
    } else {
        for (int px = 0; px < n; px++)
#pragma unroll
            for (int c = 0; c < CN; c++)
                d[px * CN + c] = (uchar)((s0[px * 2 * CN + c] + s0[px * 2 * CN + CN + c] + s1[px * 2 * CN + c] + s1[px * 2 * CN + CN + c] + 2) >> 2);
    }
}

template <int CN>
__global__ void __launch_bounds__(256) resize_area2_f32_kernel(Img src, Img dst, int dw)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x >= dw) return;
    const float* s0 = src.row<float>(f, 2 * y) + (size_t)x * 2 * CN;
    const float* s1 = src.row<float>(f, 2 * y + 1) + (size_t)x * 2 * CN;
    float* d = dst.row<float>(f, y) + (size_t)x * CN;
#pragma unroll
    for (int c = 0; c < CN; c++) {
        float a = s0[c], b = s0[c + CN], e = s1[c], g = s1[c + CN];
        // 1 / 4 channels: the 4-lane SIMD body adds row sums, (a+b)+(e+g); 3 channels and the single-channel remainder columns
        // (dw % 4, resize.cpp:3012-3024) run the scalar loop, 0 + (((a+b)+e)+g) -- its sum starts at +0, so -0 comes out as +0
        const bool seq = CN == 3 || (CN == 1 && x >= (dw & ~3));
        float sum = seq ? __fadd_rn(0.f, __fadd_rn(__fadd_rn(__fadd_rn(a, b), e), g)) : __fadd_rn(__fadd_rn(a, b), __fadd_rn(e, g));
        d[c] = __fmul_rn(sum, 0.25f);
    }
}

// ---- CUBIC ---------------------------------------------------------------------------------------------------------------
template <typename T, int CN>
__global__ void __launch_bounds__(256) resize_cubic_kernel(Img src, Img dst, ResizeParams p, const ResTab* __restrict__ xt, const ResTab* __restrict__ yt)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int yb = blockIdx.y * RS_ROWS;
    const int f = blockIdx.z;
    if (x >= p.dw) return;
    const ResTab tx = xt[x];
    const bool words_ok = sizeof(T) == 1 && (((uintptr_t)src.data | src.step | src.fstep) & 3) == 0;
    int xi[4];
#pragma unroll
    for (int j = 0; j < 4; j++) xi[j] = min(max(tx.s - 1 + j, 0), p.sw - 1) * CN;    // per-tap clamping == the while-loops of HResizeCubic
#pragma unroll 1
    for (int r = 0; r < RS_ROWS; r++) {
        const int y = yb + r;
        if (y >= p.dh) break;
        const ResTab ty = yt[y];
        const T* rows[4];
#pragma unroll
        for (int k = 0; k < 4; k++) rows[k] = src.row<T>(f, clip_i(ty.s - 1 + k, 0, p.sh));
        T* d = dst.row<T>(f, y) + (size_t)x * CN;
        if constexpr (sizeof(T) == 1) {
            const int vec_limit = ((p.dw * CN) / 8) * 8;
            const float sc = 1.f / (2048.f * 2048.f);
            constexpr int NW = (4 * CN + 3) / 4;
            int tt[CN][4];
            // taps contiguous (no edge clamping) and the NW+1 words inside the row: word loads + IDP2A
            const bool fastx = words_ok && tx.s >= 1 && tx.s + 2 <= p.sw - 1 && (tx.s - 1) * CN + 4 * CN + 7 <= p.sw * CN;
            if (fastx) {
                const int c01 = (tx.ic[0] & 0xffff) | (tx.ic[1] << 16), c23 = (tx.ic[2] & 0xffff) | (tx.ic[3] << 16);
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    unsigned w[NW];
                    load_realigned<NW>(rows[k], (unsigned)((tx.s - 1) * CN), w);
#pragma unroll
                    for (int c = 0; c < CN; c++) tt[c][k] = rs_dp2a(c23, rs_tap_pair<CN>(w, c, 2), rs_dp2a(c01, rs_tap_pair<CN>(w, c, 0), 0));
                }
            }
#pragma unroll
            for (int c = 0; c < CN; c++) {
                int t[4];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    if (fastx) { t[k] = tt[c][k]; continue; }
                    const uchar* rr = rows[k] + c;
                    t[k] = rr[xi[0]] * tx.ic[0] + rr[xi[1]] * tx.ic[1] + rr[xi[2]] * tx.ic[2] + rr[xi[3]] * tx.ic[3];
                }
                if (x * CN + c < vec_limit) {
                    float v = __fmul_rn((float)t[3], __fmul_rn((float)ty.ic[3], sc));
                    v = __fadd_rn(__fmul_rn((float)t[2], __fmul_rn((float)ty.ic[2], sc)), v);
                    v = __fadd_rn(__fmul_rn((float)t[1], __fmul_rn((float)ty.ic[1], sc)), v);
                    v = __fadd_rn(__fmul_rn((float)t[0], __fmul_rn((float)ty.ic[0], sc)), v);
                    d[c] = sat_u8(__float2int_rn(v));
                } else {
                    d[c] = sat_u8((t[0] * ty.ic[0] + t[1] * ty.ic[1] + t[2] * ty.ic[2] + t[3] * ty.ic[3] + (1 << 21)) >> 22);
                }
            }
        } else {
            const int vec_limit = ((p.dw * CN) / 4) * 4;
#pragma unroll
            for (int c = 0; c < CN; c++) {
                float t[4];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const float* rr = rows[k] + c;
                    float v = __fmul_rn(rr[xi[0]], tx.fc[0]);
                    v = __fadd_rn(v, __fmul_rn(rr[xi[1]], tx.fc[1]));
                    v = __fadd_rn(v, __fmul_rn(rr[xi[2]], tx.fc[2]));
                    v = __fadd_rn(v, __fmul_rn(rr[xi[3]], tx.fc[3]));
                    t[k] = v;
                }
                float o;
                if (x * CN + c < vec_limit) {
                    o = __fmul_rn(t[3], ty.fc[3]);
                    o = __fadd_rn(__fmul_rn(t[2], ty.fc[2]), o);
                    o = __fadd_rn(__fmul_rn(t[1], ty.fc[1]), o);
                    o = __fadd_rn(__fmul_rn(t[0], ty.fc[0]), o);
                } else {
                    o = __fmul_rn(t[0], ty.fc[0]);
                    o = __fadd_rn(o, __fmul_rn(t[1], ty.fc[1]));
                    o = __fadd_rn(o, __fmul_rn(t[2], ty.fc[2]));
                    o = __fadd_rn(o, __fmul_rn(t[3], ty.fc[3]));
                }
                d[c] = o;
            }
        }
    }
}


template <typename T>
static int launch_by_cn(int cn, int interp, const Img& s, const Img& d, const ResizeParams& p, cudaStream_t st)
{
    ResTab* tab = nullptr;
    B200_CUDA(cudaMallocAsync(&tab, sizeof(ResTab) * (size_t)(p.dw + p.dh), st));
    ResTab *xt = tab, *yt = tab + p.dw;
    const unsigned nt = div_up((unsigned)(p.dw + p.dh), 256);
    constexpr bool FIX = sizeof(T) == 1;
    if (interp == B200CV_INTER_LINEAR) resize_tab_kernel<false, FIX><<<nt, 256, 0, st>>>(xt, yt, p);
    else resize_tab_kernel<true, FIX><<<nt, 256, 0, st>>>(xt, yt, p);
    count_launch();
    if (sizeof(T) == 1) {          // 8-bit: the tiled separable kernels (resize_sep.cu)
        const int rc = resize_sep_u8(s, d, cn, interp == B200CV_INTER_CUBIC, p, xt, yt, st);
        if (rc != B200CV_NOT_IMPLEMENTED) { cudaFreeAsync(tab, st); return rc; }
    }
    dim3 grid(div_up((unsigned)p.dw, 256), div_up((unsigned)p.dh, RS_ROWS), (unsigned)s.frames);
#define L(K, CN) K<T, CN><<<grid, 256, 0, st>>>(s, d, p, xt, yt)
    if (interp == B200CV_INTER_LINEAR) {
        if (cn == 1) L(resize_linear_kernel, 1); else if (cn == 3) L(resize_linear_kernel, 3); else L(resize_linear_kernel, 4);
    } else {
        if (cn == 1) L(resize_cubic_kernel, 1); else if (cn == 3) L(resize_cubic_kernel, 3); else L(resize_cubic_kernel, 4);
    }
#undef L
    cudaError_t e = cudaGetLastError();
    cudaFreeAsync(tab, st);
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

int copy_impl(const b200cvMat* src, const b200cvMat* dst, void* stream);

}  // namespace b200cv

using namespace b200cv;

static int resize_impl(const b200cvMat* src, const b200cvMat* dst, int interpolation, double fx, double fy, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->type == dst->type, "resize: dst type must equal src type");
    B200_REQUIRE(src->data != dst->data, "resize: in-place is not supported");
    const int depth = B200CV_DEPTH(src->type), cn = B200CV_CN(src->type);
    if ((depth != B200CV_8U && depth != B200CV_32F) || (cn != 1 && cn != 3 && cn != 4)) return B200CV_NOT_IMPLEMENTED;
    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    if (s.rows >= 65536 || d.rows >= 65536 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    cudaStream_t st = as_stream(stream);
    if (src->cols == dst->cols && src->rows == dst->rows) return copy_impl(src, dst, stream);   // resize.cpp:4238

    ResizeParams p;
    p.sw = src->cols; p.sh = src->rows; p.dw = dst->cols; p.dh = dst->rows;
    // hal::resize, resize.cpp:3835-3839: the scale is dsize / ssize -- unless the caller gave fx, fy (cv::resize with an empty dsize,
    // resize.cpp:4214-4228), which then stay as they are even when cols * fx is not an integer
    const double size_x = (double)p.dw / p.sw, size_y = (double)p.dh / p.sh;
    const bool explicit_scale = fx > 0 && fy > 0 && (fx != size_x || fy != size_y);
    const double inv_x = fx > 0 && fy > 0 ? fx : size_x, inv_y = fx > 0 && fy > 0 ? fy : size_y;
    p.ifx = 1. / inv_x; p.ify = 1. / inv_y;
    p.scale_x = 1. / inv_x; p.scale_y = 1. / inv_y;
    p.inv_x = inv_x; p.inv_y = inv_y; p.area_mode = 0;
    const int pix = (int)elem_size(src->type);
    dim3 grid(div_up((unsigned)p.dw, 256), (unsigned)p.dh, (unsigned)s.frames);

    // the EXACT / AREA / LANCZOS4 kernels derive their scale from the sizes: decline factors that differ from it (a host OpenCV then runs its own code)
    if (explicit_scale && interpolation != B200CV_INTER_NEAREST && interpolation != B200CV_INTER_LINEAR && interpolation != B200CV_INTER_CUBIC) return B200CV_NOT_IMPLEMENTED;
    if (interpolation == B200CV_INTER_NEAREST_EXACT) return resize_exact_impl(s, d, depth, cn, interpolation, st);
    if (interpolation == B200CV_INTER_LINEAR_EXACT && depth == B200CV_32F) interpolation = B200CV_INTER_LINEAR;      // cv::resize, resize.cpp:4223
    if (interpolation == B200CV_INTER_NEAREST) {
        dim3 g4(div_up(div_up((unsigned)p.dw, 4), 128), (unsigned)p.dh, (unsigned)s.frames);
        int vec_ok = (((uintptr_t)d.data | d.step | d.fstep) & 3) == 0 && (pix % 4 != 0 || (((uintptr_t)s.data | s.step | s.fstep) & 3) == 0);
        const char* nn_env = getenv("B200CV_RESIZE_NN_PATH");              // "v1": the per-pixel kernel always; "walk": the walking kernel whenever it applies
        // only when rows repeat (enlarging in y): there the walking kernel reuses each gathered row; when shrinking, the per-pixel kernel
        // has 32x the threads in flight for the same gathers
        const bool walk = (nn_env && !strcmp(nn_env, "walk")) || (p.dh > p.sh && !(nn_env && !strcmp(nn_env, "v1")));
        if (walk && depth == B200CV_8U && (pix == 1 || pix == 3 || pix == 4) && (((uintptr_t)d.data | d.step | d.fstep) & 3) == 0) {
            dim3 gw(div_up(div_up((unsigned)p.dw, 4), 128), div_up((unsigned)p.dh, NN_ROWS), (unsigned)s.frames);
            if (pix == 1) resize_nn_walk_kernel<1><<<gw, 128, 0, st>>>(s, d, p);
            else if (pix == 3) resize_nn_walk_kernel<3><<<gw, 128, 0, st>>>(s, d, p);
            else resize_nn_walk_kernel<4><<<gw, 128, 0, st>>>(s, d, p);
            B200_LAUNCH_CHECK();
            return B200CV_OK;
        }
        switch (pix) {
        case 1: resize_nn_kernel<1><<<g4, 128, 0, st>>>(s, d, p, vec_ok); break;
        case 3: resize_nn_kernel<3><<<g4, 128, 0, st>>>(s, d, p, vec_ok); break;
        case 4: resize_nn_kernel<4><<<g4, 128, 0, st>>>(s, d, p, vec_ok); break;
        case 12: resize_nn_kernel<12><<<g4, 128, 0, st>>>(s, d, p, vec_ok); break;
        case 16: resize_nn_kernel<16><<<g4, 128, 0, st>>>(s, d, p, vec_ok); break;
        default: return B200CV_NOT_IMPLEMENTED;
        }
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }
    // exact 2x2 decimation: INTER_AREA, and INTER_LINEAR which the reference rewrites to it (resize.cpp:4009-4012)
    const int isx = (int)lrint(p.scale_x), isy = (int)lrint(p.scale_y);
    const bool area_fast = fabs(p.scale_x - isx) < 2.220446049250313e-16 && fabs(p.scale_y - isy) < 2.220446049250313e-16;
    if ((interpolation == B200CV_INTER_LINEAR || interpolation == B200CV_INTER_AREA || interpolation == B200CV_INTER_LINEAR_EXACT) && area_fast && isx == 2 && isy == 2) {   // LINEAR_EXACT: resize.cpp:3976-3981
        // explicit fx = fy = 0.5 on odd sizes: the reference's partial last windows (resizeAreaFast_Invoker, resize.cpp:3028-3050) are not built here
        if (2 * p.dw != p.sw || 2 * p.dh != p.sh) return B200CV_NOT_IMPLEMENTED;
        if (depth == B200CV_8U) {
            int vec_ok = (((uintptr_t)s.data | s.step | s.fstep | (uintptr_t)d.data | d.step | d.fstep) & 3) == 0;
            dim3 g4(div_up((unsigned)div_up((unsigned)p.dw, 4), 256), (unsigned)p.dh, (unsigned)s.frames);
            if (cn == 1) resize_area2_u8_kernel<1><<<g4, 256, 0, st>>>(s, d, p.dw, vec_ok);
            else if (cn == 3) resize_area2_u8_kernel<3><<<g4, 256, 0, st>>>(s, d, p.dw, vec_ok);
            else resize_area2_u8_kernel<4><<<g4, 256, 0, st>>>(s, d, p.dw, vec_ok);
        } else {
            if (cn == 1) resize_area2_f32_kernel<1><<<grid, 256, 0, st>>>(s, d, p.dw);
            else if (cn == 3) resize_area2_f32_kernel<3><<<grid, 256, 0, st>>>(s, d, p.dw);
            else resize_area2_f32_kernel<4><<<grid, 256, 0, st>>>(s, d, p.dw);
        }
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }
    if (interpolation == B200CV_INTER_LINEAR_EXACT) return resize_exact_impl(s, d, depth, cn, interpolation, st);
    if (interpolation == B200CV_INTER_LANCZOS4) return resize_lanczos_impl(s, d, depth, cn, st);
    // true area mode (both factors >= 1): resize_area.cu.  With an enlarging axis INTER_AREA is the bilinear kernel with area-mode weights
    if (interpolation == B200CV_INTER_AREA && p.scale_x >= 1 && p.scale_y >= 1) return resize_area_impl(s, d, depth, cn, st);
    if (interpolation == B200CV_INTER_AREA) { p.area_mode = 1; interpolation = B200CV_INTER_LINEAR; }
    if (interpolation != B200CV_INTER_LINEAR && interpolation != B200CV_INTER_CUBIC) return B200CV_NOT_IMPLEMENTED;
    return depth == B200CV_8U ? launch_by_cn<uchar>(cn, interpolation, s, d, p, st) : launch_by_cn<float>(cn, interpolation, s, d, p, st);
}

extern "C" int b200cv_resize(const b200cvMat* src, const b200cvMat* dst, int interpolation, void* stream)
{
    return resize_impl(src, dst, interpolation, 0., 0., stream);
}

// cv::resize(src, dst, Size(), fx, fy): dst is round(cols * fx) x round(rows * fy) and the sampling scale is fx, fy themselves
extern "C" int b200cv_resize_scaled(const b200cvMat* src, const b200cvMat* dst, int interpolation, double fx, double fy, void* stream)
{
    return resize_impl(src, dst, interpolation, fx, fy, stream);
}
