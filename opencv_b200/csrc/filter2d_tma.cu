// filter2d_tma.cu -- cv::filter2D fast path: single channel, centred odd kernels up to 31x31, rows that TMA can address.
//
// Same arithmetic as filter2d_fast_kernel (filter2d.cu): s = delta; for every tap in row-major order s = fma(k, src, s);
// dst = saturate_cast<DT>(s)  (Filter2D<ST,CastOp,VecOp>, modules/imgproc/src/filter.simd.hpp:3103-3175; taps that are zero do not
// change s, so the zero padding of the tap bucket is invisible).  What differs is the data movement, which is all there is to a
// small filter: one thread issues a 3-D TMA box load of the (192 + apron) x (32 + K - 1) source tile (zero fill outside the image =
// BORDER_CONSTANT; boundary CTAs patch the apron for the mirrored modes), 8-bit tiles are widened to float once per element
// (PRMT into the mantissa of 2^23 + FADD, no I2F), each thread keeps an 8-output row segment in registers and walks the kernel rows
// with 128-bit shared loads, and results leave as 8-byte (u8) or 2 x 16-byte (f32) stores.  The previous kernel spent its time in
// per-element border arithmetic and scalar loads/stores, far from the HBM time.
#include <cstring>
#include "common.cuh"
#include "tma.cuh"

namespace b200cv {

constexpr int FT_TW = 192, FT_TH = 32, FT_IW = 224;

struct FTParams {
    float k[31 * 31];          // KB x KB, zero padded and centred
    float delta;
    int W, H, border;
    int ky0, ky1;              // kernel rows that hold non-zero taps
};

template <typename DT> __device__ __forceinline__ void ft_store8(DT* dp, const float* v, bool vec, int n);

template <> __device__ __forceinline__ void ft_store8<uchar>(uchar* dp, const float* v, bool vec, int n)
{
    // saturate_cast<uchar>(float) = clamp(rint(v)): clamp first (the bounds are integers), then round-to-nearest-even by adding 1.5 * 2^23
    uint32_t b[8];
#pragma unroll
    for (int i = 0; i < 8; i++) b[i] = __float_as_uint(__fadd_rn(fminf(fmaxf(v[i], 0.f), 255.f), 12582912.f));
    const uint32_t lo = __byte_perm(__byte_perm(b[0], b[1], 0x0040), __byte_perm(b[2], b[3], 0x0040), 0x5410);
    const uint32_t hi = __byte_perm(__byte_perm(b[4], b[5], 0x0040), __byte_perm(b[6], b[7], 0x0040), 0x5410);
    if (vec && n == 8) *(uint2*)dp = make_uint2(lo, hi);
    else {
#pragma unroll
        for (int i = 0; i < 8; i++) if (i < n) dp[i] = (uchar)((i < 4 ? lo : hi) >> (8 * (i & 3)));
    }
}
template <> __device__ __forceinline__ void ft_store8<float>(float* dp, const float* v, bool vec, int n)
{
    if (vec && n == 8) { ((float4*)dp)[0] = make_float4(v[0], v[1], v[2], v[3]); ((float4*)dp)[1] = make_float4(v[4], v[5], v[6], v[7]); }
    else {
#pragma unroll
        for (int i = 0; i < 8; i++) if (i < n) dp[i] = v[i];
    }
}

template <int KB, typename ST, typename DT>
__global__ void __launch_bounds__(256, 2) filter2d_tma_kernel(const __grid_constant__ CUtensorMap tmap, Img dst, const __grid_constant__ FTParams p)
{
    constexpr int RB = KB / 2;
    constexpr int RA = sizeof(ST) == 1 ? 16 : ((RB + 3) / 4) * 4;   // left apron staged: the TMA box must start on a 16-byte boundary
    constexpr int OFF = RA - RB;
    constexpr int IH = FT_TH + KB - 1;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_f = (float*)smem_raw;                                   // IH x FT_IW floats
    ST* s_in = (ST*)(smem_raw + (size_t)IH * FT_IW * 4);            // raw TMA tile behind the (swizzled) float tile
    __shared__ __align__(8) uint64_t s_bar;
    const int f = blockIdx.z, x0 = blockIdx.x * FT_TW, y0 = blockIdx.y * FT_TH;
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&s_bar, 1);
        fence_barrier_init();
        mbar_arrive_expect_tx(&s_bar, (uint32_t)(FT_IW * IH * sizeof(ST)));
        tma_load_3d(s_in, &tmap, x0 - RA, y0 - RB, f, &s_bar);
        // only this thread polls the barrier; the others sleep in bar.sync instead of spending issue slots on a spin loop
        mbar_wait(&s_bar, 0);
    }
    __syncthreads();

    const int tx0 = x0 - RA;
    const bool edge = (tx0 < 0) || (y0 - RB < 0) || (tx0 + FT_IW > p.W) || (y0 - RB + IH > p.H);
    if (edge && p.border != B200CV_BORDER_CONSTANT) {
        for (int idx = tid; idx < IH * FT_IW; idx += 256) {
            int r = idx / FT_IW, c = idx - r * FT_IW;
            int gy = y0 - RB + r;
            if ((unsigned)gy < (unsigned)p.H) continue;
            int sr = border_interpolate(gy, p.H, p.border) - (y0 - RB);
            if ((unsigned)sr < (unsigned)IH) s_in[idx] = s_in[sr * FT_IW + c];   // rows beyond the apron feed no valid output
        }
        __syncthreads();
        const int c_first = p.W - tx0;                        // first tile column right of the image (may be >= FT_IW)
        const int nright = c_first < FT_IW ? min(FT_IW - c_first, RB + 4) : 0;
        const int nleft = tx0 < 0 ? RA : 0;
        const int ncol = nleft + nright;
        for (int idx = tid; idx < IH * ncol; idx += 256) {
            int r = idx / ncol, k = idx - r * ncol;
            int c = k < nleft ? k : c_first + (k - nleft);
            int sc = border_interpolate(tx0 + c, p.W, p.border) - tx0;
            if ((unsigned)sc < (unsigned)FT_IW) s_in[r * FT_IW + c] = s_in[r * FT_IW + sc];
        }
        __syncthreads();
    }
    // Build the float tile.  Its 16-byte chunks are stored XOR-swizzled (chunk c -> c ^ ((c >> 3) & 1)): a thread's window starts 32 bytes
    // after its neighbour's, so un-swizzled 128-bit loads of 8 adjacent lanes would hit every bank twice (ncu: 93 M conflicts at 7x7).
    for (int idx = tid; idx < IH * (FT_IW / 4); idx += 256) {
        float4 v;
        if constexpr (sizeof(ST) == 1) {      // widen: 4 bytes -> 4 floats (PRMT into the mantissa of 2^23, no I2F)
            const uint32_t q = ((const uint32_t*)s_in)[idx];
            v.x = __fsub_rn(__uint_as_float(__byte_perm(q, 0x4B000000u, 0x7650)), 8388608.0f);
            v.y = __fsub_rn(__uint_as_float(__byte_perm(q, 0x4B000000u, 0x7651)), 8388608.0f);
            v.z = __fsub_rn(__uint_as_float(__byte_perm(q, 0x4B000000u, 0x7652)), 8388608.0f);
            v.w = __fsub_rn(__uint_as_float(__byte_perm(q, 0x4B000000u, 0x7653)), 8388608.0f);
        } else {
            v = ((const float4*)s_in)[idx];
        }
        const int row = idx / (FT_IW / 4), c = idx - row * (FT_IW / 4);
        ((float4*)s_f)[row * (FT_IW / 4) + (c ^ ((c >> 3) & 1))] = v;
    }
    __syncthreads();

    // ---- item = 8 consecutive outputs of one row; the kernel rows stream through a register window ----
    constexpr int GPR = FT_TW / 8;
    constexpr int NEED = 8 + KB - 1;
    constexpr int NV = (OFF + NEED + 3) / 4;
    const bool dvec = (((uintptr_t)dst.data | dst.step | dst.fstep) & (8 * sizeof(DT) > 16 ? 15 : 8 * sizeof(DT) - 1)) == 0;
#pragma unroll 1
    for (int it = tid; it < FT_TH * GPR; it += 256) {
        const int r = it / GPR, g = it - r * GPR;
        const int gy = y0 + r, gx = x0 + g * 8;
        if (gy >= p.H || gx >= p.W) continue;
        float acc[8];
#pragma unroll
        for (int o = 0; o < 8; o++) acc[o] = p.delta;
        // one kernel row: the thread's window (128-bit shared loads, swizzled chunks) against the row's KB taps
        auto kernel_row = [&](int ky, const float* kr) {
            const float4* vp = (const float4*)(s_f + (r + ky) * FT_IW);
            float win[NV * 4];
#pragma unroll
            for (int w = 0; w < NV; w++) {
                int c = g * 2 + w;
                c ^= (c >> 3) & 1;
                const float4 q = vp[c];
                win[4 * w] = q.x; win[4 * w + 1] = q.y; win[4 * w + 2] = q.z; win[4 * w + 3] = q.w;
            }
#pragma unroll
            for (int i = 0; i < KB; i++) {
                const float t = kr[i];
#pragma unroll
                for (int o = 0; o < 8; o++) {
                    // 8-bit source with a float destination is the reference's scalar FilterNoVec: products rounded before the add
                    if constexpr (sizeof(ST) == 1 && sizeof(DT) == 4) acc[o] = __fadd_rn(acc[o], __fmul_rn(t, win[OFF + o + i]));
                    else acc[o] = fmaf(t, win[OFF + o + i], acc[o]);
                }
            }
        };
        if constexpr (KB <= 7) {
            // small kernels: every row unrolled, the taps are FFMA constant-bank operands at compile-time offsets (no LDC, no loop); rows of
            // zeros are not skipped -- fma(0, x, s) == s for the finite x of an image
#pragma unroll
            for (int ky = 0; ky < KB; ky++) kernel_row(ky, p.k + ky * KB);
        } else {
#pragma unroll 1
            for (int ky = p.ky0; ky < p.ky1; ky++) kernel_row(ky, p.k + ky * KB);
        }
        ft_store8<DT>(dst.row<DT>(f, gy) + gx, acc, dvec, min(8, p.W - gx));
    }
}

template <int KB, typename ST, typename DT>
static int launch_ft(const CUtensorMap& tm, const Img& d, const FTParams& p, int frames, cudaStream_t st)
{
    constexpr int IH = FT_TH + KB - 1;
    const size_t smem = (size_t)IH * FT_IW * 4 + (size_t)IH * FT_IW * sizeof(ST);
    auto kern = filter2d_tma_kernel<KB, ST, DT>;
    static PerDeviceFlag attr_pd; bool& attr = attr_pd.cur();
    if (!attr) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
    dim3 grid(div_up((unsigned)p.W, FT_TW), div_up((unsigned)p.H, FT_TH), (unsigned)frames);
    kern<<<grid, 256, smem, st>>>(tm, d, p);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

template <typename ST, typename DT>
static int filter2d_fast_t(const Img& s, const Img& d, const float* k, int kw, int kh, float delta, int border, cudaStream_t st)
{
    static const int buckets[] = {3, 5, 7, 9, 11, 13, 15, 21, 31};
    int kmax = kw > kh ? kw : kh, KB = 0;
    for (int b : buckets) if (kmax <= b) { KB = b; break; }
    if (!KB || s.cols < KB || s.rows < KB) return B200CV_NOT_IMPLEMENTED;
    static thread_local FTParams p;
    memset(&p, 0, sizeof(p));
    const int ox = (KB - kw) / 2, oy = (KB - kh) / 2;
    for (int y = 0; y < kh; y++) for (int x = 0; x < kw; x++) p.k[(oy + y) * KB + ox + x] = k[y * kw + x];
    p.delta = delta; p.W = s.cols; p.H = s.rows; p.border = border; p.ky0 = oy; p.ky1 = oy + kh;
    CUtensorMap tm;
    int rc = make_tensor_map_3d(&tm, s.data, (int)sizeof(ST), s.cols, s.rows, s.frames, s.step, s.fstep, FT_IW, FT_TH + KB - 1);
    if (rc) return rc;
    switch (KB) {
    case 3: return launch_ft<3, ST, DT>(tm, d, p, s.frames, st);
    case 5: return launch_ft<5, ST, DT>(tm, d, p, s.frames, st);
    case 7: return launch_ft<7, ST, DT>(tm, d, p, s.frames, st);
    case 9: return launch_ft<9, ST, DT>(tm, d, p, s.frames, st);
    case 11: return launch_ft<11, ST, DT>(tm, d, p, s.frames, st);
    case 13: return launch_ft<13, ST, DT>(tm, d, p, s.frames, st);
    case 15: return launch_ft<15, ST, DT>(tm, d, p, s.frames, st);
    case 21: return launch_ft<21, ST, DT>(tm, d, p, s.frames, st);
    case 31: return launch_ft<31, ST, DT>(tm, d, p, s.frames, st);
    }
    return B200CV_NOT_IMPLEMENTED;
}

// returns B200CV_NOT_IMPLEMENTED when the fast path does not apply (filter2d.cu falls back to its own kernels)
int filter2d_tma(const Img& s, const Img& d, int sd, int dd, int cn, const float* k, int kw, int kh, int ax, int ay, float delta, int border, cudaStream_t st)
{
    if (cn != 1 || !(kw & 1) || !(kh & 1) || kw > 31 || kh > 31 || ax != kw / 2 || ay != kh / 2) return B200CV_NOT_IMPLEMENTED;
    if (border == B200CV_BORDER_WRAP || !tma_compatible(s) || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    if (sd == B200CV_8U && dd == B200CV_8U) return filter2d_fast_t<uchar, uchar>(s, d, k, kw, kh, delta, border, st);
    if (sd == B200CV_8U && dd == B200CV_32F) return filter2d_fast_t<uchar, float>(s, d, k, kw, kh, delta, border, st);
    if (sd == B200CV_32F && dd == B200CV_32F) return filter2d_fast_t<float, float>(s, d, k, kw, kh, delta, border, st);
    return B200CV_NOT_IMPLEMENTED;
}

}  // namespace b200cv
