// sep_f32.cu -- single-channel separable filter in float arithmetic, fast path (GaussianBlur f32, sepFilter2D f32, the SIFT
// pyramid blurs; sepFilter2D on 8-bit data with taps that are not 8-bit exact, where the reference also computes in float):
// TMA tile load + FFMA row/column passes, optional fused difference-of-Gaussians output.
//
// Arithmetic = the operation order of the reference's AVX2 objects, so the results are bit-identical to the CPU's:
//   rows     s = fma(x[i], kx[i], s) in tap order from 0 (RowVec_32f, filter.simd.hpp:1632-1650); a float source with 3 or 5
//            (anti)symmetric taps goes centre-out: fma(x0, k0, (x-1 + x1) k1), then fma(x-2 + x2, k2, .) (SymmRowSmallVec_32f :1768-1844)
//   columns  mirrored rows first: s = fma(ky[c], S[c], delta); s = fma(ky[c+k], S[c+k] +/- S[c-k], s)  (SymmColumnVec_32f :1878-1949,
//            SymmColumnVec_32f8u :1158-1202).  Kernels that are not (anti)symmetric are left to the generic kernel.
//   Taps are centred in a zero-padded bucket of KB.  Float sources whose kernel has zero taps the reference never evaluates -- the
//   padding to the bucket (px / py), the centre of an antisymmetric column kernel or of antisymmetric 3/5-tap rows -- run an
//   instantiation (SKIP0) that skips them: fma(inf, 0, s) would be NaN where the reference has a finite value or an infinity.  Full
//   symmetric buckets keep the unpredicated loops; 8-bit rows are finite, so they need no such instantiation.
// Same arithmetic as sep_fast_kernel<.,.,M_FLOAT,KB> in sepfilter.cu -- only the data movement differs: ONE thread issues a 3-D cp.async.bulk.tensor box load of the
// (192+2r) x (32+2r) float tile into shared memory and the CTA waits on an mbarrier, so the loads of one CTA overlap the
// arithmetic of the other CTAs resident on the SM instead of stalling every thread on its own LDG (the generic kernel was
// long-scoreboard bound).  TMA zero-fills outside the image (= BORDER_CONSTANT); for
// REPLICATE / REFLECT / REFLECT_101 only boundary CTAs patch their apron from the mirrored in-tile cells.
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "tma.cuh"

namespace b200cv {

constexpr int SF_TW = 192, SF_TH = 32, SF_IW = 224;

struct SF32Params {
    float kx[32], ky[32];      // zero padded + centred to KB taps
    float delta;
    int W, H, border;
    Img dog;
    int has_dog;
    int row_small;             // float source, 3/5 (anti)symmetric taps: 1 symmetric, 2 antisymmetric (centre-out order), 0 tap order
    unsigned col_sign;         // 0: symmetric column kernel, 0x80000000: antisymmetric (S[c+k] - S[c-k])
    int px, py;                // zero taps padding kx / ky to KB on each side: skipped (SKIP0), so a non-finite pixel reaches only the real footprint
    int nch;                   // chunks of SF_TH output rows one CTA walks down (1 = the plain tile kernel)
};

// ---- up to 11 taps: the plain tile kernel (one 192 x 32 tile per CTA, 3 CTAs per SM at 80 registers) -- the walking kernel below carries
//      state that does not fit that register budget (its tile form is slower at 3 and 9 taps) ----
template <int KB, typename ST, typename DT, bool SKIP0>
__global__ void __launch_bounds__(256, 3) sep_f32_tile_kernel(const __grid_constant__ CUtensorMap tmap, Img dst, const __grid_constant__ SF32Params p)
{
    constexpr int RB = KB / 2;
    constexpr int RA = sizeof(ST) == 1 ? 16 : ((RB + 3) / 4) * 4;   // left apron staged: TMA needs the box to start on a 16-byte boundary
    constexpr int OFF = RA - RB;
    constexpr int IH = SF_TH + KB - 1;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    ST* s_in = (ST*)smem_raw;                             // IH x SF_IW
    float* s_mid = (float*)(smem_raw + (((size_t)IH * SF_IW * sizeof(ST) + 127) & ~(size_t)127));    // IH x SF_TW
    __shared__ __align__(8) uint64_t s_bar;
    const int f = blockIdx.z, x0 = blockIdx.x * SF_TW, y0 = blockIdx.y * SF_TH;
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&s_bar, 1);
        fence_barrier_init();
        mbar_arrive_expect_tx(&s_bar, (uint32_t)(SF_IW * IH * sizeof(ST)));
        tma_load_3d(s_in, &tmap, x0 - RA, y0 - RB, f, &s_bar);
        // only this thread polls the barrier; the others sleep in bar.sync instead of spending issue slots on a spin loop
        mbar_wait(&s_bar, 0);
    }
    __syncthreads();

    const int tx0 = x0 - RA;
    const bool edge = (tx0 < 0) || (y0 - RB < 0) || (tx0 + SF_IW > p.W) || (y0 - RB + IH > p.H);
    if (edge && p.border != B200CV_BORDER_CONSTANT) {
        for (int idx = tid; idx < IH * SF_IW; idx += 256) {
            int r = idx / SF_IW, c = idx - r * SF_IW;
            int gy = y0 - RB + r;
            if ((unsigned)gy < (unsigned)p.H) continue;
            int sr = border_interpolate(gy, p.H, p.border) - (y0 - RB);
            if ((unsigned)sr < (unsigned)IH) s_in[idx] = s_in[sr * SF_IW + c];   // rows beyond the apron feed no valid output
        }
        __syncthreads();
        const int c_first = p.W - tx0;                        // first tile column right of the image (may be >= SF_IW)
        const int nright = c_first < SF_IW ? min(SF_IW - c_first, RB + 4) : 0;
        const int nleft = tx0 < 0 ? RA : 0;
        const int ncol = nleft + nright;
        for (int idx = tid; idx < IH * ncol; idx += 256) {
            int r = idx / ncol, k = idx - r * ncol;
            int c = k < nleft ? k : c_first + (k - nleft);
            int sc = border_interpolate(tx0 + c, p.W, p.border) - tx0;
            if ((unsigned)sc < (unsigned)SF_IW) s_in[r * SF_IW + c] = s_in[r * SF_IW + sc];
        }
        __syncthreads();
    }

    // ---- row pass: item = NO consecutive outputs of one staged row.  Float rows: NO = 4, so that neighbouring lanes read neighbouring
    //      16-byte chunks (8 outputs = 32-byte lane stride made every 128-bit shared load a 2-way bank conflict); byte rows: NO = 8 ----
    {
        constexpr int NO = sizeof(ST) == 4 ? 4 : 8;
        constexpr int GPR = SF_TW / NO;                   // items per row
        constexpr int NEED = NO + KB - 1;
        constexpr int NV = (OFF + NEED + 3) / 4;
#pragma unroll 1
        for (int it = tid; it < IH * GPR; it += 256) {
            const int r = it / GPR, g = it - r * GPR;
            float win[NV * 4];                            // the item's window (+ alignment slack), all indices compile-time
#pragma unroll
            for (int w = 0; w < NV; w++) {
                if constexpr (sizeof(ST) == 1) {
                    // bytes -> floats through the mantissa of 2^23 (PRMT + FADD instead of the quarter-rate I2F)
                    const uint32_t q = ((const uint32_t*)(s_in + r * SF_IW + g * NO))[w];
#pragma unroll
                    for (int b = 0; b < 4; b++) win[w * 4 + b] = __fsub_rn(__uint_as_float(__byte_perm(q, 0x4B000000u, 0x7650 + b)), 8388608.0f);
                } else {
                    const float4 q = ((const float4*)(s_in + r * SF_IW + g * NO))[w];
                    win[w * 4] = q.x; win[w * 4 + 1] = q.y; win[w * 4 + 2] = q.z; win[w * 4 + 3] = q.w;
                }
            }
            float acc[NO];
            bool done = false;
            if constexpr (KB <= 5 && sizeof(ST) == 4) {
                if (p.row_small) {
                    const unsigned sg = p.row_small == 2 ? 0x80000000u : 0u;
#pragma unroll
                    for (int o = 0; o < NO; o++) {
                        const float* x = win + OFF + o + RB;      // centre tap
                        // symmetric: fma(x0, k0, (x-1 + x1) k1); antisymmetric: (x1 - x-1) k1, no centre term (SKIP0; fma(x0, 0, t) = t for finite x0)
                        float t = __fmul_rn(__fadd_rn(x[1], __uint_as_float(__float_as_uint(x[-1]) ^ sg)), p.kx[RB + 1]);
                        if (!SKIP0 || p.row_small != 2) t = fmaf(x[0], p.kx[RB], t);
                        if constexpr (KB == 5) if (!SKIP0 || !p.px) t = fmaf(__fadd_rn(x[2], __uint_as_float(__float_as_uint(x[-2]) ^ sg)), p.kx[RB + 2], t);
                        acc[o] = t;
                    }
                    done = true;
                }
            }
            if (!done) {
#pragma unroll
                for (int o = 0; o < NO; o++) {
                    float t = 0.f;
#pragma unroll
                    for (int i = 0; i < KB; i++)
                        if (!SKIP0 || (i >= p.px && i < KB - p.px)) t = fmaf(win[OFF + o + i], p.kx[i], t);
                    acc[o] = t;
                }
            }
            float4* mp = (float4*)(s_mid + r * SF_TW + g * NO);
            mp[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
            if constexpr (NO == 8) mp[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
        }
    }
    __syncthreads();

    // ---- column pass: item = CW columns x R rows; the R + KB - 1 mid rows it needs are held in registers ----
    {
        constexpr int CW = KB <= 15 ? 4 : 2, R = KB == 11 ? 4 : 8;   // window: (R + KB - 1) x CW registers, sized for 3 (KB <= 11) or 2 CTAs per SM
        constexpr int IPR = SF_TW / CW;                   // items per row group
        const bool dvec = (((uintptr_t)dst.data | dst.step | dst.fstep) & (CW * sizeof(DT) - 1)) == 0;
        const bool gvec = p.has_dog && (((uintptr_t)p.dog.data | p.dog.step | p.dog.fstep) & (CW * 4 - 1)) == 0;
#pragma unroll 1
        for (int it = tid; it < IPR * (SF_TH / R); it += 256) {
            const int q = it / IPR, cg = it - q * IPR;
            const float* mbase = s_mid + (q * R) * SF_TW + cg * CW;
            float win[R + KB - 1][CW];
#pragma unroll
            for (int m = 0; m < R + KB - 1; m++) {
                if constexpr (CW == 4) {
                    const float4 v = *(const float4*)(mbase + m * SF_TW);
                    win[m][0] = v.x; win[m][1] = v.y; win[m][2] = v.z; win[m][3] = v.w;
                } else {
                    const float2 v = *(const float2*)(mbase + m * SF_TW);
                    win[m][0] = v.x; win[m][1] = v.y;
                }
            }
            const int gx = x0 + cg * CW;
            if (gx >= p.W) continue;
#pragma unroll
            for (int o = 0; o < R; o++) {
                const int gy = y0 + q * R + o;
                if (gy >= p.H) break;
                float acc[CW];
#pragma unroll
                for (int c = 0; c < CW; c++) {
                    float t = (SKIP0 && p.col_sign) ? p.delta : fmaf(p.ky[RB], win[o + RB][c], p.delta);   // antisymmetric: no centre row
#pragma unroll
                    for (int k = 1; k <= RB; k++)
                        if (!SKIP0 || k <= RB - p.py)
                            t = fmaf(p.ky[RB + k], __fadd_rn(win[o + RB + k][c], __uint_as_float(__float_as_uint(win[o + RB - k][c]) ^ p.col_sign)), t);
                    acc[c] = t;
                }
                if constexpr (sizeof(DT) == 1) {
                    uchar* dp = dst.row<uchar>(f, gy) + gx;
                    uint32_t pk = 0;
#pragma unroll
                    for (int c = 0; c < CW; c++) pk |= (uint32_t)sat_u8(acc[c]) << (8 * c);
                    if (dvec && gx + CW <= p.W) {
                        if constexpr (CW == 4) *(uint32_t*)dp = pk; else *(unsigned short*)dp = (unsigned short)pk;
                    } else {
#pragma unroll
                        for (int c = 0; c < CW; c++) if (gx + c < p.W) dp[c] = (uchar)(pk >> (8 * c));
                    }
                } else {
                    float* dp = dst.row<float>(f, gy) + gx;
                    if (dvec && gx + CW <= p.W) {
                        if constexpr (CW == 4) *(float4*)dp = make_float4(acc[0], acc[1], acc[2], acc[3]);
                        else *(float2*)dp = make_float2(acc[0], acc[1]);
                    } else {
#pragma unroll
                        for (int c = 0; c < CW; c++) if (gx + c < p.W) dp[c] = acc[c];
                    }
                    if constexpr (sizeof(ST) == 4) {
                        if (p.has_dog) {
                            const float* ctr = (const float*)s_in + (q * R + o + RB) * SF_IW + RA + cg * CW;
                            float* gp = p.dog.row<float>(f, gy) + gx;
                            if (gvec && gx + CW <= p.W) {
                                if constexpr (CW == 4)
                                    *(float4*)gp = make_float4(__fsub_rn(acc[0], ctr[0]), __fsub_rn(acc[1], ctr[1]), __fsub_rn(acc[2], ctr[2]), __fsub_rn(acc[3], ctr[3]));
                                else *(float2*)gp = make_float2(__fsub_rn(acc[0], ctr[0]), __fsub_rn(acc[1], ctr[1]));
                            } else {
#pragma unroll
                                for (int c = 0; c < CW; c++) if (gx + c < p.W) gp[c] = __fsub_rn(acc[c], ctr[c]);
                            }
                        }
                    }
                }
            }
        }
    }
}

template <int KB, typename ST, typename DT, bool SKIP0>
static int launch_sf32_tile(const CUtensorMap& tm, const Img& d, const SF32Params& p, int frames, cudaStream_t st)
{
    constexpr int IH = SF_TH + KB - 1;
    const size_t smem = (((size_t)IH * SF_IW * sizeof(ST) + 127) & ~(size_t)127) + (size_t)IH * SF_TW * sizeof(float);
    auto kern = sep_f32_tile_kernel<KB, ST, DT, SKIP0>;
    static PerDeviceFlag attr_pd; bool& attr = attr_pd.cur();
    if (!attr) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
    dim3 grid(div_up((unsigned)p.W, SF_TW), div_up((unsigned)p.H, SF_TH), (unsigned)frames);
    kern<<<grid, 256, smem, st>>>(tm, d, p);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}


// Kernels of 13 taps and more WALK DOWN a column strip (p.nch chunks of SF_TH output rows per CTA): the SF_TH + KB - 1 row-filtered rows behind
// a chunk stay in shared memory, the last KB - 1 of them move to the top for the next chunk (a 20-word copy per thread), and every chunk after
// the first stages and row-filters only its SF_TH new source rows -- the plain tile kernel filtered SF_TH + KB - 1 rows for SF_TH outputs
// (1.9x the row-pass work at 27 taps).  The next chunk's TMA load is issued
// right after the row pass and lands during the column pass.  Rows above / below the image (mirroring borders): the row filter commutes
// with the vertical mirror, so those filtered rows are copies of the mirrored rows' filtered rows.
template <int KB, typename ST, typename DT, bool SKIP0>
__global__ void __launch_bounds__(256, (KB <= 11 ? 3 : 2)) sep_f32_tma_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_tail, Img src, Img dst,
                                                                              const __grid_constant__ SF32Params p)
{
    constexpr int RB = KB / 2;
    constexpr int RA = sizeof(ST) == 1 ? 16 : ((RB + 3) / 4) * 4;   // left apron staged: TMA needs the box to start on a 16-byte boundary
    constexpr int OFF = RA - RB;
    constexpr int IH = SF_TH + KB - 1;                    // ring rows = source rows behind one chunk of outputs
    constexpr bool MARCH = KB >= 13;                      // tmap boxes: SF_TH rows (MARCH; tmap_tail: KB - 1 rows) or the whole IH-row tile
    const int nch = MARCH ? p.nch : 1;                    // up to 11 taps: the plain tile kernel (3 CTAs per SM at 80 registers: no room for the walk's state)
    extern __shared__ __align__(128) unsigned char smem_raw[];
    ST* s_in = (ST*)smem_raw;                             // IH x SF_IW
    float* s_mid = (float*)(smem_raw + (((size_t)IH * SF_IW * sizeof(ST) + 127) & ~(size_t)127));    // IH x SF_TW: row r = strip-relative source row SF_TH * ch + r
    __shared__ __align__(8) uint64_t s_bar;
    const int f = blockIdx.z, x0 = blockIdx.x * SF_TW, y00 = blockIdx.y * (SF_TH * nch);
    const int tid = threadIdx.x;
    const int tx0 = x0 - RA;
    if (tid == 0) {
        mbar_init(&s_bar, 1);
        fence_barrier_init();
        mbar_arrive_expect_tx(&s_bar, (uint32_t)(SF_IW * IH * sizeof(ST)));
        tma_load_3d(s_in, &tmap, tx0, y00 - RB, f, &s_bar);
        if constexpr (MARCH) tma_load_3d(s_in + SF_TH * SF_IW, &tmap_tail, tx0, y00 - RB + SF_TH, f, &s_bar);       // the first chunk: SF_TH + (KB - 1) rows
    }
#pragma unroll 1
  for (int ch = 0; ch < nch; ch++) {
    const int y0 = y00 + ch * SF_TH;
    if (y0 >= p.H) break;
    const int mrow0 = ch == 0 ? 0 : KB - 1;                         // first filtered row this chunk produces (rows above it come from the previous chunk)
    const int nrows = ch == 0 ? IH : SF_TH;
    if (ch > 0) {
        // the previous chunk's last KB - 1 filtered rows are this chunk's first (the barrier that ended its column pass is behind us)
        for (int idx = tid; idx < (KB - 1) * (SF_TW / 4); idx += 256) ((float4*)s_mid)[idx] = ((const float4*)(s_mid + SF_TH * SF_TW))[idx];
    }
    // only thread 0 polls the barrier; the others sleep in bar.sync instead of spending issue slots on a spin loop
    if (tid == 0) mbar_wait(&s_bar, (uint32_t)(ch & 1));
    __syncthreads();

    if (p.border != B200CV_BORDER_CONSTANT && (tx0 < 0 || tx0 + SF_IW > p.W)) {
        const int c_first = p.W - tx0;                        // first tile column right of the image (may be >= SF_IW)
        const int nright = c_first < SF_IW ? min(SF_IW - c_first, RB + 4) : 0;
        const int nleft = tx0 < 0 ? RA : 0;
        const int ncol = nleft + nright;
        for (int idx = tid; idx < nrows * ncol; idx += 256) {
            int r = idx / ncol, k = idx - r * ncol;
            int c = k < nleft ? k : c_first + (k - nleft);
            int sc = border_interpolate(tx0 + c, p.W, p.border) - tx0;
            if ((unsigned)sc < (unsigned)SF_IW) s_in[r * SF_IW + c] = s_in[r * SF_IW + sc];
        }
        __syncthreads();
    }

    // ---- row pass: item = NO consecutive outputs of one staged row.  Float rows: NO = 4, so that neighbouring lanes read neighbouring
    //      16-byte chunks (8 outputs = 32-byte lane stride made every 128-bit shared load a 2-way bank conflict); byte rows: NO = 8 ----
    {
        constexpr int NO = sizeof(ST) == 4 ? 4 : 8;
        constexpr int GPR = SF_TW / NO;                   // items per row
        constexpr int NEED = NO + KB - 1;
        constexpr int NV = (OFF + NEED + 3) / 4;
#pragma unroll 1
        for (int it = tid; it < nrows * GPR; it += 256) {
            const int r = it / GPR, g = it - r * GPR;
            float win[NV * 4];                            // the item's window (+ alignment slack), all indices compile-time
#pragma unroll
            for (int w = 0; w < NV; w++) {
                if constexpr (sizeof(ST) == 1) {
                    // bytes -> floats through the mantissa of 2^23 (PRMT + FADD instead of the quarter-rate I2F)
                    const uint32_t q = ((const uint32_t*)(s_in + r * SF_IW + g * NO))[w];
#pragma unroll
                    for (int b = 0; b < 4; b++) win[w * 4 + b] = __fsub_rn(__uint_as_float(__byte_perm(q, 0x4B000000u, 0x7650 + b)), 8388608.0f);
                } else {
                    const float4 q = ((const float4*)(s_in + r * SF_IW + g * NO))[w];
                    win[w * 4] = q.x; win[w * 4 + 1] = q.y; win[w * 4 + 2] = q.z; win[w * 4 + 3] = q.w;
                }
            }
            float acc[NO];
            bool done = false;
            if constexpr (KB <= 5 && sizeof(ST) == 4) {
                if (p.row_small) {
                    const unsigned sg = p.row_small == 2 ? 0x80000000u : 0u;
#pragma unroll
                    for (int o = 0; o < NO; o++) {
                        const float* x = win + OFF + o + RB;      // centre tap
                        // symmetric: fma(x0, k0, (x-1 + x1) k1); antisymmetric: (x1 - x-1) k1, no centre term (SKIP0; fma(x0, 0, t) = t for finite x0)
                        float t = __fmul_rn(__fadd_rn(x[1], __uint_as_float(__float_as_uint(x[-1]) ^ sg)), p.kx[RB + 1]);
                        if (!SKIP0 || p.row_small != 2) t = fmaf(x[0], p.kx[RB], t);
                        if constexpr (KB == 5) if (!SKIP0 || !p.px) t = fmaf(__fadd_rn(x[2], __uint_as_float(__float_as_uint(x[-2]) ^ sg)), p.kx[RB + 2], t);
                        acc[o] = t;
                    }
                    done = true;
                }
            }
            if (!done) {
#pragma unroll
                for (int o = 0; o < NO; o++) {
                    float t = 0.f;
#pragma unroll
                    for (int i = 0; i < KB; i++)
                        if (!SKIP0 || (i >= p.px && i < KB - p.px)) t = fmaf(win[OFF + o + i], p.kx[i], t);
                    acc[o] = t;
                }
            }
            float4* mp = (float4*)(s_mid + (mrow0 + r) * SF_TW + g * NO);
            mp[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
            if constexpr (NO == 8) mp[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
        }
    }
    __syncthreads();
    // the staging buffer is free: the next chunk's source rows land during the column pass
    if (tid == 0 && ch + 1 < nch && y0 + SF_TH < p.H) {
        fence_proxy_async();
        mbar_arrive_expect_tx(&s_bar, (uint32_t)(SF_IW * SF_TH * sizeof(ST)));
        tma_load_3d(s_in, &tmap, tx0, y00 - RB + IH + SF_TH * ch, f, &s_bar);
    }
    {
        // filtered rows of this chunk whose source row lies above / below the image = the filtered row of the mirrored source row (in this
        // window: at most KB - 1 rows away, and already filtered)
        const int g0 = y00 - RB + SF_TH * ch;                         // image row of the window's first row
        if (p.border != B200CV_BORDER_CONSTANT && (g0 + mrow0 < 0 || g0 + IH > p.H)) {
            for (int idx = tid; idx < nrows * (SF_TW / 4); idx += 256) {
                const int r = mrow0 + idx / (SF_TW / 4), c4 = idx % (SF_TW / 4);
                const int gy = g0 + r;
                if ((unsigned)gy < (unsigned)p.H) continue;
                const int sr = border_interpolate(gy, p.H, p.border) - g0;      // window row of the mirrored source row
                if (sr < 0 || sr >= IH) continue;                               // outside the window: feeds no valid output
                ((float4*)(s_mid + r * SF_TW))[c4] = ((const float4*)(s_mid + sr * SF_TW))[c4];
            }
            __syncthreads();
        }
    }

    // ---- column pass: item = CW columns x R rows; the R + KB - 1 mid rows it needs are held in registers ----
    {
        constexpr int CW = KB <= 15 ? 4 : 2, R = KB == 11 ? 4 : 8;   // window: (R + KB - 1) x CW registers, sized for 3 (KB <= 11) or 2 CTAs per SM
        constexpr int IPR = SF_TW / CW;                   // items per row group
        const bool dvec = (((uintptr_t)dst.data | dst.step | dst.fstep) & (CW * sizeof(DT) - 1)) == 0;
        const bool gvec = p.has_dog && (((uintptr_t)p.dog.data | p.dog.step | p.dog.fstep) & (CW * 4 - 1)) == 0;
#pragma unroll 1
        for (int it = tid; it < IPR * (SF_TH / R); it += 256) {
            const int q = it / IPR, cg = it - q * IPR;
            const float* mbase = s_mid + (q * R) * SF_TW + cg * CW;
            float win[R + KB - 1][CW];
#pragma unroll
            for (int m = 0; m < R + KB - 1; m++) {
                if constexpr (CW == 4) {
                    const float4 v = *(const float4*)(mbase + m * SF_TW);
                    win[m][0] = v.x; win[m][1] = v.y; win[m][2] = v.z; win[m][3] = v.w;
                } else {
                    const float2 v = *(const float2*)(mbase + m * SF_TW);
                    win[m][0] = v.x; win[m][1] = v.y;
                }
            }
            const int gx = x0 + cg * CW;
            if (gx >= p.W) continue;
#pragma unroll
            for (int o = 0; o < R; o++) {
                const int gy = y0 + q * R + o;
                if (gy >= p.H) break;
                // difference of Gaussians: the centre value (the blur's own input).  The plain tile kernel still has it staged; a walking CTA staged
                // it a chunk ago (the buffer is being refilled): from global memory (L2), loaded BEFORE the FMA chains so the latency hides behind them
                float ctr[CW] = {};
                if constexpr (sizeof(ST) == 4) {
                    if (p.has_dog) {
                        if (nch == 1) {
                            const float* cp = (const float*)s_in + (q * R + o + RB) * SF_IW + RA + cg * CW;
#pragma unroll
                            for (int c = 0; c < CW; c++) ctr[c] = cp[c];
                        } else {
                            const float* cp = src.row<float>(f, gy) + gx;
                            if (gx + CW <= p.W) {            // 16-byte aligned rows (TMA requirement), gx a multiple of CW
                                if constexpr (CW == 4) { const float4 v = __ldg((const float4*)cp); ctr[0] = v.x; ctr[1] = v.y; ctr[2] = v.z; ctr[3] = v.w; }
                                else { const float2 v = __ldg((const float2*)cp); ctr[0] = v.x; ctr[1] = v.y; }
                            } else {
#pragma unroll
                                for (int c = 0; c < CW; c++) if (gx + c < p.W) ctr[c] = cp[c];
                            }
                        }
                    }
                }
                float acc[CW];
#pragma unroll
                for (int c = 0; c < CW; c++) {
                    float t = (SKIP0 && p.col_sign) ? p.delta : fmaf(p.ky[RB], win[o + RB][c], p.delta);   // antisymmetric: no centre row
#pragma unroll
                    for (int k = 1; k <= RB; k++)
                        if (!SKIP0 || k <= RB - p.py)
                            t = fmaf(p.ky[RB + k], __fadd_rn(win[o + RB + k][c], __uint_as_float(__float_as_uint(win[o + RB - k][c]) ^ p.col_sign)), t);
                    acc[c] = t;
                }
                if constexpr (sizeof(DT) == 1) {
                    uchar* dp = dst.row<uchar>(f, gy) + gx;
                    uint32_t pk = 0;
#pragma unroll
                    for (int c = 0; c < CW; c++) pk |= (uint32_t)sat_u8(acc[c]) << (8 * c);
                    if (dvec && gx + CW <= p.W) {
                        if constexpr (CW == 4) *(uint32_t*)dp = pk; else *(unsigned short*)dp = (unsigned short)pk;
                    } else {
#pragma unroll
                        for (int c = 0; c < CW; c++) if (gx + c < p.W) dp[c] = (uchar)(pk >> (8 * c));
                    }
                } else {
                    float* dp = dst.row<float>(f, gy) + gx;
                    if (dvec && gx + CW <= p.W) {
                        if constexpr (CW == 4) *(float4*)dp = make_float4(acc[0], acc[1], acc[2], acc[3]);
                        else *(float2*)dp = make_float2(acc[0], acc[1]);
                    } else {
#pragma unroll
                        for (int c = 0; c < CW; c++) if (gx + c < p.W) dp[c] = acc[c];
                    }
                    if constexpr (sizeof(ST) == 4) {
                        if (p.has_dog) {
                            float* gp = p.dog.row<float>(f, gy) + gx;
                            if (gvec && gx + CW <= p.W) {
                                if constexpr (CW == 4)
                                    *(float4*)gp = make_float4(__fsub_rn(acc[0], ctr[0]), __fsub_rn(acc[1], ctr[1]), __fsub_rn(acc[2], ctr[2]), __fsub_rn(acc[3], ctr[3]));
                                else *(float2*)gp = make_float2(__fsub_rn(acc[0], ctr[0]), __fsub_rn(acc[1], ctr[1]));
                            } else {
#pragma unroll
                                for (int c = 0; c < CW; c++) if (gx + c < p.W) gp[c] = __fsub_rn(acc[c], ctr[c]);
                            }
                        }
                    }
                }
            }
        }
    }
    __syncthreads();            // the next chunk moves and overwrites filtered rows this column pass has read
  }
}

template <int KB, typename ST, typename DT, bool SKIP0>
static int launch_sf32(const CUtensorMap& tm, const CUtensorMap& tm_tail, const Img& s, const Img& d, SF32Params& p, int frames, cudaStream_t st)
{
    constexpr int IH = SF_TH + KB - 1;
    const size_t smem = (((size_t)IH * SF_IW * sizeof(ST) + 127) & ~(size_t)127) + (size_t)IH * SF_TW * sizeof(float);
    // chunks per CTA: 4 (128 rows) for 13 taps and more when the grid stays several waves deep; small kernels keep the plain tile form
    const long tiles = (long)div_up((unsigned)p.W, SF_TW) * div_up((unsigned)p.H, SF_TH) * frames;
    p.nch = (KB >= 13 && tiles >= 8L * 2 * num_sms()) ? 4 : (KB >= 13 && tiles >= 4L * 2 * num_sms()) ? 2 : 1;
    auto kern = sep_f32_tma_kernel<KB, ST, DT, SKIP0>;
    static PerDeviceFlag attr_pd; bool& attr = attr_pd.cur();
    if (!attr) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
    dim3 grid(div_up((unsigned)p.W, SF_TW), div_up((unsigned)p.H, (unsigned)(SF_TH * p.nch)), (unsigned)frames);
    kern<<<grid, 256, smem, st>>>(tm, tm_tail, s, d, p);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

// 1: k[i] == k[n-1-i] for all i, 2: k[i] == -k[n-1-i], 0: neither (reference: getKernelType, filter.dispatch.cpp:225-259)
static int symmetry_of(const float* k, int n)
{
    bool sy = true, as = true;
    for (int i = 0; i < n; i++) { if (k[i] != k[n - 1 - i]) sy = false; if (k[i] != -k[n - 1 - i]) as = false; }
    return sy ? 1 : as ? 2 : 0;
}

template <typename ST, typename DT, bool SKIP0>
static int launch_kb(int KB, const CUtensorMap& tm, const CUtensorMap& tm_tail, const Img& s, const Img& d, SF32Params& p, cudaStream_t st);

template <typename ST, typename DT>
static int sep_float_fast(const Img& s, const Img& d, const float* kx, int nx, const float* ky, int ny, float delta, int border, const Img* dog, cudaStream_t st)
{
    if (!(nx & 1) || !(ny & 1) || nx > 31 || ny > 31) return B200CV_NOT_IMPLEMENTED;
    const int csym = symmetry_of(ky, ny);
    if (!csym) return B200CV_NOT_IMPLEMENTED;                       // scalar ColumnFilter order: generic kernel
    const int rsym = (sizeof(ST) == 4 && nx <= 5 && nx >= 3) ? symmetry_of(kx, nx) : 0;
    if (rsym && (nx > ny ? nx : ny) > 5) return B200CV_NOT_IMPLEMENTED;   // small-row order inside a wide bucket: generic kernel
    if (border == B200CV_BORDER_WRAP || !tma_compatible(s) || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    static const int buckets[] = {3, 5, 7, 9, 11, 13, 15, 17, 21, 25, 27, 31};
    int kmax = nx > ny ? nx : ny, KB = 0;
    for (int b : buckets) if (kmax <= b) { KB = b; break; }
    if (!KB || s.cols < KB || s.rows < KB) return B200CV_NOT_IMPLEMENTED;
    SF32Params p;
    memset(&p, 0, sizeof(p));
    for (int i = 0; i < nx; i++) p.kx[(KB - nx) / 2 + i] = kx[i];
    for (int i = 0; i < ny; i++) p.ky[(KB - ny) / 2 + i] = ky[i];
    p.delta = delta; p.W = s.cols; p.H = s.rows; p.border = border;
    p.row_small = rsym; p.col_sign = csym == 2 ? 0x80000000u : 0u;
    p.px = (KB - nx) / 2; p.py = (KB - ny) / 2;
    if (dog) { p.dog = *dog; p.has_dog = 1; }
    CUtensorMap tm, tm_tail;
    const bool march = KB >= 13;
    int rc = make_tensor_map_3d(&tm, s.data, (int)sizeof(ST), s.cols, s.rows, s.frames, s.step, s.fstep, SF_IW, march ? SF_TH : SF_TH + KB - 1);
    if (rc) return rc;
    if ((rc = make_tensor_map_3d(&tm_tail, s.data, (int)sizeof(ST), s.cols, s.rows, s.frames, s.step, s.fstep, SF_IW, KB - 1))) return rc;
    if (sizeof(ST) == 4 && (p.px || p.py || rsym == 2 || csym == 2)) return launch_kb<ST, DT, true>(KB, tm, tm_tail, s, d, p, st);
    return launch_kb<ST, DT, false>(KB, tm, tm_tail, s, d, p, st);
}

template <typename ST, typename DT, bool SKIP0>
static int launch_kb(int KB, const CUtensorMap& tm, const CUtensorMap& tm_tail, const Img& s, const Img& d, SF32Params& p, cudaStream_t st)
{
    switch (KB) {
    case 3: return launch_sf32_tile<3, ST, DT, SKIP0>(tm, d, p, s.frames, st);
    case 5: return launch_sf32_tile<5, ST, DT, SKIP0>(tm, d, p, s.frames, st);
    case 7: return launch_sf32_tile<7, ST, DT, SKIP0>(tm, d, p, s.frames, st);
    case 9: return launch_sf32_tile<9, ST, DT, SKIP0>(tm, d, p, s.frames, st);
    case 11: return launch_sf32_tile<11, ST, DT, SKIP0>(tm, d, p, s.frames, st);
    case 13: return launch_sf32<13, ST, DT, SKIP0>(tm, tm_tail, s, d, p, s.frames, st);
    case 15: return launch_sf32<15, ST, DT, SKIP0>(tm, tm_tail, s, d, p, s.frames, st);
    case 17: return launch_sf32<17, ST, DT, SKIP0>(tm, tm_tail, s, d, p, s.frames, st);
    case 21: return launch_sf32<21, ST, DT, SKIP0>(tm, tm_tail, s, d, p, s.frames, st);
    case 25: return launch_sf32<25, ST, DT, SKIP0>(tm, tm_tail, s, d, p, s.frames, st);
    case 27: return launch_sf32<27, ST, DT, SKIP0>(tm, tm_tail, s, d, p, s.frames, st);
    case 31: return launch_sf32<31, ST, DT, SKIP0>(tm, tm_tail, s, d, p, s.frames, st);
    }
    return B200CV_NOT_IMPLEMENTED;
}

// return B200CV_NOT_IMPLEMENTED when the fast path does not apply
int sep_f32_fast(const Img& s, const Img& d, const float* kx, int nx, const float* ky, int ny, float delta, int border, const Img* dog, cudaStream_t st)
{
    return sep_float_fast<float, float>(s, d, kx, nx, ky, ny, delta, border, dog, st);
}

int sep_u8_float_fast(const Img& s, const Img& d, const float* kx, int nx, const float* ky, int ny, float delta, int border, cudaStream_t st)
{
    return sep_float_fast<uchar, uchar>(s, d, kx, nx, ky, ny, delta, border, nullptr, st);
}

}  // namespace b200cv
