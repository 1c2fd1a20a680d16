// gauss_u8_binomial.cu -- cv::GaussianBlur on 8-bit single-channel images for the two kernels almost every caller uses: 3 x 3 and 5 x 5 with
// sigma = 0, whose 8.8 fixed-point taps are the binomial rows {64, 128, 64} and {16, 64, 96, 64, 16} (smooth.dispatch.cpp:87-146, 224-258).
//
// Reference arithmetic (fixedSmoothInvoker<uint8_t, ufixedpoint16>, smooth.simd.hpp:1925-2197): rows in 8.8, columns in 16.16,
//   dst = (sum_j ky[j] * sum_i kx[i] * src + 32768) >> 16,  no intermediate saturation (the taps add up to 256).
// With kx = ky = 64 * {1, 2, 1} this is exactly (B + 8) >> 4, B = the 3 x 3 binomial sum (<= 16 * 255); with 16 * {1, 4, 6, 4, 1} it is
// (B + 128) >> 8, B <= 256 * 255 -- both fit 16 bits, rounding constant included.  So two pixels ride in one 32-bit register as 16-bit halves
// and the whole filter is adds and shifts on the integer pipes, with no multiplier in the loop:
//   IDP4A / IDP2A issue at half rate on the FMA-heavy pipe; the general tile kernel (gauss_u8.cu) spends ~3.5 of the ~11 issue slots per pixel that
//   the HBM roofline leaves on them alone, and is instruction-issue bound at 3 x 3.
// A thread owns 16 adjacent columns (one 128-bit load per row) and walks down GB_SEG output rows: per word E / O = even / odd pixels as halves, the
// shifted pairs by PRMT, row sums for the even and the odd pixels; the last K - 1 row sums stay in registers (ring resolved at compile time by
// unrolling); column sums, rounding, one PRMT to bytes per word, one 128-bit store.  Rows outside the image are fetched from the reflected row
// (or are zero for BORDER_CONSTANT, which contributes zero here: smooth.simd.hpp:963-995).  Widths that are not multiples of 16 and unaligned
// rows stay on the tile kernel.
#include <cstdlib>
#include <cstring>
#include "common.cuh"

namespace b200cv {

namespace {

constexpr int GB_SEG = 64;      // output rows per thread

// row sums of the even (pixels 0, 2) and odd (pixels 1, 3) columns of word w0 as 16-bit halves; wl / wr = the words left and right of it
template <int K>
__device__ __forceinline__ void gb_row(unsigned wl, unsigned w0, unsigned wr, unsigned& he, unsigned& ho)
{
    const unsigned E = __byte_perm(w0, 0u, 0x4240), O = __byte_perm(w0, 0u, 0x4341);       // (b0, b2), (b1, b3)
    const unsigned Om1 = __byte_perm(wl, O, 0x5453);                                          // (b-1, b1)
    const unsigned Ep1 = __byte_perm(E, wr, 0x1412);                                          // (b2, b4)
    if constexpr (K == 3) {
        he = Om1 + O + 2u * E;
        ho = E + Ep1 + 2u * O;
    } else {
        const unsigned Em1 = __byte_perm(wl, E, 0x5452);                                      // (b-2, b0)
        const unsigned Op1 = __byte_perm(O, wr, 0x1512);                                      // (b3, b5)
        he = (Em1 + Ep1) + 4u * (Om1 + O) + 6u * E;
        ho = (Om1 + Op1) + 4u * (E + Ep1) + 6u * O;
    }
}

struct GbBorder { unsigned sel_l, sel_r; int zero; };     // PRMT selectors that build the two halo bytes from the row's own first / last word

constexpr int GB_DEPTH = 8;     // rows of copies in flight per thread (a power of two)

__device__ __forceinline__ void gb_cp16(void* smem, const void* g, int src_bytes, unsigned dep)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(g), "r"(src_bytes), "r"(dep) : "memory");
}
__device__ __forceinline__ void gb_cp4(void* smem, const void* g, int src_bytes)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(g), "r"(src_bytes) : "memory");
}

// A thread owns 16 adjacent columns and walks down GB_SEG rows.  Its rows arrive through a lane-private ring in shared memory filled by cp.async
// (one 16-byte copy per row and lane = 512 contiguous bytes per warp and row, GB_DEPTH rows in flight, no registers held by loads in flight: with
// loads into registers the kernel was latency bound).  Nothing in the ring is shared
// between lanes, so cp.async.wait_group is the only synchronisation.  The word left of the thread's first and right of its last word come from the
// neighbouring lanes by shuffle; lanes 0 and 31 copy theirs; at the image edges they are built from the row's own bytes by the border rule.
template <int K, bool FAST>
__device__ __forceinline__ void gb_walk(const Img& src, const Img& dst, int border, GbBorder gb, int x0, int y0, int y1, int f, bool active, int lane,
                                        uint4* ring, unsigned* ering)
{
    constexpr int R = K / 2, D = GB_DEPTH;
    const int W = src.cols, H = src.rows, tid = threadIdx.x;
    auto row_ptr = [&](int r) -> const uchar* {
        const int sr = (unsigned)r < (unsigned)H ? r : border_interpolate(r, H, border);
        return sr < 0 ? nullptr : src.row<uchar>(f, sr);
    };
    const bool first = x0 == 0, last = x0 + 16 == W;
    const int ew_off = lane == 0 ? -4 : 16;                                   // the extra word lanes 0 / 31 copy themselves
    const bool ew_lane = lane == 0 || lane == 31;
    const bool ew_need = active && ((lane == 0 && !first) || (lane == 31 && !last));
    const uchar* qf = FAST ? src.row<uchar>(f, y0 - R) + x0 : nullptr;
    const int N = (y1 - y0) + K - 1;
    int issued = 0;                                                           // input rows requested so far (image row y0 - R + issued is next)
    auto issue = [&](unsigned dep) {
        if (issued < N) {
            const uchar* rp = FAST ? qf : row_ptr(y0 - R + issued);
            const bool have = rp != nullptr;
            const uchar* g = have ? (FAST ? rp : rp + x0) : src.data;
            const int slot = issued & (D - 1);
            gb_cp16(&ring[slot * 128 + tid], g, have && active ? 16 : 0, dep);      // 0 source bytes = zero fill (rows of a BORDER_CONSTANT frame, idle lanes)
            if (ew_lane) gb_cp4(&ering[slot * 128 + tid], have && ew_need ? g + ew_off : src.data, have && ew_need ? 4 : 0);
            if (FAST) qf += src.step;
        }
        asm volatile("cp.async.commit_group;" ::: "memory");                  // an (empty) group per call keeps the wait count uniform at the tail
        issued++;
    };
#pragma unroll
    for (int u = 0; u < D; u++) issue(0u);
    unsigned he[K][4], ho[K][4];
    uchar* dp = dst.row<uchar>(f, y0) + x0;
    for (int base = 0; base < N; base += K) {
#pragma unroll
        for (int u = 0; u < K; u++) {
            const int i = base + u;
            if (i < N) {
                asm volatile("cp.async.wait_group %0;" ::"n"(D - 1) : "memory");
                const int slot = i & (D - 1);
                const uint4 v = ring[slot * 128 + tid];
                const unsigned e = ew_lane ? ering[slot * 128 + tid] : 0u;
                unsigned hl = __shfl_up_sync(0xffffffffu, v.w, 1), hr = __shfl_down_sync(0xffffffffu, v.x, 1);
                if (lane == 0) hl = e;
                if (lane == 31) hr = e;
                if (first) hl = gb.zero ? 0u : __byte_perm(v.x, v.x, gb.sel_l);
                if (last) hr = gb.zero ? 0u : __byte_perm(v.w, v.w, gb.sel_r);
                gb_row<K>(hl, v.x, v.y, he[u][0], ho[u][0]);
                gb_row<K>(v.x, v.y, v.z, he[u][1], ho[u][1]);
                gb_row<K>(v.y, v.z, v.w, he[u][2], ho[u][2]);
                gb_row<K>(v.z, v.w, hr, he[u][3], ho[u][3]);
                // refill the slot just read: the copy is issued after instructions that needed the slot's data (the operand `dep` makes that explicit)
                issue(he[u][0] ^ he[u][3] ^ e);
                if (i >= K - 1) {                                   // output row y0 + i - (K - 1): input rows i - K + 1 .. i, oldest in slot (u + 1) % K
                    unsigned out[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        unsigned se, so;
                        if constexpr (K == 3) {
                            se = he[(u + 1) % K][j] + he[u][j] + 2u * he[(u + 2) % K][j] + 0x00080008u;
                            so = ho[(u + 1) % K][j] + ho[u][j] + 2u * ho[(u + 2) % K][j] + 0x00080008u;
                            out[j] = __byte_perm(se >> 4, so >> 4, 0x6240);
                        } else {
                            se = (he[(u + 1) % K][j] + he[u][j]) + 4u * (he[(u + 2) % K][j] + he[(u + 4) % K][j]) + 6u * he[(u + 3) % K][j] + 0x00800080u;
                            so = (ho[(u + 1) % K][j] + ho[u][j]) + 4u * (ho[(u + 2) % K][j] + ho[(u + 4) % K][j]) + 6u * ho[(u + 3) % K][j] + 0x00800080u;
                            out[j] = __byte_perm(se, so, 0x7351);
                        }
                    }
                    if (active) *(uint4*)dp = make_uint4(out[0], out[1], out[2], out[3]);
                    dp += dst.step;
                }
            }
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

template <int K>
__global__ void __launch_bounds__(128) gauss_u8_binomial_kernel(Img src, Img dst, int border, GbBorder gb)
{
    constexpr int R = K / 2;
    extern __shared__ __align__(16) unsigned char gb_smem[];
    uint4* ring = (uint4*)gb_smem;                                           // [GB_DEPTH][128]: lane-private row ring
    unsigned* ering = (unsigned*)(gb_smem + sizeof(uint4) * GB_DEPTH * 128);  // [GB_DEPTH][128]: the extra word of lanes 0 / 31
    const int W = src.cols, H = src.rows;
    const int x0 = (blockIdx.x * 128 + threadIdx.x) * 16, f = blockIdx.z;
    const int y0 = blockIdx.y * GB_SEG, y1 = min(y0 + GB_SEG, H);
    const int lane = threadIdx.x & 31;
    if ((blockIdx.x * 128 + (threadIdx.x & ~31)) * 16 >= W) return;            // the whole warp is past the row end
    const bool active = x0 < W;
    const int xc = active ? x0 : 0;                                            // idle lanes of the last warp take part in the shuffles only
    if (y0 - R >= 0 && y1 + R <= H) gb_walk<K, true>(src, dst, border, gb, xc, y0, y1, f, active, lane, ring, ering);
    else gb_walk<K, false>(src, dst, border, gb, xc, y0, y1, f, active, lane, ring, ering);
}

}  // namespace

// taps as 8.8 integers (what gauss_u8_fast receives); returns NOT_IMPLEMENTED when the case is not the binomial one
int gauss_u8_binomial(const Img& s, const Img& d, int cn, const int64_t* fx, int kw, const int64_t* fy, int kh, int border, cudaStream_t st)
{
    if (cn != 1 || kw != kh || (kw != 3 && kw != 5) || s.cols < 32 || (s.cols & 15) || s.rows < kw) return B200CV_NOT_IMPLEMENTED;
    static const int64_t t3[3] = {64, 128, 64}, t5[5] = {16, 64, 96, 64, 16};
    const int64_t* t = kw == 3 ? t3 : t5;
    for (int i = 0; i < kw; i++) if (fx[i] != t[i] || fy[i] != t[i]) return B200CV_NOT_IMPLEMENTED;
    if (s.rows >= 65536 * GB_SEG || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    if ((((uintptr_t)s.data | s.step | s.fstep) & 15) || (((uintptr_t)d.data | d.step | d.fstep) & 15)) return B200CV_NOT_IMPLEMENTED;   // 128-bit rows
    GbBorder gb = {0, 0, 0};
    // halo bytes (b-2, b-1) in bytes 2, 3 of the word left of the row and (bW, bW+1) in bytes 0, 1 of the word right of it, picked from the row's own
    // first / last word by cv::borderInterpolate's rule
    switch (border & ~B200CV_BORDER_ISOLATED) {
    case B200CV_BORDER_CONSTANT: gb.zero = 1; break;
    case B200CV_BORDER_REPLICATE: gb.sel_l = 0x0000; gb.sel_r = 0x0033; break;
    case B200CV_BORDER_REFLECT: gb.sel_l = 0x0100; gb.sel_r = 0x0023; break;
    case B200CV_BORDER_REFLECT_101: gb.sel_l = 0x1200; gb.sel_r = 0x0012; break;
    default: return B200CV_NOT_IMPLEMENTED;
    }
    const dim3 grid(div_up(div_up((unsigned)s.cols, 16), 128), div_up((unsigned)s.rows, GB_SEG), (unsigned)s.frames);
    const size_t smem = (sizeof(uint4) + sizeof(unsigned)) * GB_DEPTH * 128;
    if (kw == 3) gauss_u8_binomial_kernel<3><<<grid, 128, smem, st>>>(s, d, border & ~B200CV_BORDER_ISOLATED, gb);
    else gauss_u8_binomial_kernel<5><<<grid, 128, smem, st>>>(s, d, border & ~B200CV_BORDER_ISOLATED, gb);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace b200cv
