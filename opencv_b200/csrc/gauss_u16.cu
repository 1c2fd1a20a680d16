// gauss_u16.cu -- cv::GaussianBlur for CV_16U images ("u8 / u16: integer 8.8 / 16.16 fixed point, bit-exact").
//
// Reference: fixedSmoothInvoker<uint16_t, ufixedpoint32> (smooth.simd.hpp:1925-2197), taps getGaussianKernelFixedPoint_ED with 16 fractional
// bits (smooth.dispatch.cpp:224-258), arithmetic fixedpoint.inl.hpp (ufixedpoint32 / ufixedpoint64):
//   rows      H = sum tap_x * p     32-bit unsigned, products and sums saturate at 2^32 - 1 (the taps sum to 2^16, so real taps never saturate)
//   columns   V = sum tap_y * H     64-bit unsigned (32.32), saturating adds;   result = min((V + 2^31) >> 32, 65535)
// Bit-exact for every border mode the reference's engine accepts; BORDER_CONSTANT pads with zeros.  Up to 33 x 33 taps.
// Separable and tiled: a CTA stages the source tile + apron once in shared memory (border rule applied per staged element, pixels of CN
// interleaved channels), row-filters every staged row ONCE into a 32-bit tile, then column-filters: kw + kh multiply-adds per element
// instead of kw * kh, and every source element is fetched once per tile instead of kw * kh times through L1.
#include "common.cuh"

namespace b200cv {

namespace {

constexpr int GS_TE = 128, GS_TH = 32;          // tile: elements (pixels x channels) per row, rows

// dynamic shared memory of one CTA: the staged 16-bit tile + apron (16-byte aligned), then the 32-bit row-filtered tile
constexpr size_t gs_smem_bytes(int kw, int kh, int cn)
{
    return (((size_t)(GS_TH + 2 * (kh / 2)) * (GS_TE + 2 * (kw / 2) * cn) * 2 + 15) & ~(size_t)15) + (size_t)(GS_TH + 2 * (kh / 2)) * GS_TE * 4;
}
static_assert(gs_smem_bytes(33, 33, 4) <= 96 * 1024, "the largest kernel (33 x 33 taps, 4 channels) must fit the 96 KB opt-in");

struct U16SepTaps { unsigned kx[33], ky[33]; int nx, ny; };

template <int CN>
__global__ void __launch_bounds__(256) gauss_u16_sep_kernel(Img src, Img dst, int W, int H, const __grid_constant__ U16SepTaps t, int border)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int rx = t.nx / 2, ry = t.ny / 2;
    const int SW = GS_TE + 2 * rx * CN, SH = GS_TH + 2 * ry;          // staged elements per row, rows
    unsigned short* s_in = (unsigned short*)smem;                       // SH x SW
    unsigned* s_mid = (unsigned*)(smem + (((size_t)SH * SW * 2 + 15) & ~(size_t)15));   // SH x GS_TE
    const int e0 = blockIdx.x * GS_TE, y0 = blockIdx.y * GS_TH, f = blockIdx.z;
    const int WE = W * CN;
    // ---- stage: element (r, k) = source element e0 - rx * CN + k of row y0 - ry + r under the border rule (per PIXEL) ----
    for (int idx = threadIdx.x; idx < SH * SW; idx += 256) {
        const int r = idx / SW, k = idx - r * SW;
        const int sy = border_interpolate(y0 - ry + r, H, border);
        const int ge = e0 - rx * CN + k;                              // element index in the row, may be outside
        int px = ge >= 0 ? ge / CN : -((-ge + CN - 1) / CN);
        const int c = ge - px * CN;
        px = border_interpolate(px, W, border);
        s_in[idx] = (sy >= 0 && px >= 0) ? src.row<unsigned short>(f, sy)[px * CN + c] : (unsigned short)0;
    }
    __syncthreads();
    // ---- rows: 32-bit saturating (products and sums) ----
    for (int idx = threadIdx.x; idx < SH * GS_TE; idx += 256) {
        const int r = idx / GS_TE, k = idx - r * GS_TE;
        const unsigned short* p = s_in + r * SW + k;
        unsigned long long line = 0;
        for (int i = 0; i < t.nx; i++) {
            unsigned long long pr = (unsigned long long)t.kx[i] * p[i * CN];
            pr = min(pr, 0xFFFFFFFFull);
            line = min(line + pr, 0xFFFFFFFFull);
        }
        s_mid[idx] = (unsigned)line;
    }
    __syncthreads();
    // ---- columns: 64-bit saturating adds; rows outside a CONSTANT border were staged as zeros, and a zero line adds nothing ----
    for (int idx = threadIdx.x; idx < GS_TH * GS_TE; idx += 256) {
        const int r = idx / GS_TE, k = idx - r * GS_TE;
        const int y = y0 + r, e = e0 + k;
        if (y >= H || e >= WE) continue;
        unsigned long long acc = 0;
        for (int j = 0; j < t.ny; j++) {
            const unsigned long long pr = (unsigned long long)t.ky[j] * s_mid[(r + j) * GS_TE + k], s = acc + pr;
            acc = s < acc ? ~0ull : s;
        }
        const unsigned long long v = (acc + (1ull << 31)) >> 32;
        dst.row<unsigned short>(f, y)[e] = (unsigned short)min(v, 65535ull);
    }
}

}  // namespace

// fx / fy: the 16.16 fixed-point taps (host); src / dst: 16UC1/3/4 of equal size and batch, distinct buffers
int gauss_u16_impl(const Img& s, const Img& d, int cn, const long long* fx, int kw, const long long* fy, int kh, int border, cudaStream_t st)
{
    if (kw > 33 || kh > 33 || (cn != 1 && cn != 3 && cn != 4) || s.rows >= 65536 * GS_TH || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    U16SepTaps t;
    t.nx = kw; t.ny = kh;
    for (int i = 0; i < 33; i++) { t.kx[i] = i < kw ? (unsigned)fx[i] : 0u; t.ky[i] = i < kh ? (unsigned)fy[i] : 0u; }
    const size_t smem = gs_smem_bytes(kw, kh, cn);
    const dim3 grid(div_up((unsigned)(s.cols * cn), GS_TE), div_up((unsigned)s.rows, GS_TH), (unsigned)s.frames);
    static PerDeviceFlag a_pd; bool& a = a_pd.cur();
    if (!a) {
        B200_CUDA(cudaFuncSetAttribute(gauss_u16_sep_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        B200_CUDA(cudaFuncSetAttribute(gauss_u16_sep_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        B200_CUDA(cudaFuncSetAttribute(gauss_u16_sep_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        a = true;
    }
    if (cn == 1) gauss_u16_sep_kernel<1><<<grid, 256, smem, st>>>(s, d, s.cols, s.rows, t, border);
    else if (cn == 3) gauss_u16_sep_kernel<3><<<grid, 256, smem, st>>>(s, d, s.cols, s.rows, t, border);
    else gauss_u16_sep_kernel<4><<<grid, 256, smem, st>>>(s, d, s.cols, s.rows, t, border);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace b200cv
