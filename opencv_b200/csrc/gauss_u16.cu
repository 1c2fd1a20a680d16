// gauss_u16.cu -- cv::GaussianBlur for CV_16U images ("u8 / u16: integer 8.8 / 16.16 fixed point, bit-exact").
//
// Reference: fixedSmoothInvoker<uint16_t, ufixedpoint32> (smooth.simd.hpp:1925-2197), taps getGaussianKernelFixedPoint_ED with 16 fractional
// bits (smooth.dispatch.cpp:224-258), arithmetic fixedpoint.inl.hpp (ufixedpoint32 / ufixedpoint64):
//   rows      H = sum tap_x * p     32-bit unsigned, products and sums saturate at 2^32 - 1 (the taps sum to 2^16, so real taps never saturate)
//   columns   V = sum tap_y * H     64-bit unsigned (32.32), saturating adds;   result = min((V + 2^31) >> 32, 65535)
// Bit-exact for every border mode the reference's engine accepts; BORDER_CONSTANT pads with zeros.
// One thread per destination element evaluating the kw x kh window directly (rows are not shared between neighbours): exact and simple, the
// shared-memory separable version is what the 8-bit path has (gauss_u8.cu) and the next step here.  Up to 33 x 33 taps.
#include "common.cuh"

namespace b200cv {

namespace {

struct U16Taps { unsigned kx[33], ky[33]; int nx, ny; };

template <int CN>
__global__ void __launch_bounds__(256) gauss_u16_kernel(Img src, Img dst, int W, int H, U16Taps t, int border)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;           // destination element x * CN + c
    const int y = blockIdx.y, f = blockIdx.z;
    if (e >= W * CN) return;
    const int x = e / CN, c = e - x * CN;
    const int rx = t.nx / 2, ry = t.ny / 2;
    unsigned long long acc = 0;
    for (int j = 0; j < t.ny; j++) {
        const int sy = border_interpolate(y + j - ry, H, border);
        if (sy < 0) continue;
        const unsigned short* row = src.row<unsigned short>(f, sy);
        unsigned long long line = 0;
        for (int i = 0; i < t.nx; i++) {
            const int sx = border_interpolate(x + i - rx, W, border);
            if (sx < 0) continue;
            unsigned long long pr = (unsigned long long)t.kx[i] * row[sx * CN + c];
            pr = min(pr, 0xFFFFFFFFull);
            line = min(line + pr, 0xFFFFFFFFull);
        }
        const unsigned long long pr = (unsigned long long)t.ky[j] * line, s = acc + pr;
        acc = s < acc ? ~0ull : s;
    }
    const unsigned long long r = (acc + (1ull << 31)) >> 32;
    dst.row<unsigned short>(f, y)[e] = (unsigned short)min(r, 65535ull);
}

}  // namespace

// fx / fy: the 16.16 fixed-point taps (host); src / dst: 16UC1/3/4 of equal size and batch, distinct buffers
int gauss_u16_impl(const Img& s, const Img& d, int cn, const long long* fx, int kw, const long long* fy, int kh, int border, cudaStream_t st)
{
    if (kw > 33 || kh > 33 || (cn != 1 && cn != 3 && cn != 4) || s.rows >= 65536 || s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    U16Taps t;
    t.nx = kw; t.ny = kh;
    for (int i = 0; i < 33; i++) { t.kx[i] = i < kw ? (unsigned)fx[i] : 0u; t.ky[i] = i < kh ? (unsigned)fy[i] : 0u; }
    const dim3 block(256);
    const dim3 grid(div_up((unsigned)(s.cols * cn), 256), (unsigned)s.rows, (unsigned)s.frames);
    if (cn == 1) gauss_u16_kernel<1><<<grid, block, 0, st>>>(s, d, s.cols, s.rows, t, border);
    else if (cn == 3) gauss_u16_kernel<3><<<grid, block, 0, st>>>(s, d, s.cols, s.rows, t, border);
    else gauss_u16_kernel<4><<<grid, block, 0, st>>>(s, d, s.cols, s.rows, t, border);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace b200cv
