// pyramid.cu -- cv::pyrDown / cv::pyrUp (the image-pyramid callers of the blur path).
//
// pyrDown (pyramids.cpp:884-1039): 5-tap [1 4 6 4 1] rows into an intermediate at every second column, the same taps over every
// second row, then a 1/256 cast; borders through cv::borderInterpolate on the SOURCE coordinates (any mode but CONSTANT).
//   8-bit:  row = 6 s[2x] + 4 (s[2x-1] + s[2x+1]) + s[2x-2] + s[2x+2]  (int);  dst = (6 r2 + 4 (r1 + r3) + r0 + r4 + 128) >> 8       bit-exact
//   float:  the operation order of the reference's 4-lane SSE bodies (pyramids.cpp:324-341, :497-516; un-fused multiply-adds):
//           row = r2*6 + ((r1 + r3)*4 + (r0 + r4));   dst = (((r1 + r3) + r2)*4 + ((r0 + r4) + (r2 + r2))) * (1/256)
//           (the reference's first / last columns and vector remainders use its scalar order: <= 1 ulp there)
// pyrUp (pyramids.cpp:1041-1155): even columns s[x-1] + 6 s[x] + s[x+1], odd columns 4 (s[x] + s[x+1]), special first / last columns;
// the same vertically (source row -1 -> 1, row H -> H-1), 1/64 cast.  8-bit bit-exact; float in the order of its bodies (:710-728).
// Only the default destination sizes ((W+1)/2 x (H+1)/2 and 2W x 2H): other sizes run a differently shifted tap table in the reference.
// One thread per destination element; every tap comes straight from global memory (L1/L2 absorb the 25-fold / 9-fold reuse).
#include "common.cuh"

namespace b200cv {

template <typename T> struct PyrAcc;
template <> struct PyrAcc<uchar> { typedef int type; };
template <> struct PyrAcc<float> { typedef float type; };

template <typename T, int CN>
__global__ void __launch_bounds__(256) pyr_down_kernel(Img src, Img dst, int border)
{
    typedef typename PyrAcc<T>::type WT;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;          // destination element (x * CN + c)
    const int y = blockIdx.y, f = blockIdx.z;
    if (e >= dst.cols * CN) return;
    const int x = e / CN, c = e - x * CN;
    int sx[5];
#pragma unroll
    for (int k = 0; k < 5; k++) sx[k] = border_interpolate(2 * x + k - 2, src.cols, border) * CN + c;
    WT r[5];
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const T* s = src.row<T>(f, border_interpolate(2 * y + j - 2, src.rows, border));
        if constexpr (sizeof(T) == 1) r[j] = s[sx[2]] * 6 + (s[sx[1]] + s[sx[3]]) * 4 + s[sx[0]] + s[sx[4]];
        else r[j] = __fadd_rn(__fmul_rn(s[sx[2]], 6.f), __fadd_rn(__fmul_rn(__fadd_rn(s[sx[1]], s[sx[3]]), 4.f), __fadd_rn(s[sx[0]], s[sx[4]])));
    }
    T out;
    if constexpr (sizeof(T) == 1) out = (uchar)((r[2] * 6 + (r[1] + r[3]) * 4 + r[0] + r[4] + 128) >> 8);
    else out = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fadd_rn(r[1], r[3]), r[2]), 4.f), __fadd_rn(__fadd_rn(r[0], r[4]), __fadd_rn(r[2], r[2]))), 1.f / 256);
    dst.row<T>(f, y)[e] = out;
}

// horizontal pyrUp value of destination column dx (channel c) in source row s
template <typename T, int CN>
__device__ __forceinline__ typename PyrAcc<T>::type pyr_up_h(const T* s, int dx, int c, int sw)
{
    typedef typename PyrAcc<T>::type WT;
    const int x = dx >> 1;
    const bool odd = dx & 1;
    if (sw == 1) return (WT)s[c] * 8;
    if (x == 0) return odd ? ((WT)s[c] + (WT)s[CN + c]) * 4 : (sizeof(T) == 1 ? (WT)s[c] * 6 + (WT)s[CN + c] * 2
                                                                           : (WT)__fadd_rn(__fmul_rn((float)s[c], 6.f), __fmul_rn((float)s[CN + c], 2.f)));
    if (x == sw - 1) {
        if (odd) return (WT)s[x * CN + c] * 8;
        return sizeof(T) == 1 ? (WT)s[(x - 1) * CN + c] + (WT)s[x * CN + c] * 7 : (WT)__fadd_rn((float)s[(x - 1) * CN + c], __fmul_rn((float)s[x * CN + c], 7.f));
    }
    if (odd) {
        if constexpr (sizeof(T) == 1) return ((WT)s[x * CN + c] + (WT)s[(x + 1) * CN + c]) * 4;
        else return __fmul_rn(__fadd_rn(s[x * CN + c], s[(x + 1) * CN + c]), 4.f);
    }
    if constexpr (sizeof(T) == 1) return (WT)s[(x - 1) * CN + c] + (WT)s[x * CN + c] * 6 + (WT)s[(x + 1) * CN + c];
    else return __fadd_rn(__fadd_rn(s[(x - 1) * CN + c], __fmul_rn(s[x * CN + c], 6.f)), s[(x + 1) * CN + c]);
}

template <typename T, int CN>
__global__ void __launch_bounds__(256) pyr_up_kernel(Img src, Img dst)
{
    typedef typename PyrAcc<T>::type WT;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int dy = blockIdx.y, f = blockIdx.z;
    if (e >= dst.cols * CN) return;
    const int dx = e / CN, c = e - dx * CN;
    const int y = dy >> 1, H = src.rows, W = src.cols;
    // ring rows of the reference: source rows y-1, y, y+1 with -1 -> 1 (REFLECT_101 on the doubled grid) and H -> H-1
    const int y0 = y - 1 < 0 ? (H > 1 ? 1 : 0) : y - 1, y2 = y + 1 >= H ? H - 1 : y + 1;
    const WT r1 = pyr_up_h<T, CN>(src.row<T>(f, y), dx, c, W);
    const WT r2 = pyr_up_h<T, CN>(src.row<T>(f, y2), dx, c, W);
    T out;
    if (dy & 1) {
        if constexpr (sizeof(T) == 1) out = (uchar)(((r1 + r2) * 4 + 32) >> 6);
        else out = __fmul_rn(1.f / 16, __fadd_rn(r1, r2));
    } else {
        const WT r0 = pyr_up_h<T, CN>(src.row<T>(f, y0), dx, c, W);
        if constexpr (sizeof(T) == 1) out = (uchar)((r0 + r1 * 6 + r2 + 32) >> 6);
        else out = __fmul_rn(1.f / 64, __fadd_rn(__fadd_rn(__fmul_rn(6.f, r1), r0), r2));
    }
    dst.row<T>(f, dy)[e] = out;
}

template <typename T>
static int pyr_launch(bool down, const Img& s, const Img& d, int cn, int border, cudaStream_t st)
{
    dim3 grid(div_up((unsigned)(d.cols * cn), 256), (unsigned)d.rows, (unsigned)s.frames);
#define GO(CN) do { if (down) pyr_down_kernel<T, CN><<<grid, 256, 0, st>>>(s, d, border); else pyr_up_kernel<T, CN><<<grid, 256, 0, st>>>(s, d); } while (0)
    if (cn == 1) GO(1); else if (cn == 3) GO(3); else GO(4);
#undef GO
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

static int pyr_common(bool down, const b200cvMat* src, const b200cvMat* dst, int border, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->type == dst->type, "pyramid: dst type must equal src type");
    B200_REQUIRE(src->data != dst->data, "pyramid: in-place is not supported");
    const int depth = B200CV_DEPTH(src->type), cn = B200CV_CN(src->type);
    if ((depth != B200CV_8U && depth != B200CV_32F) || (cn != 1 && cn != 3 && cn != 4)) return B200CV_NOT_IMPLEMENTED;
    border &= ~B200CV_BORDER_ISOLATED;
    if (down) {
        B200_REQUIRE(border != B200CV_BORDER_CONSTANT, "pyrDown: BORDER_CONSTANT is not allowed (pyramids.cpp:1352)");
        if (border < 0 || border > B200CV_BORDER_REFLECT_101) return B200CV_NOT_IMPLEMENTED;
        if (dst->cols != (src->cols + 1) / 2 || dst->rows != (src->rows + 1) / 2) return B200CV_NOT_IMPLEMENTED;
    } else {
        B200_REQUIRE(border == B200CV_BORDER_REFLECT_101, "pyrUp: only BORDER_DEFAULT (pyramids.cpp:1463)");
        if (dst->cols != src->cols * 2 || dst->rows != src->rows * 2) return B200CV_NOT_IMPLEMENTED;
    }
    if (dst->rows >= 65536) return B200CV_NOT_IMPLEMENTED;
    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    cudaStream_t st = as_stream(stream);
    return depth == B200CV_8U ? pyr_launch<uchar>(down, s, d, cn, border, st) : pyr_launch<float>(down, s, d, cn, border, st);
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_pyr_down(const b200cvMat* src, const b200cvMat* dst, int border, void* stream) { return pyr_common(true, src, dst, border, stream); }
extern "C" int b200cv_pyr_up(const b200cvMat* src, const b200cvMat* dst, int border, void* stream) { return pyr_common(false, src, dst, border, stream); }
