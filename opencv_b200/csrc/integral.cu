// integral.cu -- cv::integral for 8UC1 images: sum (CV_32S) and, optionally, the sum of squares (CV_64F).
//
// Reference (sumpixels.dispatch.cpp:192-235, :415-451): sum is (H+1) x (W+1), first row and column zero,
//     sum[y+1][x+1] = sum[y][x+1] + (src[y][0] + ... + src[y][x]);  int arithmetic (it wraps for images beyond 2^31 / 255 pixels, as the
//     reference's does); squares accumulate in double, where every partial sum is an integer below 2^53: exact in any order.
// Two kernels with warp scans:
//   rows     one warp per (frame, row): 128 pixels per step -- a 32-bit load of 4 pixels per lane, the prefix of the 4 in the lane, an
//            inclusive shuffle scan of the lane totals, the running total of the row carried from step to step -- written as row prefixes to
//            sum[y + 1][1 ..]; the same kernel zeroes column 0 and row 0
//   columns  one thread per column walks down the image adding in place, 8 rows of loads in flight; coalesced across the threads of a warp
// Traffic: 1 byte read + 4 written (rows) + 4 read + 4 written (columns) = 13 bytes per pixel against 5 algorithmic.
#include "common.cuh"

namespace b200cv {

namespace {

template <typename T, bool SQ> __device__ __forceinline__ T ig_val(uchar v)
{
    if constexpr (SQ) return (T)((int)v * (int)v);
    else return (T)v;
}

template <typename T> __device__ __forceinline__ T ig_shfl_up(T v, int d)
{
    if constexpr (sizeof(T) == 8) {
        const long long b = __double_as_longlong((double)v);
        const int lo = __shfl_up_sync(0xffffffffu, (int)(b & 0xffffffffll), d), hi = __shfl_up_sync(0xffffffffu, (int)(b >> 32), d);
        return (T)__longlong_as_double(((long long)hi << 32) | (unsigned)lo);
    } else return (T)__shfl_up_sync(0xffffffffu, (int)v, d);
}
template <typename T> __device__ __forceinline__ T ig_shfl(T v, int l)
{
    if constexpr (sizeof(T) == 8) {
        const long long b = __double_as_longlong((double)v);
        const int lo = __shfl_sync(0xffffffffu, (int)(b & 0xffffffffll), l), hi = __shfl_sync(0xffffffffu, (int)(b >> 32), l);
        return (T)__longlong_as_double(((long long)hi << 32) | (unsigned)lo);
    } else return (T)__shfl_sync(0xffffffffu, (int)v, l);
}

template <typename T, bool SQ>
__global__ void __launch_bounds__(256) integral_rows_kernel(Img src, Img out, int W, int H)
{
    const int lane = threadIdx.x & 31;
    const int y = blockIdx.x * 8 + (threadIdx.x >> 5), f = blockIdx.y;
    if (y >= H) return;
    const uchar* s = src.row<uchar>(f, y);
    T* o = out.row<T>(f, y + 1) + 1;
    const bool al = (((uintptr_t)s) & 3) == 0;
    if (lane == 0) o[-1] = 0;                                       // first column
    if (y == 0) { T* z = out.row<T>(f, 0); for (int x = lane; x <= W; x += 32) z[x] = 0; }      // first row
    T carry = 0;
    for (int x0 = 0; x0 < W; x0 += 128) {
        const int x = x0 + 4 * lane;
        unsigned w = 0;
        if (x + 4 <= W && al) w = __ldg((const unsigned*)(s + x));
        else {
#pragma unroll
            for (int i = 0; i < 4; i++) if (x + i < W) w |= (unsigned)s[x + i] << (8 * i);
        }
        T p0 = ig_val<T, SQ>((uchar)(w & 255)), p1 = p0 + ig_val<T, SQ>((uchar)((w >> 8) & 255)), p2 = p1 + ig_val<T, SQ>((uchar)((w >> 16) & 255)),
          p3 = p2 + ig_val<T, SQ>((uchar)(w >> 24));
        T tot = p3;                                                 // inclusive scan of the lane totals
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const T up = ig_shfl_up<T>(tot, d); if (lane >= d) tot += up; }
        const T base = carry + (tot - p3);                          // everything left of this lane's 4 pixels
        if (x + 4 <= W) { o[x] = base + p0; o[x + 1] = base + p1; o[x + 2] = base + p2; o[x + 3] = base + p3; }
        else {
            if (x < W) o[x] = base + p0;
            if (x + 1 < W) o[x + 1] = base + p1;
            if (x + 2 < W) o[x + 2] = base + p2;
        }
        carry += ig_shfl<T>(tot, 31);
    }
}

template <typename T>
__global__ void __launch_bounds__(128) integral_cols_kernel(Img out, int W, int H)
{
    const int x = blockIdx.x * 128 + threadIdx.x, f = blockIdx.y;
    if (x > W) return;
    T run = 0;
    int y = 1;
    for (; y + 8 <= H + 1; y += 8) {
        T v[8];
#pragma unroll
        for (int i = 0; i < 8; i++) v[i] = out.row<T>(f, y + i)[x];
#pragma unroll
        for (int i = 0; i < 8; i++) { run += v[i]; out.row<T>(f, y + i)[x] = run; }
    }
    for (; y <= H; y++) { T* p = out.row<T>(f, y) + x; run += *p; *p = run; }
}

template <typename T, bool SQ>
int integral_launch(const Img& s, const Img& o, cudaStream_t st)
{
    const int W = s.cols, H = s.rows, frames = s.frames;
    const dim3 gr(div_up((unsigned)H, 8), (unsigned)frames), gc(div_up((unsigned)W + 1, 128), (unsigned)frames);
    integral_rows_kernel<T, SQ><<<gr, 256, 0, st>>>(s, o, W, H);
    integral_cols_kernel<T><<<gc, 128, 0, st>>>(o, W, H);
    const cudaError_t e = cudaGetLastError();
    count_launch(2);
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

}  // namespace

// src: 8UC1 W x H;  sum: 32SC1 (W+1) x (H+1);  sqsum: null or 64FC1 (W+1) x (H+1)
int integral_impl(const b200cvMat* src, const b200cvMat* sum, const b200cvMat* sqsum, cudaStream_t st)
{
    if (src->type != B200CV_MAKETYPE(B200CV_8U, 1) || sum->type != B200CV_MAKETYPE(B200CV_32S, 1)) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(sum->cols == src->cols + 1 && sum->rows == src->rows + 1, "integral: sum must be (width + 1) x (height + 1)");
    Img s = make_img(src), o = make_img(sum);
    B200_REQUIRE(s.frames == o.frames, "src/dst batch mismatch");
    if (s.rows >= 65535 || s.frames >= 65536 || (size_t)s.rows * s.frames >= (1u << 31)) return B200CV_NOT_IMPLEMENTED;
    int rc = integral_launch<int, false>(s, o, st);
    if (rc || !sqsum || !sqsum->data) return rc;
    if (sqsum->type != B200CV_MAKETYPE(B200CV_64F, 1)) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(sqsum->cols == src->cols + 1 && sqsum->rows == src->rows + 1, "integral: sqsum must be (width + 1) x (height + 1)");
    Img q = make_img(sqsum);
    B200_REQUIRE(s.frames == q.frames, "src/dst batch mismatch");
    return integral_launch<double, true>(s, q, st);
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_integral(const b200cvMat* src, const b200cvMat* sum, const b200cvMat* sqsum, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(sum, "sum"))) return rc;
    if (sqsum && sqsum->data && (rc = check_mat(sqsum, "sqsum"))) return rc;
    return integral_impl(src, sum, sqsum, as_stream(stream));
}
