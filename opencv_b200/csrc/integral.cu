// integral.cu -- cv::integral for 8UC1 images: sum (CV_32S) and, optionally, the sum of squares (CV_64F) .
//
// Reference (sumpixels.dispatch.cpp:192-235, :415-451): sum is (H+1) x (W+1), first row and column zero,
//     sum[y+1][x+1] = sum[y][x+1] + (src[y][0] + ... + src[y][x]);  int arithmetic (it wraps for images beyond 2^31 / 255 pixels, as the
//     reference's does); squares accumulate in double, where every partial sum is an integer below 2^53: exact in any order.
// Six small kernels, none of which needs threads to talk to each other (every stage is a map over independent pieces, so the whole op
// also runs under the host emulation of tests/):
//   rows:     H1 sum of every 16-pixel chunk            H2 exclusive scan of the chunk sums of a row      H3 prefix inside the chunk + offset -> sum
//   columns:  V1 sum of every 32-row block of a column  V2 exclusive scan of the block sums of a column   V3 prefix inside the block + offset, in place
// Algorithmic traffic: 1 byte read + 4 (12 with squares) written per pixel; this version re-reads the source once and the output twice.
#include <stdlib.h>
#include <string.h>
#include "common.cuh"

namespace b200cv {

int integral_scan_run(const Img& s, const Img& o, int squares, cudaStream_t st);      // integral_scan.cu

namespace {

enum { IG_CHUNK = 16, IG_ROWS = 32 };

template <typename T, bool SQ> __device__ __forceinline__ T ig_val(uchar v)
{
    if constexpr (SQ) return (T)((int)v * (int)v);
    else return (T)v;
}

struct IgDims { int W, H, NC, NB; };

template <typename T, bool SQ>
__global__ void __launch_bounds__(256) integral_h1_kernel(Img src, T* cs, IgDims g)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    if (c >= g.NC) return;
    const uchar* s = src.row<uchar>(f, y) + c * IG_CHUNK;
    const int n = min((int)IG_CHUNK, g.W - c * IG_CHUNK);
    T acc = 0;
    for (int i = 0; i < n; i++) acc += ig_val<T, SQ>(s[i]);
    cs[((size_t)f * g.H + y) * g.NC + c] = acc;
}

template <typename T>
__global__ void __launch_bounds__(256) integral_h2_kernel(T* cs, IgDims g, int frames)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;            // row index over all frames
    if (r >= g.H * frames) return;
    T* p = cs + (size_t)r * g.NC;
    T run = 0;
    for (int c = 0; c < g.NC; c++) { const T v = p[c]; p[c] = run; run += v; }
}

template <typename T, bool SQ>
__global__ void __launch_bounds__(256) integral_h3_kernel(Img src, Img out, const T* cs, IgDims g)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    if (c >= g.NC) return;
    const uchar* s = src.row<uchar>(f, y) + c * IG_CHUNK;
    const int n = min((int)IG_CHUNK, g.W - c * IG_CHUNK);
    T* o = out.row<T>(f, y + 1) + 1 + c * IG_CHUNK;
    T run = cs[((size_t)f * g.H + y) * g.NC + c];
    for (int i = 0; i < n; i++) { run += ig_val<T, SQ>(s[i]); o[i] = run; }
    if (c == 0) out.row<T>(f, y + 1)[0] = 0;                        // first column
    if (y == 0) {                                                   // first row
        T* z = out.row<T>(f, 0) + 1 + c * IG_CHUNK;
        for (int i = 0; i < n; i++) z[i] = 0;
        if (c == 0) out.row<T>(f, 0)[0] = 0;
    }
}

template <typename T>
__global__ void __launch_bounds__(256) integral_v1_kernel(Img out, T* bs, IgDims g)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y, f = blockIdx.z;
    if (x >= g.W) return;
    const int y0 = b * IG_ROWS, y1 = min(y0 + (int)IG_ROWS, g.H);
    T acc = 0;
    for (int y = y0; y < y1; y++) acc += out.row<T>(f, y + 1)[x + 1];
    bs[((size_t)f * g.NB + b) * g.W + x] = acc;
}

template <typename T>
__global__ void __launch_bounds__(256) integral_v2_kernel(T* bs, IgDims g)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, f = blockIdx.z;
    if (x >= g.W) return;
    T* p = bs + (size_t)f * g.NB * g.W + x;
    T run = 0;
    for (int b = 0; b < g.NB; b++) { const T v = p[(size_t)b * g.W]; p[(size_t)b * g.W] = run; run += v; }
}

template <typename T>
__global__ void __launch_bounds__(256) integral_v3_kernel(Img out, const T* bs, IgDims g)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y, f = blockIdx.z;
    if (x >= g.W) return;
    const int y0 = b * IG_ROWS, y1 = min(y0 + (int)IG_ROWS, g.H);
    T run = bs[((size_t)f * g.NB + b) * g.W + x];
    for (int y = y0; y < y1; y++) { T* o = out.row<T>(f, y + 1) + x + 1; run += *o; *o = run; }
}

template <typename T, bool SQ>
int integral_run(const Img& s, const Img& o, cudaStream_t st)
{
    IgDims g;
    g.W = s.cols; g.H = s.rows; g.NC = (int)div_up((unsigned)g.W, IG_CHUNK); g.NB = (int)div_up((unsigned)g.H, IG_ROWS);
    const int frames = s.frames;
#ifndef B200CV_HOST_EMULATION
    {
        // second version (integral_scan.cu): two kernels with warp scans; B200CV_INTEGRAL_PATH=v1 keeps the six map-only kernels below
        const char* path = getenv("B200CV_INTEGRAL_PATH");
        if (!(path && !strcmp(path, "v1"))) return integral_scan_run(s, o, SQ ? 1 : 0, st);
    }
#endif
    T* scratch = nullptr;
    const size_t ncs = (size_t)frames * g.H * g.NC, nbs = (size_t)frames * g.NB * g.W;
    B200_CUDA(cudaMallocAsync((void**)&scratch, sizeof(T) * (ncs + nbs), st));
    T* cs = scratch; T* bs = scratch + ncs;
    const dim3 block(256);
    {
        const dim3 grid(div_up((unsigned)g.NC, 256), (unsigned)g.H, (unsigned)frames);
        integral_h1_kernel<T, SQ><<<grid, block, 0, st>>>(s, cs, g);
    }
    {
        const dim3 grid(div_up((unsigned)(g.H * frames), 256));
        integral_h2_kernel<T><<<grid, block, 0, st>>>(cs, g, frames);
    }
    {
        const dim3 grid(div_up((unsigned)g.NC, 256), (unsigned)g.H, (unsigned)frames);
        integral_h3_kernel<T, SQ><<<grid, block, 0, st>>>(s, o, cs, g);
    }
    {
        const dim3 grid(div_up((unsigned)g.W, 256), (unsigned)g.NB, (unsigned)frames);
        integral_v1_kernel<T><<<grid, block, 0, st>>>(o, bs, g);
    }
    {
        const dim3 grid(div_up((unsigned)g.W, 256), 1, (unsigned)frames);
        integral_v2_kernel<T><<<grid, block, 0, st>>>(bs, g);
    }
    {
        const dim3 grid(div_up((unsigned)g.W, 256), (unsigned)g.NB, (unsigned)frames);
        integral_v3_kernel<T><<<grid, block, 0, st>>>(o, bs, g);
    }
    const cudaError_t e = cudaGetLastError();
    count_launch(6);
    cudaFreeAsync(scratch, st);
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
    int rc = integral_run<int, false>(s, o, st);
    if (rc || !sqsum || !sqsum->data) return rc;
    if (sqsum->type != B200CV_MAKETYPE(B200CV_64F, 1)) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(sqsum->cols == src->cols + 1 && sqsum->rows == src->rows + 1, "integral: sqsum must be (width + 1) x (height + 1)");
    Img q = make_img(sqsum);
    B200_REQUIRE(s.frames == q.frames, "src/dst batch mismatch");
    return integral_run<double, true>(s, q, st);
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
