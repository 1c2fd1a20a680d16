// distance.cu -- cv::distanceTransform (imgproc/src/distransform.cpp) on sm_90a, bit-exact, 8UC1 sources.
//
// Chamfer 3x3 / 5x5 (DIST_C, DIST_L1, DIST_L2 with mask 3 or 5) and the 8-bit L1 call: dist_chamfer_kernel, one launch.
//   One CTA walks one frame (frames side by side along grid x) in the reference's raster order: the forward pass top-down into a
//   4 B/px scratch from the stream-ordered pool, then the backward pass bottom-up, which updates the scratch in place and writes dst.
//   The weights are 16.16 fixed point and everything is unsigned integer arithmetic, so the answer is exact by construction.
//   Each row is evaluated in parallel: with u[j] the candidate from the rows above (0 at a zero pixel), the forward recurrence
//   t[j] = min(DIST_MAX, u[j], t[j-1] + HV) unrolls to t[j] = min(DIST_MAX, j*HV + min_{k<=j}(u[k] - k*HV)), a prefix minimum in
//   64-bit integers; the backward recurrence t[j] = min(a[j], t[j+1] + HV) is the mirrored suffix minimum.  The backward pass skips
//   the rows below when t0 <= HV, as the reference does (every weight is >= HV, so the skip cannot change a value).  The latency of a
//   frame is 2 * H dependent row steps.  The 8-bit L1 call runs the L1 3x3 chamfer (weights 1, 2) and stores min(t >> 16, 255): the
//   L1 chamfer is the exact city-block distance, and the reference's saturating 8-bit scans are min(255, that distance)
//   (tests/test_dist_reference.py checks the two restatements agree on every case).  The source is read only by the forward pass and
//   dst written only by the backward pass, so src == dst works.
//
// Precise (mask 0, any type but DIST_C / DIST_L1): two launches.
//   dist_column_kernel  one thread per column: a bottom-up scan stores the distance to the nearest zero at or below each pixel as int
//                       bits in dst, a top-down scan turns it into (float)(unsigned)d^2 (UINT_MAX where the column has no zero or
//                       d >= 65536).  Threads along a row give coalesced accesses.
//   dist_row_kernel     one row per warp: lane 0 builds the reference's lower envelope of parabolas (stack v, z, and f[v] of 12 B per
//                       entry) with the reference's float operations in the reference's order (__fsub_rn / __fadd_rn / __fmul_rn, so
//                       nothing is contracted); then the 32 lanes each find k for their columns by a binary search over z, which is
//                       strictly increasing along the stack, so it picks the k of the reference's walk `while (z[k+1] < q) k++`, and
//                       write sqrt((float)sq[|q - p|] + f[p]).
//                       The stacks live in shared memory for rows of up to 19 370 columns (12 B per column per warp);
//                       wider rows use a global scratch from the stream-ordered pool, one stack per resident warp.
// Requires W * H < 2^31.
#include <algorithm>
#include <climits>
#include "common.cuh"

namespace b200cv {

namespace {

constexpr int CT = 1024;                 // chamfer: threads per CTA at most (fewer for narrow images: one warp per 128 columns)
constexpr int CPT = 4;                   // chamfer: columns per thread per tile
constexpr int RW_MAX = 8;                // row pass: warps per CTA at most
constexpr int SMEM_MAX = 232448;         // sm_90: dynamic shared memory per block, opt-in maximum
constexpr int PRECISE_MAX = 1 << 16;     // the reference's PRECISE_DIST_MAX

__host__ __device__ __forceinline__ size_t stack_bytes(int n) { return ((size_t)12 * n + 4 + 15) & ~(size_t)15; }

struct ChamferArgs {
    Img src, dst;
    unsigned* tmp;                       // W * H per frame
    unsigned hv, diag, lng, dmax;
    int out8;
};

// block-wide inclusive prefix minimum of CPT values per thread (thread-major order), started from `carry`; returns the new carry
// (the minimum over the whole tile).  One __syncthreads; `red` is the buffer of this tile's parity, one entry per warp.
__device__ __forceinline__ long long block_prefix_min(long long (&x)[CPT], long long carry, long long* red)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int e = 1; e < CPT; e++) x[e] = min(x[e], x[e - 1]);
    long long s = x[CPT - 1];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s = min(s, y);
    }
    long long excl = __shfl_up_sync(0xffffffffu, s, 1);
    if (lane == 31) red[warp] = s;
    __syncthreads();
    long long before = carry, all = carry;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) {
        const long long r = red[w];
        if (w < warp) before = min(before, r);
        all = min(all, r);
    }
    if (lane > 0) before = min(before, excl);
#pragma unroll
    for (int e = 0; e < CPT; e++) x[e] = min(x[e], before);
    return all;
}

template <int R>
__global__ void __launch_bounds__(CT) dist_chamfer_kernel(const ChamferArgs a)
{
    __shared__ long long red[2][CT / 32];
    const int W = a.src.cols, H = a.src.rows, f = blockIdx.x;
    const int CTILE = blockDim.x * CPT;                 // columns per tile
    unsigned* T = a.tmp + (size_t)f * W * H;
    const unsigned HV = a.hv, DG = a.diag, LG = a.lng, DM = a.dmax;
    const long long hv = HV;
    auto at = [&](int y, int x) -> unsigned {           // the reference's temp with its DIST_MAX border
        return (y < 0 || y >= H || x < 0 || x >= W) ? DM : T[(size_t)y * W + x];
    };
    int par = 0;

    // forward pass: rows top-down, each row's columns left to right as a prefix minimum
    for (int i = 0; i < H; i++) {
        const uchar* s = a.src.row<const uchar>(f, i);
        long long carry = LLONG_MAX;
        for (int c0 = 0; c0 < W; c0 += CTILE) {
            long long x[CPT];
            const int j0 = c0 + threadIdx.x * CPT;
#pragma unroll
            for (int e = 0; e < CPT; e++) {
                const int j = j0 + e;
                long long v = LLONG_MAX;
                if (j < W) {
                    unsigned u = 0;
                    if (s[j]) {
                        if (R == 1) {
                            u = min(min(at(i - 1, j - 1) + DG, at(i - 1, j) + HV), at(i - 1, j + 1) + DG);
                        } else {
                            u = min(at(i - 2, j - 1) + LG, at(i - 2, j + 1) + LG);
                            u = min(u, min(at(i - 1, j - 2) + LG, at(i - 1, j - 1) + DG));
                            u = min(u, min(at(i - 1, j) + HV, at(i - 1, j + 1) + DG));
                            u = min(u, at(i - 1, j + 2) + LG);
                        }
                    }
                    v = (long long)u - (long long)j * hv;
                }
                x[e] = v;
            }
            carry = block_prefix_min(x, carry, red[par]);
            par ^= 1;
#pragma unroll
            for (int e = 0; e < CPT; e++) {
                const int j = j0 + e;
                if (j < W) T[(size_t)i * W + j] = (unsigned)min((long long)DM, (long long)j * hv + x[e]);
            }
        }
        __syncthreads();
    }

    // backward pass: rows bottom-up, each row's columns right to left as a suffix minimum (thread 0 takes the rightmost columns)
    for (int i = H - 1; i >= 0; i--) {
        long long carry = LLONG_MAX;
        for (int c0 = 0; c0 < W; c0 += CTILE) {
            long long x[CPT];
            const int r0 = c0 + threadIdx.x * CPT;
#pragma unroll
            for (int e = 0; e < CPT; e++) {
                const int j = W - 1 - (r0 + e);
                long long v = LLONG_MAX;
                if (j >= 0) {
                    unsigned t0 = T[(size_t)i * W + j];
                    if (t0 > HV) {
                        if (R == 1) {
                            t0 = min(t0, min(min(at(i + 1, j + 1) + DG, at(i + 1, j) + HV), at(i + 1, j - 1) + DG));
                        } else {
                            t0 = min(t0, min(at(i + 2, j + 1) + LG, at(i + 2, j - 1) + LG));
                            t0 = min(t0, min(at(i + 1, j + 2) + LG, at(i + 1, j + 1) + DG));
                            t0 = min(t0, min(at(i + 1, j) + HV, at(i + 1, j - 1) + DG));
                            t0 = min(t0, at(i + 1, j - 2) + LG);
                        }
                    }
                    v = (long long)t0 + (long long)j * hv;
                }
                x[e] = v;
            }
            carry = block_prefix_min(x, carry, red[par]);
            par ^= 1;
#pragma unroll
            for (int e = 0; e < CPT; e++) {
                const int j = W - 1 - (r0 + e);
                if (j < 0) continue;
                const unsigned t = (unsigned)(x[e] - (long long)j * hv);
                T[(size_t)i * W + j] = t;
                if (a.out8) a.dst.row<uchar>(f, i)[j] = (uchar)min(t >> 16, 255u);
                else a.dst.row<float>(f, i)[j] = __fmul_rn(__uint2float_rn(t), 1.f / 65536.f);
            }
        }
        __syncthreads();
    }
}

// precise, stage 1: per column the squared distance to the nearest zero pixel in the column, as (float)(unsigned)
__global__ void __launch_bounds__(128) dist_column_kernel(const Img src, const Img dst)
{
    const int x = blockIdx.x * 128 + threadIdx.x, f = blockIdx.z, m = src.rows;
    if (x >= src.cols) return;
    int dist = m - 1;
    for (int j = m - 1; j >= 0; j--) {                  // distance to the nearest zero at or below (no zero: m - 1 + rows to the bottom)
        dist = src.row<const uchar>(f, j)[x] == 0 ? 0 : dist + 1;
        dst.row<int>(f, j)[x] = dist;
    }
    dist = m - 1;
    for (int j = 0; j < m; j++) {
        float* p = dst.row<float>(f, j) + x;
        dist = min(dist + 1, *(const int*)p);
        const unsigned sq = (dist < m && dist < PRECISE_MAX) ? (unsigned)dist * (unsigned)dist : UINT_MAX;
        *p = __uint2float_rn(sq);
    }
}

__device__ __forceinline__ unsigned sq_tab(int i) { return i < PRECISE_MAX ? (unsigned)i * (unsigned)i : UINT_MAX; }

// precise, stage 2: the lower envelope of each row (one row per warp).  scratch == NULL: stacks in dynamic shared memory, one per warp
// of the CTA; otherwise one stack per warp of the grid at scratch + warp * stack_bytes(n).
__global__ void __launch_bounds__(RW_MAX * 32) dist_row_kernel(const Img dst, int rows_total, uchar* scratch)
{
    extern __shared__ __align__(16) uchar smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int n = dst.cols, H = dst.rows;
    const int gw = blockIdx.x * nw + wib, gstride = gridDim.x * nw;
    uchar* base = scratch ? scratch + (size_t)gw * stack_bytes(n) : smem + (size_t)wib * stack_bytes(n);
    float* z = (float*)base;                             // n + 1
    int* v = (int*)(z + n + 1);                          // n
    float* fv = (float*)(v + n);                         // n: f[v[k]]
    const float inf = 1e15f;

    for (int row = gw; row < rows_total; row += gstride) {
        float* d = dst.row<float>(row / H, row % H);
        int k = 0;
        for (int c0 = 0; c0 < n; c0 += 32) {
            const float mine = c0 + lane < n ? d[c0 + lane] : 0.f;
            const int cnt = min(32, n - c0);
            for (int e = 0; e < cnt; e++) {
                const float fq = __shfl_sync(0xffffffffu, mine, e);
                const int q = c0 + e;
                if (lane != 0) continue;
                if (q == 0) { v[0] = 0; fv[0] = fq; z[0] = -inf; z[1] = inf; continue; }
                for (;; k--) {
                    const int p = v[k];
                    const float fp = fv[k];
                    const float inv = __double2float_rn(0.5 / (double)(q - p));
                    const float dsq = q < PRECISE_MAX ? __uint2float_rn(sq_tab(q) - sq_tab(p))
                                                      : __fmul_rn(__int2float_rn(q + p), __int2float_rn(q - p));
                    const float s = __fmul_rn(__fadd_rn(__fsub_rn(fq, fp), dsq), inv);
                    if (s > z[k]) {
                        k++;
                        v[k] = q; fv[k] = fq; z[k] = s; z[k + 1] = inf;
                        break;
                    }
                }
            }
        }
        const int K = __shfl_sync(0xffffffffu, k, 0);
        __syncwarp();
        for (int q = lane; q < n; q += 32) {
            const float qf = (float)q;
            int lo = 0, hi = K;                          // smallest k with z[k + 1] >= q (z[K + 1] = inf)
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (z[mid + 1] < qf) lo = mid + 1; else hi = mid;
            }
            const int p = v[lo];
            d[q] = __fsqrt_rn(__fadd_rn(__uint2float_rn(sq_tab(abs(q - p))), fv[lo]));
        }
        __syncwarp();
    }
}

PerDeviceFlag g_row_attr;

// 16.16 weights of getDistanceTransformMask, cvRound(w * 65536) on the float metric
unsigned fix16(float w) { return (unsigned)__builtin_lrint((double)(w * 65536.f)); }

}  // namespace

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_distance_transform(const b200cvMat* src, const b200cvMat* dst, int distance_type, int mask_size, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    B200_REQUIRE(src->type == B200CV_MAKETYPE(B200CV_8U, 1), "distanceTransform: src must be 8UC1");
    const int frames = src->frames > 1 ? src->frames : 1;
    B200_REQUIRE(dst->cols == src->cols && dst->rows == src->rows && (dst->frames > 1 ? dst->frames : 1) == frames,
                 "distanceTransform: dst must have the source size");
    const int W = src->cols, H = src->rows;
    B200_REQUIRE((long long)W * H < (1ll << 31), "distanceTransform: W * H must be below 2^31");
    B200_REQUIRE(frames <= 65535, "distanceTransform: at most 65535 frames per call");

    // the reference's argument rules (distransform.cpp, cv::distanceTransform): the 8-bit call is L1 whatever the mask; otherwise the
    // mask must be 0, 3 or 5, C and L1 always run the 3x3 mask, a precise mask runs the exact transform whatever the type, and the
    // chamfer masks take C, L1 or L2 only
    const bool out8 = dst->type == B200CV_MAKETYPE(B200CV_8U, 1);
    float hvf = 1.f, dgf = 2.f, lgf = 0.f;
    int mask = 3;
    if (out8) {
        B200_REQUIRE(distance_type == B200CV_DIST_L1, "distanceTransform: an 8UC1 destination needs DIST_L1");
    } else {
        B200_REQUIRE(dst->type == B200CV_MAKETYPE(B200CV_32F, 1), "distanceTransform: dst must be 32FC1, or 8UC1 with DIST_L1");
        B200_REQUIRE(mask_size == B200CV_DIST_MASK_3 || mask_size == B200CV_DIST_MASK_5 || mask_size == B200CV_DIST_MASK_PRECISE,
                     "distanceTransform: mask size should be 3, 5 or 0 (precise)");
        mask = (distance_type == B200CV_DIST_C || distance_type == B200CV_DIST_L1) ? 3 : mask_size;
        if (mask != B200CV_DIST_MASK_PRECISE) {
            B200_REQUIRE(distance_type == B200CV_DIST_C || distance_type == B200CV_DIST_L1 || distance_type == B200CV_DIST_L2,
                         "distanceTransform: a 3x3 or 5x5 mask needs DIST_C, DIST_L1 or DIST_L2");
            if (distance_type == B200CV_DIST_C) { hvf = 1.f; dgf = 1.f; lgf = 2.f; }
            else if (distance_type == B200CV_DIST_L1) { hvf = 1.f; dgf = 2.f; lgf = 3.f; }
            else if (mask == 3) { hvf = 0.955f; dgf = 1.3693f; }
            else { hvf = 1.f; dgf = 1.4f; lgf = 2.1969f; }
        }
    }

    cudaStream_t st = as_stream(stream);
    if (mask == B200CV_DIST_MASK_PRECISE) {
        dist_column_kernel<<<dim3(div_up(W, 128), 1, frames), 128, 0, st>>>(make_img(src), make_img(dst));
        B200_LAUNCH_CHECK();
        const int rows = H * frames;
        const size_t per = stack_bytes(W);
        if (per <= (size_t)SMEM_MAX) {
            const int nw = (int)std::min<size_t>(RW_MAX, SMEM_MAX / per);
            bool& done = g_row_attr.cur();
            if (!done) {
                B200_CUDA(cudaFuncSetAttribute(dist_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
                done = true;
            }
            dist_row_kernel<<<div_up(rows, nw), nw * 32, nw * per, st>>>(make_img(dst), rows, nullptr);
            B200_LAUNCH_CHECK();
        } else {
            const int nw = 4, blocks = std::min(div_up(rows, nw), (unsigned)num_sms() * 2);
            uchar* scratch = nullptr;
            B200_CUDA(cudaMallocAsync(&scratch, per * nw * blocks, st));
            dist_row_kernel<<<blocks, nw * 32, 0, st>>>(make_img(dst), rows, scratch);
            count_launch();
            const cudaError_t e = cudaGetLastError();
            cudaFreeAsync(scratch, st);
            if (e != cudaSuccess) return cuda_fail(e, "dist_row_kernel launch", __FILE__, __LINE__);
        }
        return B200CV_OK;
    }

    ChamferArgs a;
    a.src = make_img(src);
    a.dst = make_img(dst);
    a.hv = fix16(hvf);
    a.diag = fix16(dgf);
    a.lng = mask == 5 ? fix16(lgf) : 0u;
    a.dmax = UINT_MAX - (mask == 5 ? a.lng : a.diag);
    a.out8 = out8 ? 1 : 0;
    unsigned* tmp = nullptr;
    B200_CUDA(cudaMallocAsync(&tmp, (size_t)W * H * frames * sizeof(unsigned), st));
    a.tmp = tmp;
    // a row step costs a block barrier or two: narrow images get a smaller block (at least one warp, at most CT threads)
    const int threads = (int)std::min<unsigned>(CT, div_up(div_up(W, CPT), 32) * 32);
    if (mask == 5) dist_chamfer_kernel<2><<<frames, threads, 0, st>>>(a);
    else dist_chamfer_kernel<1><<<frames, threads, 0, st>>>(a);
    count_launch();
    const cudaError_t e = cudaGetLastError();
    cudaFreeAsync(tmp, st);
    if (e != cudaSuccess) return cuda_fail(e, "dist_chamfer_kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}
