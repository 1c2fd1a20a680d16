// canny.cu -- cv::Canny (imgproc/src/canny.cpp:823-1003) on sm_90a, bit-exact for 8-bit sources and for 16S derivatives.
//
// Four launches per call, whatever the image holds:
//   1. canny_nms_kernel     one 32 x 16 tile per block: the source tile and its apron (ksize/2 + 1) are staged in shared memory with
//                           the replicate border, the 16S Sobel / Scharr derivatives and the L1 / L2 magnitude (strongest channel, first
//                           channel on ties) are computed in integers for the tile plus a one-pixel ring, non-maximum suppression
//                           classifies each pixel as none / weak / strong, and a union-find in shared memory joins the tile's
//                           8-connected candidates.  Only the labels reach global memory: no gradient or magnitude plane.
//   2. canny_merge_kernel   joins candidates across tile edges and corners with a lock-free atomicCAS union.
//   3. canny_mark_kernel    points every candidate at its root (the trees are final) and lets each strong pixel flag its root.
//   4. canny_final_kernel   writes 255 where a candidate's root is flagged, 0 everywhere else.  Only this kernel touches dst, so
//                           src == dst is safe for 8UC1.
// The edge set of the reference's stack flood fill (canny.cpp:647-678, :914-927) is the set of candidates connected to a strong pixel,
// which does not depend on the order of traversal; union-find computes the same set with no host round trip.
//
// Labels: int32 per pixel per frame from the stream-ordered pool (4 B per pixel per frame: 531 MB for 16 4K frames).
//   NONE (0x7fffffff) = not a candidate; otherwise bits 0-30 = parent (y * W + x within the frame, a root points at itself) and bit 31 =
//   the pixel is strong (before step 3) / the component reaches a strong pixel (on a root after step 3).  Parents always have a smaller
//   index than their children, so the forest has no cycles.  Requires W * H < 2^31.
#include <climits>
#include <cmath>
#include <utility>
#include "common.cuh"

namespace b200cv {

namespace {

constexpr int TW = 32, TH = 16;                 // tile of output pixels per block
constexpr int BX = 32, BY = 8;                  // block shape
constexpr int NT = BX * BY;
constexpr unsigned FLAG = 0x80000000u;
constexpr int MASK = 0x7fffffff;
constexpr int NONE = 0x7fffffff;
constexpr int TG22 = 13573;                     // tan(22.5 deg) * 2^15, canny.cpp:35

// separable integer taps of getDerivKernels (deriv.cpp:38-105): KS 3/5/7 = Sobel, KS 1 = Scharr (aperture -1)
template <int KS> struct Taps;
template <> struct Taps<1> { __device__ static int s(int i) { const int t[3] = {3, 10, 3}; return t[i]; }
                             __device__ static int d(int i) { const int t[3] = {-1, 0, 1}; return t[i]; } };
template <> struct Taps<3> { __device__ static int s(int i) { const int t[3] = {1, 2, 1}; return t[i]; }
                             __device__ static int d(int i) { const int t[3] = {-1, 0, 1}; return t[i]; } };
template <> struct Taps<5> { __device__ static int s(int i) { const int t[5] = {1, 4, 6, 4, 1}; return t[i]; }
                             __device__ static int d(int i) { const int t[5] = {-1, -2, 0, 2, 1}; return t[i]; } };
template <> struct Taps<7> { __device__ static int s(int i) { const int t[7] = {1, 6, 15, 20, 15, 6, 1}; return t[i]; }
                             __device__ static int d(int i) { const int t[7] = {-1, -4, -5, 0, 5, 4, 1}; return t[i]; } };

// Sobel(..., CV_16S, ..., scale = 1/16) for aperture 7: the exact sum / 16 rounded half to even (cvRound of an exact float)
__device__ __forceinline__ int div16_rhe(int s)
{
    const int q = s >> 4, r = s & 15;
    return q + (r > 8 || (r == 8 && (q & 1)));
}

__device__ __forceinline__ int magnitude(int dx, int dy, bool l2)
{
    // L2 wraps in int32 like the reference (only Canny(dx, dy) can reach it): computed in unsigned
    return l2 ? (int)((unsigned)(dx * dx) + (unsigned)(dy * dy)) : abs(dx) + abs(dy);
}

// find with path halving: a non-root's parent is only ever replaced by one of its ancestors, so the plain store is safe next to the
// atomicCAS links, which only touch roots
__device__ __forceinline__ int find_s(volatile int* lab, int x)
{
    while (true) {
        const int p = lab[x];
        if (p == x) return x;
        const int gp = lab[p];
        if (gp == p) return p;
        lab[x] = gp;
        x = gp;
    }
}

__device__ __forceinline__ void unite_s(int* lab, int a, int b)
{
    while (true) {
        a = find_s(lab, a); b = find_s(lab, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        if (atomicCAS(&lab[a], a, b) == a) return;   // a was still a root: linked under the smaller root
    }
}

__device__ __forceinline__ int find_g(const int* L, int x)
{
    while (true) {
        const int p = __ldcg(L + x) & MASK;
        if (p == x) return x;
        x = p;
    }
}

// find with path halving, while the forest is built: a non-root's parent is only ever replaced by one of its ancestors and its flag bit
// does not change, so the plain store is safe next to the atomicCAS links (which only touch roots).  Not used once canny_mark_kernel
// starts pointing pixels straight at their roots: a late halving store could move a pixel off its root again.
__device__ __forceinline__ int find_halve(int* L, int x)
{
    while (true) {
        const int v = __ldcg(L + x), p = v & MASK;
        if (p == x) return x;
        const int gp = __ldcg(L + p) & MASK;
        if (gp == p) return p;
        __stcg(L + x, (int)(((unsigned)v & FLAG) | (unsigned)gp));
        x = gp;
    }
}

__device__ __forceinline__ void unite_g(int* L, int a, int b)
{
    while (true) {
        a = find_halve(L, a); b = find_halve(L, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = __ldcg(L + a);
        if ((old & MASK) != a) continue;
        if (atomicCAS(L + a, old, (int)(((unsigned)old & FLAG) | (unsigned)b)) == old) return;
    }
}

struct CannyArgs {
    Img src, dst;
    Img dy;                     // Canny(dx, dy): src is dx, this is dy
    int* labels;
    int low, high, l2;
};

// KS: 3 / 5 / 7 = Sobel aperture, 1 = Scharr, 0 = the 16S derivatives are given (src = dx, a.dy = dy)
template <int KS, int CN>
__global__ void __launch_bounds__(NT) canny_nms_kernel(const CannyArgs a)
{
    constexpr int R = KS == 0 ? 0 : (KS == 1 ? 1 : KS / 2);
    constexpr int A = KS == 0 ? 1 : R + 1;      // apron of the staged source
    constexpr int SW = TW + 2 * A, SH = TH + 2 * A;
    constexpr int MW = TW + 2, MH = TH + 2;     // magnitude tile with its one-pixel ring
    __shared__ uchar ssrc[KS == 0 ? 1 : SH * SW * CN];
    __shared__ int smag[MH * MW];
    __shared__ short sdx[TH * TW], sdy[TH * TW];
    __shared__ uchar scls[TH * TW];
    __shared__ int slab[TH * TW];

    const int W = a.src.cols, H = a.src.rows, f = blockIdx.z;
    const int tiles_x = (W + TW - 1) / TW;       // the tiles of a frame run along grid x: no 65535 limit on the height
    const int tx0 = (blockIdx.x % tiles_x) * TW, ty0 = (blockIdx.x / tiles_x) * TH;
    const int tid = threadIdx.y * BX + threadIdx.x;

    if (KS != 0) {
        for (int i = tid; i < SH * SW * CN; i += NT) {
            const int sy = i / (SW * CN), b = i - sy * (SW * CN), sx = b / CN, c = b - sx * CN;
            const int gy = min(max(ty0 - A + sy, 0), H - 1), gx = min(max(tx0 - A + sx, 0), W - 1);
            ssrc[i] = a.src.row<const uchar>(f, gy)[gx * CN + c];
        }
        __syncthreads();
    }

    for (int i = tid; i < MH * MW; i += NT) {
        const int my = i / MW, mx = i - my * MW;
        const int py = ty0 - 1 + my, px = tx0 - 1 + mx;
        int m = 0, bdx = 0, bdy = 0;
        if (py >= 0 && py < H && px >= 0 && px < W) {
#pragma unroll
            for (int c = 0; c < CN; c++) {
                int dx = 0, dy = 0;
                if (KS == 0) {
                    dx = a.src.row<const short>(f, py)[px * CN + c];
                    dy = a.dy.row<const short>(f, py)[px * CN + c];
                } else {
                    typedef Taps<KS == 0 ? 3 : KS> T;
                    const int sy0 = my - 1 + A - R, sx0 = mx - 1 + A - R;
#pragma unroll
                    for (int u = 0; u < 2 * R + 1; u++) {
                        int rs = 0, rd = 0;
#pragma unroll
                        for (int v = 0; v < 2 * R + 1; v++) {
                            const int p = ssrc[((sy0 + u) * SW + sx0 + v) * CN + c];
                            rs += T::s(v) * p;
                            rd += T::d(v) * p;
                        }
                        dx += T::s(u) * rd;
                        dy += T::d(u) * rs;
                    }
                    if (KS == 7) { dx = div16_rhe(dx); dy = div16_rhe(dy); }
                }
                const int mc = magnitude(dx, dy, a.l2);
                if (c == 0 || mc > m) { m = mc; bdx = dx; bdy = dy; }   // strict >: the first channel wins ties (canny.cpp:486-495)
            }
        }
        smag[i] = m;
        if (my >= 1 && my <= TH && mx >= 1 && mx <= TW) {
            sdx[(my - 1) * TW + mx - 1] = (short)bdx;
            sdy[(my - 1) * TW + mx - 1] = (short)bdy;
        }
    }
    __syncthreads();

    // non-maximum suppression (canny.cpp:596-640); magnitude outside the image is 0
    for (int i = tid; i < TH * TW; i += NT) {
        const int ly = i / TW, lx = i - ly * TW;
        const int* mr = smag + (ly + 1) * MW + lx + 1;
        const int m = mr[0];
        int cls = 0;
        if (ty0 + ly < H && tx0 + lx < W && m > a.low) {
            const int xs = sdx[i], ys = sdy[i];
            const int x = abs(xs), y = abs(ys) << 15;
            const int tg22x = x * TG22;
            bool keep;
            if (y < tg22x) {
                keep = m > mr[-1] && m >= mr[1];
            } else {
                const int tg67x = (int)((unsigned)tg22x + ((unsigned)x << 16));   // wraps for |dx| > 27146, as the reference's int does
                if (y > tg67x) {
                    keep = m > mr[-MW] && m >= mr[MW];
                } else {
                    const int s = (xs ^ ys) < 0 ? -1 : 1;
                    keep = m > mr[-MW - s] && m > mr[MW + s];
                }
            }
            if (keep) cls = m > a.high ? 2 : 1;
        }
        scls[i] = (uchar)cls;
    }
    __syncthreads();

    // union-find of the tile's 8-connected candidates.  Of the four earlier neighbours (upper-left, upper, upper-right, left) a pixel needs
    // at most two links: the upper neighbour is adjacent to the other three, and the left one to the upper-left one, so their own links
    // already join them.  The first link is the pixel's initial parent (an earlier, smaller index); only an upper-right neighbour next to
    // an upper-left or left one without an upper one between them needs a union.
    int second[(TH * TW + NT - 1) / NT];
#pragma unroll
    for (int k = 0; k < (TH * TW + NT - 1) / NT; k++) {
        const int i = tid + k * NT;
        second[k] = -1;
        int parent = i;
        if (i < TH * TW && scls[i]) {
            const int ly = i / TW, lx = i - ly * TW;
            const bool ul = ly > 0 && lx > 0 && scls[i - TW - 1], up = ly > 0 && scls[i - TW];
            const bool ur = ly > 0 && lx < TW - 1 && scls[i - TW + 1], le = lx > 0 && scls[i - 1];
            if (up) {
                parent = i - TW;
            } else {
                const int first = ul ? i - TW - 1 : le ? i - 1 : -1;
                if (first >= 0) { parent = first; if (ur) second[k] = i - TW + 1; }
                else if (ur) parent = i - TW + 1;
            }
        }
        if (i < TH * TW) slab[i] = parent;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < (TH * TW + NT - 1) / NT; k++)
        if (second[k] >= 0) unite_s(slab, tid + k * NT, second[k]);
    __syncthreads();

    int* L = a.labels + (size_t)f * W * H;
    for (int i = tid; i < TH * TW; i += NT) {
        const int ly = i / TW, lx = i - ly * TW;
        const int py = ty0 + ly, px = tx0 + lx;
        if (py >= H || px >= W) continue;
        int v = NONE;
        if (scls[i]) {
            const int r = find_s(slab, i);
            const int ry = r / TW, rx = r - ry * TW;
            v = (int)((unsigned)((ty0 + ry) * W + tx0 + rx) | (scls[i] == 2 ? FLAG : 0u));
        }
        L[py * W + px] = v;
    }
}

// tile edges: thread t < TW takes the tile's bottom row (pairs with the row below), TW <= t < TW + TH its right column (pairs with the
// column to the right); together they cover every 8-neighbour pair that crosses a tile edge or corner
__global__ void __launch_bounds__(64) canny_merge_kernel(int* labels, int W, int H)
{
    int* L = labels + (size_t)blockIdx.z * W * H;
    const int tiles_x = (W + TW - 1) / TW;
    const int tx0 = (blockIdx.x % tiles_x) * TW, ty0 = (blockIdx.x / tiles_x) * TH, t = threadIdx.x;
    if (t < TW) {
        const int x = tx0 + t, y = ty0 + TH - 1;
        if (y + 1 >= H || x >= W) return;
        const int p = y * W + x;
        if (__ldcg(L + p) == NONE) return;
        for (int dx = -1; dx <= 1; dx++) {
            const int nx = x + dx;
            if (nx < 0 || nx >= W) continue;
            const int q = (y + 1) * W + nx;
            if (__ldcg(L + q) != NONE) unite_g(L, p, q);
        }
    } else if (t < TW + TH) {
        const int x = tx0 + TW - 1, y = ty0 + t - TW;
        if (x + 1 >= W || y >= H) return;
        const int p = y * W + x;
        if (__ldcg(L + p) == NONE) return;
        for (int dy = -1; dy <= 1; dy++) {
            const int ny = y + dy;
            if (ny < 0 || ny >= H) continue;
            const int q = ny * W + x + 1;
            if (__ldcg(L + q) != NONE) unite_g(L, p, q);
        }
    }
}

// the forest no longer changes: point each candidate straight at its root; a strong pixel flags its root
__global__ void __launch_bounds__(256) canny_mark_kernel(int* labels, int n)
{
    const int p = blockIdx.x * 256 + threadIdx.x;
    if (p >= n) return;
    int* L = labels + (size_t)blockIdx.y * n;
    const int v = L[p];
    if (v == NONE) return;
    const int r = find_g(L, p);
    if (r == p) return;                         // a strong root already carries its flag
    L[p] = (int)(((unsigned)v & FLAG) | (unsigned)r);
    if ((unsigned)v & FLAG) atomicOr(L + r, (int)FLAG);
}

__global__ void __launch_bounds__(NT) canny_final_kernel(const int* labels, Img dst, int W, int H)
{
    const int blocks_x = (W + BX - 1) / BX;
    const int x = (blockIdx.x % blocks_x) * BX + threadIdx.x, y = (blockIdx.x / blocks_x) * BY + threadIdx.y;
    if (x >= W || y >= H) return;
    const int* L = labels + (size_t)blockIdx.z * W * H;
    const int v = L[y * W + x];
    const bool edge = v != NONE && ((unsigned)L[v & MASK] & FLAG);
    dst.row<uchar>(blockIdx.z, y)[x] = edge ? 255 : 0;
}

template <int KS, int CN>
static void launch_nms(const CannyArgs& a, dim3 grid, cudaStream_t st)
{
    canny_nms_kernel<KS, CN><<<grid, dim3(BX, BY), 0, st>>>(a);
}

// cvFloor as the reference's x86-64 build computes it: (int)__builtin_floor(v) is cvttsd2si, which gives INT_MIN for NaN and for any
// value outside the int range, of either sign (core/fast_math.hpp:231-235)
static int cv_floor_x86(double v)
{
    if (!(v >= -2147483648.0 && v < 2147483648.0)) return INT_MIN;
    return (int)std::floor(v);
}

}  // namespace

// cv::Canny's argument handling before the HAL call (canny.cpp:838-856): the legacy CV_CANNY_L2_GRADIENT bit, the aperture check, /16 for
// aperture 7 and the low/high swap.  The HAL entry receives thresholds already through this step.
int canny_user_args(double* low, double* high, int* aperture, int* l2)
{
    const int L2_BIT = (int)(1u << 31);
    int ap = *aperture;
    if (!*l2 && (ap & L2_BIT) == L2_BIT) { ap &= ~L2_BIT; *l2 = 1; }
    if ((ap & 1) == 0 || (ap != -1 && (ap < 3 || ap > 7))) {
        set_error("Canny: aperture size should be odd between 3 and 7, or -1 (Scharr); got %d", ap);
        return B200CV_ERR_BAD_ARG;
    }
    if (ap == 7) { *low = *low / 16.0; *high = *high / 16.0; }
    if (*low > *high) std::swap(*low, *high);
    *aperture = ap;
    return B200CV_OK;
}

// integer thresholds (canny.cpp:884-893): L2 clamps at 32767 and squares positive values, then cvFloor
static void canny_int_thresholds(double lo, double hi, bool l2, int* low, int* high)
{
    if (l2) {
        lo = std::min(32767.0, lo);
        hi = std::min(32767.0, hi);
        if (lo > 0) lo *= lo;
        if (hi > 0) hi *= hi;
    }
    *low = cv_floor_x86(lo);
    *high = cv_floor_x86(hi);
}

// thresholds after canny_user_args; dx_or_src is 8-bit (aperture 3/5/7/-1) or 16S with dy != NULL (the derivatives are given)
int canny_prepared(const b200cvMat* src, const b200cvMat* dy, const b200cvMat* dst, double lo, double hi, int aperture, int l2, void* stream)
{
    int rc;
    if ((rc = check_mat(src, dy ? "dx" : "src")) || (dy && (rc = check_mat(dy, "dy"))) || (rc = check_mat(dst, "dst"))) return rc;
    const int depth = B200CV_DEPTH(src->type), cn = B200CV_CN(src->type);
    if (dy) {
        if (depth != B200CV_16S || (cn != 1 && cn != 3)) { set_error("Canny(dx, dy): 16SC1 / 16SC3 derivatives only"); return B200CV_NOT_IMPLEMENTED; }
        B200_REQUIRE(dy->type == src->type && dy->cols == src->cols && dy->rows == src->rows &&
                     (dy->frames > 1 ? dy->frames : 1) == (src->frames > 1 ? src->frames : 1), "Canny: dx and dy differ in type or size");
    } else {
        if (depth != B200CV_8U || cn > 4) { set_error("Canny: 8-bit sources with 1 to 4 channels only"); return B200CV_NOT_IMPLEMENTED; }
    }
    B200_REQUIRE(dst->type == B200CV_MAKETYPE(B200CV_8U, 1) && dst->cols == src->cols && dst->rows == src->rows &&
                 (dst->frames > 1 ? dst->frames : 1) == (src->frames > 1 ? src->frames : 1), "Canny: dst must be 8UC1 of the source size");
    const int W = src->cols, H = src->rows;
    B200_REQUIRE((long long)W * H < (1ll << 31), "Canny: W * H must be below 2^31");
    const int frames = src->frames > 1 ? src->frames : 1;
    B200_REQUIRE(frames <= 65535, "Canny: at most 65535 frames per call");

    CannyArgs a;
    a.src = make_img(src);
    a.dst = make_img(dst);
    a.dy = dy ? make_img(dy) : a.src;
    a.l2 = l2 ? 1 : 0;
    canny_int_thresholds(lo, hi, l2 != 0, &a.low, &a.high);

    cudaStream_t st = as_stream(stream);
    const size_t n = (size_t)W * H;
    int* labels = nullptr;
    B200_CUDA(cudaMallocAsync(&labels, n * frames * sizeof(int), st));
    a.labels = labels;
    const dim3 tiles(div_up(W, TW) * div_up(H, TH), 1, frames);   // tiles along grid x (W * H < 2^31 keeps it in range)
    auto fail = [&](const char* what, int line) { cudaError_t e = cudaGetLastError(); cudaFreeAsync(labels, st); return cuda_fail(e, what, __FILE__, line); };

    if (dy) {
        if (cn == 1) launch_nms<0, 1>(a, tiles, st); else launch_nms<0, 3>(a, tiles, st);
    } else {
        const int ks = aperture < 0 ? 1 : aperture;
#define CANNY_CN(KS) switch (cn) { case 1: launch_nms<KS, 1>(a, tiles, st); break; case 2: launch_nms<KS, 2>(a, tiles, st); break; \
                                   case 3: launch_nms<KS, 3>(a, tiles, st); break; default: launch_nms<KS, 4>(a, tiles, st); }
        switch (ks) {
            case 1: CANNY_CN(1); break;
            case 3: CANNY_CN(3); break;
            case 5: CANNY_CN(5); break;
            case 7: CANNY_CN(7); break;
            default: cudaFreeAsync(labels, st); set_error("Canny: aperture %d", aperture); return B200CV_ERR_BAD_ARG;
        }
#undef CANNY_CN
    }
    count_launch();
    if (cudaPeekAtLastError() != cudaSuccess) return fail("canny_nms_kernel launch", __LINE__);
    canny_merge_kernel<<<tiles, 64, 0, st>>>(labels, W, H);
    count_launch();
    if (cudaPeekAtLastError() != cudaSuccess) return fail("canny_merge_kernel launch", __LINE__);
    canny_mark_kernel<<<dim3((unsigned)div_up_sz(n, 256), frames), 256, 0, st>>>(labels, (int)n);
    count_launch();
    if (cudaPeekAtLastError() != cudaSuccess) return fail("canny_mark_kernel launch", __LINE__);
    canny_final_kernel<<<dim3(div_up(W, BX) * div_up(H, BY), 1, frames), dim3(BX, BY), 0, st>>>(labels, a.dst, W, H);
    count_launch();
    if (cudaPeekAtLastError() != cudaSuccess) return fail("canny_final_kernel launch", __LINE__);
    B200_CUDA(cudaFreeAsync(labels, st));
    return B200CV_OK;
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_canny(const b200cvMat* src, const b200cvMat* dst, double threshold1, double threshold2, int aperture_size, int l2gradient,
                            void* stream)
{
    int rc, l2 = l2gradient ? 1 : 0;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    if (B200CV_DEPTH(src->type) != B200CV_8U || B200CV_CN(src->type) > 4) {
        set_error("Canny: 8-bit sources with 1 to 4 channels only");
        return B200CV_NOT_IMPLEMENTED;
    }
    if ((rc = canny_user_args(&threshold1, &threshold2, &aperture_size, &l2))) return rc;
    return canny_prepared(src, nullptr, dst, threshold1, threshold2, aperture_size, l2, stream);
}

extern "C" int b200cv_canny_derivs(const b200cvMat* dx, const b200cvMat* dy, const b200cvMat* dst, double threshold1, double threshold2,
                                   int l2gradient, void* stream)
{
    int rc;
    if ((rc = check_mat(dx, "dx")) || (rc = check_mat(dy, "dy"))) return rc;
    if (threshold1 > threshold2) std::swap(threshold1, threshold2);     // canny.cpp:944 (no /16 step on this overload)
    return canny_prepared(dx, dy, dst, threshold1, threshold2, 3, l2gradient ? 1 : 0, stream);
}
