// morph.cu -- cv::erode / cv::dilate / cv::morphologyEx (reference: modules/imgproc/src/morph.dispatch.cpp, morph.simd.hpp).
//
// Argument rules (morphOp and morphologyEx in the reference), applied on the host by resolve():
//   the anchor is normalised against the element ((-1, -1) is its centre; an empty element counts as 3x3) and must lie inside it;
//   iterations == 0 or a 1x1 element (even a zero one) copies src -- run here as a 1x1 pass;
//   cv::erode / cv::dilate with an empty element use a (1+2it) x (1+2it) rectangle anchored at (it, it), once (negative it: refused);
//   morphologyEx with an empty element uses a 3x3 rectangle (the caller passes op >= MORPH_OPEN, or the 3x3 mask itself);
//   an all-ones element with it > 1 grows to ksize + (it-1)(ksize-1), its anchor to anchor * it, and runs once;
//   any other element runs max(it, 1) passes, each reading the previous pass's output (its border included).
// Compound ops chain erodes and dilates through pooled scratch planes; GRADIENT, TOPHAT and BLACKHAT fuse their saturating subtraction
// into the store of the last pass.  The default CONSTANT border value is the reference's: UCHAR_MAX / USHRT_MAX / SHRT_MAX / FLT_MAX
// for erode, 0 / 0 / SHRT_MIN / -FLT_MAX for dilate; an explicit value is saturate_cast to the depth per channel.
//
// Two kernels:
//   morph_runs_kernel (one launch per pass): every non-rectangular element up to 63x63, and rectangles up to M_RECT_FUSED on both axes.
//     The element is split into horizontal runs per element row.  A CTA stages a tile of 32 output words (4, 2 or 1 elements each) by
//     TH rows plus the element's apron in shared memory, then for each distinct run length L (ascending) extends a shared plane of
//     horizontal run minima R_L from R_{L'} (the previous length) and folds every run of length L into per-thread accumulators.  A
//     rectangle is one length, kw, and kh runs: the separable row pass with the column pass fused.  Min / max act on whole 32-bit
//     words: __vminu4 / __vmaxu4 for 8U, __vminu2 / __vmins2 (and max) for 16U / 16S, fminf / fmaxf for 32F; an element offset that is
//     not a multiple of 4 bytes is read as a funnel shift of two words.
//   morph_vh_kernel (two launches per pass, through a pooled scratch plane): larger rectangles, one axis at a time, in the van Herk /
//     Gil-Werman form.  A thread owns a block of k outputs of one line: a suffix scan over the block and a prefix scan over the next,
//     about 3 min / max per output whatever k, and no apron in shared memory.
// Known limit (32F): the reference takes min / max with minps / maxps in its vector body and std::min / std::max in its scalar tail, so
// which operand wins when a window holds a NaN, or both -0.0 and +0.0, depends on the column.  Those windows are not reproduced.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>
#include "common.cuh"

namespace b200cv {

constexpr int M_MAXK = 63;               // largest non-rectangular element on each axis
constexpr int M_MAXRUNS = 63 * 32;       // 63 rows of at most 32 runs
constexpr int M_RECT_FUSED = 32;         // rectangles up to this size on both axes run the fused kernel
constexpr int M_TX = 32, M_TY = 8;       // a thread owns one output word column and the rows ty, ty + 8, ...
constexpr int M_TW = 32;                 // output words per tile row
constexpr int M_SMEM_MAX = 227 * 1024;

enum { FUSE_NONE = 0, FUSE_RES_MINUS_OTHER = 1, FUSE_OTHER_MINUS_RES = 2 };

struct MorphRuns {
    int cn, border, kh, ax, ay, TH, aw, fuse, nlen;
    unsigned bv[4];                          // CONSTANT border value per channel, as the element's bits
    unsigned char len[M_MAXK];               // distinct run lengths, ascending
    unsigned short first[M_MAXK + 1];       // the runs of len[l] are runs first[l] .. first[l + 1] - 1
    unsigned char rp[(3 * M_MAXRUNS + 1) / 2];  // run q: 12 bits from bit 12q, (element row << 6) | first column
};
// within the classic 4 KB kernel-parameter limit, so the kernel does not depend on large-parameter support
static_assert(sizeof(MorphRuns) <= 4096, "MorphRuns must fit in 4 KB of kernel parameters");

static void pack_run(MorphRuns& p, int q, int i, int j)
{
    const unsigned v = (unsigned)(i << 6 | j), b = (unsigned)(q * 3 / 2);
    if (q & 1) { p.rp[b] = (unsigned char)((p.rp[b] & 0x0F) | (v & 0x0F) << 4); p.rp[b + 1] = (unsigned char)(v >> 4); }
    else { p.rp[b] = (unsigned char)v; p.rp[b + 1] = (unsigned char)((p.rp[b + 1] & 0xF0) | v >> 8); }
}
__device__ __forceinline__ unsigned unpack_run(const MorphRuns& p, int q)
{
    const int b = q * 3 / 2;
    return (q & 1) ? (unsigned)(p.rp[b] >> 4 | p.rp[b + 1] << 4) : (unsigned)(p.rp[b] | (p.rp[b + 1] & 0x0F) << 8);
}

struct VHArgs {
    int k, a, cn, border, fuse;
    unsigned bv[4];
};

// ---- whole-word and element operations -----------------------------------------------------------------------------
template <typename T> struct WordOps;
template <> struct WordOps<uchar> {
    static __device__ __forceinline__ unsigned mn(unsigned a, unsigned b) { return __vminu4(a, b); }
    static __device__ __forceinline__ unsigned mx(unsigned a, unsigned b) { return __vmaxu4(a, b); }
    static __device__ __forceinline__ unsigned sub(unsigned a, unsigned b) { return __vsubus4(a, b); }
};
template <> struct WordOps<unsigned short> {
    static __device__ __forceinline__ unsigned mn(unsigned a, unsigned b) { return __vminu2(a, b); }
    static __device__ __forceinline__ unsigned mx(unsigned a, unsigned b) { return __vmaxu2(a, b); }
    static __device__ __forceinline__ unsigned sub(unsigned a, unsigned b) { return __vsubus2(a, b); }
};
template <> struct WordOps<short> {
    static __device__ __forceinline__ unsigned mn(unsigned a, unsigned b) { return __vmins2(a, b); }
    static __device__ __forceinline__ unsigned mx(unsigned a, unsigned b) { return __vmaxs2(a, b); }
    static __device__ __forceinline__ unsigned sub(unsigned a, unsigned b) { return __vsubss2(a, b); }
};
template <> struct WordOps<float> {
    static __device__ __forceinline__ unsigned mn(unsigned a, unsigned b) { return __float_as_uint(fminf(__uint_as_float(a), __uint_as_float(b))); }
    static __device__ __forceinline__ unsigned mx(unsigned a, unsigned b) { return __float_as_uint(fmaxf(__uint_as_float(a), __uint_as_float(b))); }
    // x86 subss: a NaN operand comes back quieted (the first one first); inf - inf is the default NaN 0xFFC00000, as in the reference
    static __device__ __forceinline__ unsigned sub(unsigned a, unsigned b)
    {
        const float fa = __uint_as_float(a), fb = __uint_as_float(b), r = __fsub_rn(fa, fb);
        if (!isnan(r)) return __float_as_uint(r);
        return isnan(fa) ? (a | 0x400000u) : isnan(fb) ? (b | 0x400000u) : 0xFFC00000u;
    }
};
template <typename T, bool MAX> __device__ __forceinline__ unsigned wop(unsigned a, unsigned b)
{
    return MAX ? WordOps<T>::mx(a, b) : WordOps<T>::mn(a, b);
}

template <typename T> __device__ __forceinline__ unsigned to_bits(T v)
{
    if constexpr (sizeof(T) == 4) return __float_as_uint(v);
    else if constexpr (sizeof(T) == 2) return (unsigned short)v;
    else return (unsigned)v;
}
template <typename T> __device__ __forceinline__ T from_bits(unsigned b)
{
    if constexpr (sizeof(T) == 4) return __uint_as_float(b);
    else return (T)b;
}
// one element of the scalar van Herk path, through the word operations (lane 0 of a word)
template <typename T, bool MAX> __device__ __forceinline__ T eop(T a, T b) { return from_bits<T>(wop<T, MAX>(to_bits(a), to_bits(b))); }
template <typename T> __device__ __forceinline__ T esub(T a, T b) { return from_bits<T>(WordOps<T>::sub(to_bits(a), to_bits(b))); }

// the 32-bit word that starts `boff` bytes after p (p word-aligned)
__device__ __forceinline__ unsigned ld_shift(const unsigned* p, int boff)
{
    const unsigned* q = p + (boff >> 2);
    const int s = boff & 3;
    return s ? __funnelshift_r(q[0], q[1], 8 * s) : q[0];
}

// ---- fused kernel: staged tile, run planes, accumulators -------------------------------------------------------------
template <typename T, bool MAX>
__global__ void __launch_bounds__(M_TX * M_TY) morph_runs_kernel(Img src, Img dst, Img other, const __grid_constant__ MorphRuns p)
{
    constexpr int EPW = 4 / sizeof(T);
    extern __shared__ __align__(16) unsigned sm[];
    const int cn = p.cn, TH = p.TH, nk = TH / M_TY;
    const int IW = M_TW + p.aw + 2, RWMAX = M_TW + p.aw + 1;
    const int rows = TH + p.kh - 1;
    unsigned* s_in = sm;                          // rows x IW words: the source tile and its apron
    unsigned* s_r = sm + rows * IW;               // rows x RWMAX words: horizontal run minima of the current length
    const int f = blockIdx.z;
    const int e0 = blockIdx.x * M_TW * EPW;       // first output element of the tile (row-major, channels interleaved)
    const int y0 = blockIdx.y * TH;
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * M_TX + tx;

    for (int r = ty; r < rows; r += M_TY) {
        const int sy = border_interpolate(y0 + r - p.ay, src.rows, p.border);
        const T* srow = sy < 0 ? nullptr : src.row<T>(f, sy);
        T* d = (T*)(s_in + r * IW);
        for (int e = tx; e < IW * EPW; e += M_TX) {
            const int ge = e0 + e - p.ax * cn;                        // element index in the source row, negative left of it
            const int px = ge >= 0 ? ge / cn : -((cn - 1 - ge) / cn);
            const int c = ge - px * cn;
            const int sx = border_interpolate(px, src.cols, p.border);
            d[e] = (srow == nullptr || sx < 0) ? from_bits<T>(p.bv[c]) : srow[(size_t)sx * cn + c];
        }
    }

    unsigned acc[4] = {0u, 0u, 0u, 0u};
    const int esz_cn = cn * (int)sizeof(T);       // bytes per pixel
    int prev = 0;
    for (int l = 0; l < p.nlen; l++) {
        const int L = p.len[l];
        // R_L is read at word offsets up to (kw - L) pixels right of the tile's last word; it reads the tile up to L - 1 pixels further
        const int rw = M_TW + (int)(((p.aw * EPW - (L - 1) * cn) + EPW - 1) / EPW) + 1;
        __syncthreads();
        for (int i = tid; i < rows * rw; i += M_TX * M_TY) {
            const int r = i / rw, w = i - r * rw;
            const unsigned* in = s_in + r * IW + w;
            unsigned v = prev == 0 ? in[0] : s_r[r * RWMAX + w];
            for (int d = prev == 0 ? 1 : prev; d < L; d++) v = wop<T, MAX>(v, ld_shift(in, d * esz_cn));
            s_r[r * RWMAX + w] = v;
        }
        prev = L;
        __syncthreads();
        for (int q = p.first[l]; q < p.first[l + 1]; q++) {
            const unsigned r = unpack_run(p, q);
            const int i = (int)(r >> 6), boff = (int)(r & 63) * esz_cn;
            const bool init = l == 0 && q == 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                if (k < nk) {
                    const unsigned v = ld_shift(s_r + (ty + k * M_TY + i) * RWMAX + tx, boff);
                    acc[k] = init ? v : wop<T, MAX>(acc[k], v);
                }
            }
        }
    }

    const int we = dst.cols * cn, eb = e0 + tx * EPW;
    if (eb >= we) return;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int y = y0 + ty + k * M_TY;
        if (k >= nk || y >= dst.rows) break;
        unsigned v = acc[k];
        if (p.fuse != FUSE_NONE) {
            const T* orow = other.row<T>(f, y);
            unsigned o = 0;
#pragma unroll
            for (int u = 0; u < EPW; u++)
                if (eb + u < we) o |= to_bits(orow[eb + u]) << (u * 8 * sizeof(T) & 31);
            v = p.fuse == FUSE_RES_MINUS_OTHER ? WordOps<T>::sub(v, o) : WordOps<T>::sub(o, v);
        }
        T* drow = dst.row<T>(f, y);
#pragma unroll
        for (int u = 0; u < EPW; u++) {
            if (eb + u >= we) break;
            if constexpr (sizeof(T) == 4) drow[eb + u] = from_bits<T>(v);
            else drow[eb + u] = from_bits<T>((v >> (u * 8 * sizeof(T))) & ((1u << (8 * sizeof(T))) - 1u));
        }
    }
}

// ---- van Herk / Gil-Werman pass along one axis ---------------------------------------------------------------------
// out[x] = op over g[x .. x + k - 1], g[q] = the source at border_interpolate(q - a) along the line (the border value outside for
// CONSTANT).  A thread owns the outputs [bk, bk + k) of one line: a suffix scan S over g[bk .. bk + k) stored in place, then a prefix
// scan P over g[bk + k .. bk + 2k - 1) combined as out[x] = op(S[x], P[x + k - 1]).
template <typename T, bool MAX, bool COL>
__global__ void __launch_bounds__(256) morph_vh_kernel(Img src, Img dst, Img other, const VHArgs p)
{
    const int cn = p.cn, k = p.k;
    const int len = COL ? src.rows : src.cols;
    const int nb = (len + k - 1) / k;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int f = blockIdx.z;
    int e, c, y, b;
    if (COL) {                        // a line is one element column; neighbouring threads read neighbouring elements
        const int we = src.cols * cn;
        if (t >= (long long)we * nb) return;
        e = (int)(t % we); b = (int)(t / we); c = e % cn; y = 0;
    } else {                          // a line is one channel of one row
        if (t >= (long long)src.rows * cn * nb) return;
        c = (int)(t % cn);
        const long long rest = t / cn;
        y = (int)(rest % src.rows); b = (int)(rest / src.rows); e = 0;
    }
    const T bv = from_bits<T>(c == 0 ? p.bv[0] : c == 1 ? p.bv[1] : c == 2 ? p.bv[2] : p.bv[3]);
    auto g = [&](int q) -> T {
        const int s = border_interpolate(q - p.a, len, p.border);
        if (s < 0) return bv;
        return COL ? src.row<T>(f, s)[e] : src.row<T>(f, y)[(size_t)s * cn + c];
    };
    auto at = [&](int x) -> T* { return COL ? dst.row<T>(f, x) + e : dst.row<T>(f, y) + (size_t)x * cn + c; };
    auto fin = [&](T v, int x) -> T {
        if (p.fuse == FUSE_NONE) return v;
        const T o = COL ? other.row<T>(f, x)[e] : other.row<T>(f, y)[(size_t)x * cn + c];
        return p.fuse == FUSE_RES_MINUS_OTHER ? esub(v, o) : esub(o, v);
    };
    const int bk = b * k;
    T s = g(bk + k - 1);
    for (int x = bk + k - 1;; x--) {
        if (x < bk + k - 1) s = eop<T, MAX>(s, g(x));
        if (x < len) *at(x) = x == bk ? fin(s, x) : s;
        if (x == bk) break;
    }
    T pr = s;
    for (int q = bk + k; q < bk + 2 * k - 1 && q - k + 1 < len; q++) {
        pr = q == bk + k ? g(q) : eop<T, MAX>(pr, g(q));
        const int x = q - k + 1;
        *at(x) = fin(eop<T, MAX>(*at(x), pr), x);
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------------
static int cv_round(double v)         // cvRound as x86 cvtsd2si: half to even; NaN and anything outside int32 give INT_MIN
{
    const double r = std::nearbyint(v);
    return (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : INT_MIN;
}

// the CONSTANT border value of channel c as the element's bits
static unsigned border_bits(int depth, bool is_max, const double bv[4], int c)
{
    const bool dflt = bv == nullptr || (bv[0] == DBL_MAX && bv[1] == DBL_MAX && bv[2] == DBL_MAX && bv[3] == DBL_MAX);
    if (depth == B200CV_32F) {
        float f = dflt ? (is_max ? -FLT_MAX : FLT_MAX) : (float)bv[c];
        unsigned u;
        std::memcpy(&u, &f, 4);
        return u;
    }
    int v;
    if (dflt) v = depth == B200CV_8U ? (is_max ? 0 : UCHAR_MAX) : depth == B200CV_16U ? (is_max ? 0 : USHRT_MAX) : (is_max ? SHRT_MIN : SHRT_MAX);
    else {
        v = cv_round(bv[c]);
        const int lo = depth == B200CV_16S ? SHRT_MIN : 0, hi = depth == B200CV_8U ? UCHAR_MAX : depth == B200CV_16U ? USHRT_MAX : SHRT_MAX;
        v = std::min(std::max(v, lo), hi);
    }
    return depth == B200CV_16S ? (unsigned)(unsigned short)(short)v : (unsigned)v;
}

// A window of a rectangle reaches `a` pixels before its output and k - 1 - a after it.  Reaching more than 2 * len pixels past either
// end of a line of len pixels adds no value the window does not already hold: every output's window holds [0, x] or [x, len - 1], and
// 2 * len positions past an end cover a whole period of every border rule (a constant for CONSTANT).  So k and a shrink to that
// reach, which bounds the van Herk kernel's serial walk by the image instead of by iterations.  false: the positions the kernel walks
// (up to len + 2k) would not fit in an int.
static bool vh_extent(int& k, int& a, int len)
{
    const long long reach = 2LL * len;
    const long long a2 = std::min<long long>(a, reach), r2 = std::min<long long>((long long)k - 1 - a, reach);
    const long long k2 = a2 + r2 + 1;
    if (len + 2 * k2 + 2 > INT_MAX) return false;
    k = (int)k2;
    a = (int)a2;
    return true;
}

struct Element {
    int kw = 1, kh = 1, ax = 0, ay = 0, passes = 1;
    bool rect = true;
    std::vector<uchar> m;            // kh x kw, 0 / 1
};

static size_t runs_smem(int aw, int kh, int TH)
{
    return (size_t)(TH + kh - 1) * (2 * M_TW + 2 * aw + 3) * sizeof(unsigned);
}

template <typename T>
struct MorphCall {
    Img s, d;
    int depth, cn, border;
    const double* bv;
    Element el;
    bool fused;
    MorphRuns runs;
    int esz;
    cudaStream_t st;

    void prepare_runs()
    {
        constexpr int EPW = 4 / sizeof(T);
        std::vector<std::pair<int, std::pair<int, int>>> all;      // (length, (row, first column))
        for (int i = 0; i < el.kh; i++)
            for (int j = 0; j < el.kw;) {
                if (el.rect) { all.push_back({el.kw, {i, 0}}); break; }     // grown and empty-element rectangles keep no mask
                if (!el.m[(size_t)i * el.kw + j]) { j++; continue; }
                int j2 = j;
                while (j2 < el.kw && el.m[(size_t)i * el.kw + j2]) j2++;
                all.push_back({j2 - j, {i, j}});
                j = j2;
            }
        std::stable_sort(all.begin(), all.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
        memset(&runs, 0, sizeof(runs));
        runs.nlen = 0;
        for (size_t q = 0; q < all.size(); q++) {
            if (q == 0 || all[q].first != all[q - 1].first) {
                runs.len[runs.nlen] = (unsigned char)all[q].first;
                runs.first[runs.nlen] = (unsigned short)q;
                runs.nlen++;
            }
            pack_run(runs, (int)q, all[q].second.first, all[q].second.second);
        }
        runs.first[runs.nlen] = (unsigned short)all.size();
        runs.cn = cn; runs.border = border; runs.kh = el.kh; runs.ax = el.ax; runs.ay = el.ay;
        runs.aw = (int)div_up((unsigned)((el.kw - 1) * cn), (unsigned)EPW);
        runs.TH = 32;
        while (runs.TH > 8 && runs_smem(runs.aw, el.kh, runs.TH) > 64 * 1024) runs.TH /= 2;
    }

    template <bool MAX> int launch_runs(const Img& in, const Img& out, int fuse, const Img& other)
    {
        constexpr int EPW = 4 / sizeof(T);
        MorphRuns p = runs;
        p.fuse = fuse;
        for (int c = 0; c < 4; c++) p.bv[c] = border_bits(depth, MAX, bv, c < cn ? c : 0);
        const size_t smem = runs_smem(p.aw, p.kh, p.TH);
        B200_REQUIRE(smem <= (size_t)M_SMEM_MAX, "morphology: element tile exceeds shared memory");
        auto kern = morph_runs_kernel<T, MAX>;
        static PerDeviceFlag attr_pd;
        bool& attr = attr_pd.cur();
        if (!attr) { B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, M_SMEM_MAX)); attr = true; }
        dim3 grid(div_up((unsigned)(in.cols * cn), (unsigned)(M_TW * EPW)), div_up((unsigned)in.rows, (unsigned)p.TH), (unsigned)in.frames);
        kern<<<grid, dim3(M_TX, M_TY), smem, st>>>(in, out, other, p);
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }

    template <bool MAX> int launch_vh(const Img& in, const Img& out, int fuse, const Img& other, const Img& mid)
    {
        VHArgs a;
        a.cn = cn; a.border = border;
        for (int c = 0; c < 4; c++) a.bv[c] = border_bits(depth, MAX, bv, c < cn ? c : 0);
        a.k = el.kw; a.a = el.ax; a.fuse = FUSE_NONE;
        const long long nrow = (long long)in.rows * cn * div_up((unsigned)in.cols, (unsigned)el.kw);
        morph_vh_kernel<T, MAX, false><<<dim3((unsigned)div_up_sz((size_t)nrow, 256), 1, (unsigned)in.frames), 256, 0, st>>>(in, mid, other, a);
        B200_LAUNCH_CHECK();
        a.k = el.kh; a.a = el.ay; a.fuse = fuse;
        const long long ncol = (long long)in.cols * cn * div_up((unsigned)in.rows, (unsigned)el.kh);
        morph_vh_kernel<T, MAX, true><<<dim3((unsigned)div_up_sz((size_t)ncol, 256), 1, (unsigned)in.frames), 256, 0, st>>>(mid, out, other, a);
        B200_LAUNCH_CHECK();
        return B200CV_OK;
    }

    int pass(bool is_max, const Img& in, const Img& out, int fuse, const Img& other, const Img& mid)
    {
        if (fused) return is_max ? launch_runs<true>(in, out, fuse, other) : launch_runs<false>(in, out, fuse, other);
        return is_max ? launch_vh<true>(in, out, fuse, other, mid) : launch_vh<false>(in, out, fuse, other, mid);
    }

    // el.passes passes from `in` to `out`; passes between go through a / b; the last one fuses the subtraction
    int chain(bool is_max, const Img& in, const Img& out, int fuse, const Img& other, const Img* pp, const Img& mid)
    {
        int rc;
        for (int i = 0; i < el.passes; i++) {
            const Img& pin = i == 0 ? in : pp[(i - 1) & 1];
            const bool last = i == el.passes - 1;
            const Img& pout = last ? out : pp[i & 1];
            if ((rc = pass(is_max, pin, pout, last ? fuse : FUSE_NONE, other, mid))) return rc;
        }
        return B200CV_OK;
    }

    int run(int op)
    {
        fused = !el.rect || (el.kw <= M_RECT_FUSED && el.kh <= M_RECT_FUSED);
        if (fused) prepare_runs();
        else if (!vh_extent(el.kw, el.ax, s.cols) || !vh_extent(el.kh, el.ay, s.rows)) {
            set_error("morphology: a rectangle this large on a line of this length overflows the kernel's int positions");
            return B200CV_NOT_IMPLEMENTED;
        }
        const bool compound = op >= B200CV_MORPH_OPEN;
        const int nplanes = (fused ? 0 : 1) + std::min(el.passes - 1, 2) + (compound ? 1 : 0);
        Img plane = s;
        plane.step = (size_t)s.cols * esz;
        plane.fstep = plane.step * s.rows;
        const size_t pbytes = plane.fstep * s.frames;
        if (s.frames <= 1) plane.fstep = 0;
        uchar* scratch = nullptr;
        if (nplanes > 0) B200_CUDA(cudaMallocAsync(&scratch, pbytes * nplanes, st));
        Img pl[4];
        for (int i = 0; i < nplanes; i++) { pl[i] = plane; pl[i].data = scratch + pbytes * i; }
        int q = 0;
        const Img mid = fused ? Img{} : pl[q++];
        Img pp[2] = {Img{}, Img{}};
        for (int i = 0; i < std::min(el.passes - 1, 2); i++) pp[i] = pl[q++];
        const Img tmp = compound ? pl[q++] : Img{};
        int rc;
        switch (op) {
        case B200CV_MORPH_ERODE: rc = chain(false, s, d, FUSE_NONE, s, pp, mid); break;
        case B200CV_MORPH_DILATE: rc = chain(true, s, d, FUSE_NONE, s, pp, mid); break;
        case B200CV_MORPH_OPEN:
            if (!(rc = chain(false, s, tmp, FUSE_NONE, s, pp, mid))) rc = chain(true, tmp, d, FUSE_NONE, s, pp, mid);
            break;
        case B200CV_MORPH_CLOSE:
            if (!(rc = chain(true, s, tmp, FUSE_NONE, s, pp, mid))) rc = chain(false, tmp, d, FUSE_NONE, s, pp, mid);
            break;
        case B200CV_MORPH_GRADIENT:        // dilate(src) - erode(src)
            if (!(rc = chain(false, s, tmp, FUSE_NONE, s, pp, mid))) rc = chain(true, s, d, FUSE_RES_MINUS_OTHER, tmp, pp, mid);
            break;
        case B200CV_MORPH_TOPHAT:          // src - open(src)
            if (!(rc = chain(false, s, tmp, FUSE_NONE, s, pp, mid))) rc = chain(true, tmp, d, FUSE_OTHER_MINUS_RES, s, pp, mid);
            break;
        default:                           // BLACKHAT: close(src) - src
            if (!(rc = chain(true, s, tmp, FUSE_NONE, s, pp, mid))) rc = chain(false, tmp, d, FUSE_RES_MINUS_OTHER, s, pp, mid);
            break;
        }
        if (scratch) cudaFreeAsync(scratch, st);
        return rc;
    }
};

// cv::morphOp's element rules; B200CV_OK with `el` filled, or the refusal
static int resolve(int op, const unsigned char* kdata, size_t kstep, int kw, int kh, int ax, int ay, int it, Element& el)
{
    bool empty = kdata == nullptr || kw <= 0 || kh <= 0;
    std::vector<uchar> m;
    if (empty && op >= B200CV_MORPH_OPEN) {          // morphologyEx: a 3x3 rectangle, then the rules below
        empty = false;
        kw = kh = 3;
        m.assign(9, 1);
    } else if (!empty) {
        m.resize((size_t)kw * kh);
        for (int i = 0; i < kh; i++)
            for (int j = 0; j < kw; j++) m[(size_t)i * kw + j] = kdata[(size_t)i * kstep + j] != 0;
    }
    const int sw = empty ? 3 : kw, sh = empty ? 3 : kh;
    if (ax == -1) ax = sw / 2;
    if (ay == -1) ay = sh / 2;
    B200_REQUIRE(ax >= 0 && ax < sw && ay >= 0 && ay < sh, "morphology: the anchor must lie inside the element");
    if (it == 0 || (!empty && kw * kh == 1)) {      // a copy
        el = Element();
        el.m.assign(1, 1);
        return B200CV_OK;
    }
    if (empty) {
        B200_REQUIRE(it > 0 && it <= (INT_MAX - 1) / 2, "morphology: an empty element needs 1 <= iterations");
        el.kw = el.kh = 1 + 2 * it;
        el.ax = el.ay = it;
        el.rect = true;
        el.passes = 1;
        return B200CV_OK;
    }
    size_t nz = 0;
    for (uchar v : m) nz += v;
    B200_REQUIRE(nz > 0, "morphology: an element larger than 1x1 needs a non-zero entry");
    el.rect = nz == m.size();
    if (el.rect && it > 1) {
        const long long gw = kw + (long long)(it - 1) * (kw - 1), gh = kh + (long long)(it - 1) * (kh - 1);
        B200_REQUIRE(gw <= INT_MAX && gh <= INT_MAX && (long long)ax * it <= INT_MAX && (long long)ay * it <= INT_MAX,
                     "morphology: the grown element is too large");
        el.kw = (int)gw; el.kh = (int)gh; el.ax = ax * it; el.ay = ay * it;
        el.passes = 1;
        return B200CV_OK;
    }
    el.kw = kw; el.kh = kh; el.ax = ax; el.ay = ay;
    el.passes = el.rect ? 1 : std::max(it, 1);
    el.m = std::move(m);
    if (!el.rect && (kw > M_MAXK || kh > M_MAXK)) return B200CV_NOT_IMPLEMENTED;
    return B200CV_OK;
}

static void byte_range(const b200cvMat* m, uintptr_t& lo, uintptr_t& hi)
{
    const int frames = m->frames > 1 ? m->frames : 1;
    lo = (uintptr_t)m->data;
    hi = lo + (size_t)(frames - 1) * m->frame_step + (size_t)(m->rows - 1) * m->step + (size_t)m->cols * elem_size(m->type);
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_morphology(const b200cvMat* src, const b200cvMat* dst, int op, const unsigned char* kernel_data, size_t kernel_step,
                                 int kw, int kh, int anchor_x, int anchor_y, int iterations, int border, const double border_value[4],
                                 void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src")) || (rc = check_mat(dst, "dst"))) return rc;
    if (op == B200CV_MORPH_HITMISS) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(op >= B200CV_MORPH_ERODE && op <= B200CV_MORPH_BLACKHAT, "morphology: unknown operation");
    const int depth = B200CV_DEPTH(src->type), cn = B200CV_CN(src->type);
    if (depth != B200CV_8U && depth != B200CV_16U && depth != B200CV_16S && depth != B200CV_32F) return B200CV_NOT_IMPLEMENTED;
    if (cn > 4) return B200CV_NOT_IMPLEMENTED;
    border &= ~B200CV_BORDER_ISOLATED;      // a device view has no parent image to read past its edges
    if (border == B200CV_BORDER_WRAP) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(border >= B200CV_BORDER_CONSTANT && border <= B200CV_BORDER_REFLECT_101, "morphology: unknown border type");
    B200_REQUIRE(src->type == dst->type && src->cols == dst->cols && src->rows == dst->rows, "src/dst type or size mismatch");
    B200_REQUIRE((long long)src->cols * src->rows < (1LL << 31), "morphology: W * H must stay below 2^31");
    B200_REQUIRE((long long)(src->cols + 2 * M_TW + 2 * M_MAXK) * cn < (1LL << 31), "morphology: a row of W * cn elements must stay below 2^31");
    B200_REQUIRE(kernel_data == nullptr || kw <= 0 || kh <= 0 || kernel_step >= (size_t)kw, "morphology: kernel_step < kw");
    Img s = make_img(src), d = make_img(dst);
    B200_REQUIRE(s.frames == d.frames, "src/dst batch mismatch");
    B200_REQUIRE(s.frames <= 65535, "morphology: at most 65535 frames per call");
    uintptr_t slo, shi, dlo, dhi;
    byte_range(src, slo, shi);
    byte_range(dst, dlo, dhi);
    B200_REQUIRE(shi <= dlo || dhi <= slo, "morphology: src and dst overlap (in-place calls are not supported)");
    Element el;
    if ((rc = resolve(op, kernel_data, kernel_step, kw, kh, anchor_x, anchor_y, iterations, el))) return rc;
    cudaStream_t st = as_stream(stream);
    switch (depth) {
    case B200CV_8U: { MorphCall<uchar> c{s, d, depth, cn, border, border_value, el}; c.esz = cn; c.st = st; return c.run(op); }
    case B200CV_16U: { MorphCall<unsigned short> c{s, d, depth, cn, border, border_value, el}; c.esz = 2 * cn; c.st = st; return c.run(op); }
    case B200CV_16S: { MorphCall<short> c{s, d, depth, cn, border, border_value, el}; c.esz = 2 * cn; c.st = st; return c.run(op); }
    default: { MorphCall<float> c{s, d, depth, cn, border, border_value, el}; c.esz = 4 * cn; c.st = st; return c.run(op); }
    }
}
