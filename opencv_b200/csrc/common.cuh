// common.cuh -- shared device/host helpers for the b200cv kernels (sm_90a only).
#pragma once
#ifdef B200CV_HOST_EMULATION      // tests/emu/cuda_emu.h: simple kernels compiled for the host by tests/test_kernel_emulation.py
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <stdio.h>
#include "../../include/b200cv.h"

namespace b200cv {

typedef unsigned char uchar;

// ---- error plumbing -------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);
void count_launch(int n = 1);

#define B200_CUDA(call)                                                         \
    do {                                                                        \
        cudaError_t e__ = (call);                                               \
        if (e__ != cudaSuccess) return ::b200cv::cuda_fail(e__, #call, __FILE__, __LINE__); \
    } while (0)

#define B200_REQUIRE(cond, msg)                                                 \
    do {                                                                        \
        if (!(cond)) { ::b200cv::set_error("%s (%s)", msg, #cond); return B200CV_ERR_BAD_ARG; } \
    } while (0)

#define B200_LAUNCH_CHECK()                                                     \
    do {                                                                        \
        ::b200cv::count_launch();                                               \
        cudaError_t e__ = cudaGetLastError();                                   \
        if (e__ != cudaSuccess) return ::b200cv::cuda_fail(e__, "kernel launch", __FILE__, __LINE__); \
    } while (0)

static inline cudaStream_t as_stream(void* s) { return (cudaStream_t)s; }
int num_sms();
#ifdef B200CV_HOST_EMULATION
struct PerDeviceFlag { bool done = false; bool& cur() { return done; } };
#else
// "done once" state that exists PER DEVICE: kernel attributes (cudaFuncSetAttribute) and __device__ tables (cudaMemcpyToSymbol) belong to
// the device that was current when they were set; a process that drives several GPUs needs them on each.
struct PerDeviceFlag {
    bool done[64] = {};
    bool& cur() { int dev = 0; cudaGetDevice(&dev); return done[dev & 63]; }
};
#endif

// ---- device image descriptor (kernel parameter) -----------------------------------------------------------------
struct Img {
    uchar* data;
    size_t step;
    size_t fstep;
    int cols, rows, frames;
    template <typename T> __host__ __device__ __forceinline__ T* row(int f, int y) const {
        return (T*)(data + (size_t)f * fstep + (size_t)y * step);
    }
};

static inline Img make_img(const b200cvMat* m)
{
    Img i;
    i.data = (uchar*)m->data; i.step = m->step; i.cols = m->cols; i.rows = m->rows;
    i.frames = m->frames > 1 ? m->frames : 1;
    i.fstep = i.frames > 1 ? m->frame_step : 0;
    return i;
}

int check_mat(const b200cvMat* m, const char* name);
static inline size_t elem_size(int type) { int d = B200CV_DEPTH(type); return (size_t)B200CV_CN(type) * (d == 0 || d == 1 ? 1 : d == 2 || d == 3 ? 2 : d == 6 ? 8 : 4); }

// ---- cv::borderInterpolate (reference: modules/core/src/copy.cpp:748-793) --------------------------------------------
// returns -1 for BORDER_CONSTANT outside the image
__host__ __device__ __forceinline__ int border_interpolate(int p, int len, int border)
{
    if ((unsigned)p < (unsigned)len) return p;
    if (border == B200CV_BORDER_REPLICATE) return p < 0 ? 0 : len - 1;
    if (border == B200CV_BORDER_REFLECT || border == B200CV_BORDER_REFLECT_101) {
        int delta = border == B200CV_BORDER_REFLECT_101;
        if (len == 1) return 0;
        do {
            if (p < 0) p = -p - 1 + delta;
            else p = len - 1 - (p - len) - delta;
        } while ((unsigned)p >= (unsigned)len);
        return p;
    }
    if (border == B200CV_BORDER_WRAP) {
        if (p < 0) p -= ((p - len + 1) / len) * len;
        if (p >= len) p %= len;
        return p;
    }
    return -1;  // CONSTANT
}

// ---- saturate_cast family (reference: modules/core/include/opencv2/core/saturate.hpp:103-133) ---------------------------
__device__ __forceinline__ uchar sat_u8(int v) { return (uchar)min(max(v, 0), 255); }
// saturate_cast<uchar>(float) = cvRound (round-half-even) then clamp
__device__ __forceinline__ uchar sat_u8(float v) { return sat_u8(__float2int_rn(v)); }
__device__ __forceinline__ short sat_s16(int v) { return (short)min(max(v, -32768), 32767); }
__device__ __forceinline__ short sat_s16(float v) { return sat_s16(__float2int_rn(v)); }

template <typename T> struct OutCast;
template <> struct OutCast<uchar> { __device__ __forceinline__ static uchar from(float v) { return sat_u8(v); } };
template <> struct OutCast<short> { __device__ __forceinline__ static short from(float v) { return sat_s16(v); } };
template <> struct OutCast<float> { __device__ __forceinline__ static float from(float v) { return v; } };

#ifndef B200CV_HOST_EMULATION
// streaming (evict-first) 128-bit global accesses: every pixel is touched once per launch
__device__ __forceinline__ uint4 ldg_stream(const uint4* p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_stream(uint4* p, const uint4& v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
#endif

static inline unsigned div_up(unsigned a, unsigned b) { return (a + b - 1) / b; }
static inline size_t div_up_sz(size_t a, size_t b) { return (a + b - 1) / b; }

// ---- per-op implementation entry points (defined in the .cu files) -------------------------------------------------
struct SepTaps {           // up to 33 taps per direction, by value in kernel params
    float kx[33];
    float ky[33];
    int nx, ny, ax, ay;
};

// epilogue of cv::boxFilter on the 8-bit TMA kernel (gauss_u8.cu; box_filter.simd.hpp): sep_mode 2 = ColumnSum<ushort,uchar>,
// (s + div_delta) * div_scale >> 23; sep_mode 3 = ColumnSum<int,uchar>, cvRound(float(s) * scale_f) for elements < tail_from and
// cvRound(double(s) * scale) after them; !have_scale: saturate
struct GU8Box {
    int have_scale, tail_from;
    unsigned div_scale, div_delta;
    float scale_f;
    double scale;
};
int resize_lanczos_impl(const Img& s, const Img& d, int depth, int cn, cudaStream_t st);        // resize_lanczos.cu
int resize_exact_impl(const Img& s, const Img& d, int depth, int cn, int interpolation, cudaStream_t st);   // resize_exact.cu
int resize_area_impl(const Img& s, const Img& d, int depth, int cn, cudaStream_t st);           // resize_area.cu
int integral_impl(const b200cvMat* src, const b200cvMat* sum, const b200cvMat* sqsum, cudaStream_t st);   // integral.cu
int gauss_u16_impl(const Img& s, const Img& d, int cn, const long long* fx, int kw, const long long* fy, int kh, int border, cudaStream_t st);   // gauss_u16.cu
int gauss_u16_sep_impl(const Img& s, const Img& d, int cn, const long long* fx, int kw, const long long* fy, int kh, int border, cudaStream_t st);   // gauss_u16_sep.cu
int cvt_color_xyz(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st);        // cvtcolor_lab.cu
int cvt_color_lab(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st);        // cvtcolor_lab.cu
int demosaic_bilinear(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st);   // demosaic.cu
int cvt_color_two_plane(const b200cvMat* ysrc, const b200cvMat* uvsrc, const b200cvMat* dst, int code, cudaStream_t st);   // cvtcolor_yuv.cu
int cvt_color_yuv(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st);      // cvtcolor_yuv.cu
int cvt_color_depth(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st);    // cvtcolor_depth.cu (16U / 32F)
int gauss_u8_binomial(const Img& s, const Img& d, int cn, const int64_t* fx, int kw, const int64_t* fy, int kh, int border, cudaStream_t st);   // gauss_u8_binomial.cu
int gauss_u8_march(const Img& s, const Img& d, int KB, const unsigned char* tx, const unsigned char* ty, int border, cudaStream_t st, int sep_mode, int even_limit);   // gauss_u8_march.cu
int gauss_u8_fast(const Img& s, const Img& d, int cn, const int64_t* fx, int kw, const int64_t* fy, int kh, int border, cudaStream_t st, int sep_mode = 0, int even_limit = 0,
                  const GU8Box* box = nullptr);

}  // namespace b200cv
