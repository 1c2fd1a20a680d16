/*
 * b200cv.h -- C ABI of the H100-native dense-imgproc hot path (OpenCV drop-in boundary).
 *
 * Plain C: pointers, sizes, ints, doubles.  No C++ / torch / OpenCV types cross this line.
 * Everything above it (the cv::-signature C++ mirror in opencv_b200/host/, the cv_hal_*
 * replacement header include/b200cv_hal.h, the Python ctypes binding) is a thin caller.
 *
 * Two families of entry points:
 *
 *  (1) b200cv_*        -- DEVICE API.  Images are b200cvMat descriptors over device memory
 *                         (row-major, interleaved channels, `step` bytes per row -- the cv::Mat /
 *                         cv::cuda::GpuMat layout, reference: modules/core/include/opencv2/core/mat.hpp:2151-2178,
 *                         modules/core/include/opencv2/core/cuda.hpp:105-340).  A descriptor can describe a
 *                         BATCH of `frames` equally-shaped frames `frame_step` bytes apart: independent
 *                         frames are processed by one launch (grid z / persistent tile loop).  Work is
 *                         enqueued on `stream` (a cudaStream_t passed as void*, NULL = legacy default
 *                         stream) and the call returns without synchronising, like cv::cuda::* functions
 *                         taking a cv::cuda::Stream& (cuda.hpp:909-975).
 *
 *  (2) b200cv_hal_*    -- HOST API with the exact argument lists of the reference's imgproc HAL seam
 *                         (modules/imgproc/src/hal_replacement.hpp): raw host pointers + step, synchronous,
 *                         result in `dst` on return.  Declared in include/b200cv_hal.h.
 *
 * Return convention = the HAL's (modules/core/include/opencv2/core/hal/interface.h:9-11):
 *   0  B200CV_OK               done
 *   1  B200CV_NOT_IMPLEMENTED  unsupported type/border/size: caller should use its own path
 *  <0  error (bad argument / CUDA failure); b200cv_last_error() returns a thread-local message.
 * There is NO CPU fallback anywhere behind this ABI.
 *
 * Type / border / interpolation / colour codes are numerically OpenCV's:
 *   type   = CV_MAKETYPE(depth, cn)   depth: CV_8U=0 CV_16S=3 CV_32F=5        (core/hal/interface.h:70-85)
 *   border = CV_HAL_BORDER_*          CONSTANT 0 REPLICATE 1 REFLECT 2 WRAP 3 REFLECT_101 4 (:151-157)
 *   interp = CV_HAL_INTER_*           NEAREST 0 LINEAR 1 CUBIC 2 AREA 3; WARP_INVERSE_MAP 16 (imgproc/hal/interface.h:10-20)
 *   code   = cv::ColorConversionCodes (imgproc.hpp:538-642)
 *   method = cv::TemplateMatchModes   (imgproc.hpp:3845-3879)
 */
#ifndef B200CV_H
#define B200CV_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200CV_API __attribute__((visibility("default")))
#else
#define B200CV_API
#endif

#define B200CV_OK 0
#define B200CV_NOT_IMPLEMENTED 1
#define B200CV_ERR_BAD_ARG (-2)
#define B200CV_ERR_CUDA (-3)
#define B200CV_ERR_NO_DEVICE (-4)

/* depth / type codes (== CV_8U ...) */
#define B200CV_8U 0
#define B200CV_16U 2
#define B200CV_16S 3
#define B200CV_32S 4
#define B200CV_32F 5
#define B200CV_64F 6
#define B200CV_MAKETYPE(depth, cn) (((depth) & 7) + (((cn) - 1) << 3))
#define B200CV_DEPTH(type) ((type) & 7)
#define B200CV_CN(type) ((((type) >> 3) & 511) + 1)

#define B200CV_BORDER_CONSTANT 0
#define B200CV_BORDER_REPLICATE 1
#define B200CV_BORDER_REFLECT 2
#define B200CV_BORDER_WRAP 3
#define B200CV_BORDER_REFLECT_101 4
#define B200CV_BORDER_TRANSPARENT 5
#define B200CV_BORDER_ISOLATED 16

#define B200CV_INTER_NEAREST 0
#define B200CV_INTER_LINEAR 1
#define B200CV_INTER_CUBIC 2
#define B200CV_INTER_AREA 3
#define B200CV_INTER_LANCZOS4 4
#define B200CV_INTER_LINEAR_EXACT 5
#define B200CV_INTER_NEAREST_EXACT 6
#define B200CV_WARP_INVERSE_MAP 16
#define B200CV_WARP_RELATIVE_MAP 32

#define B200CV_TM_SQDIFF 0
#define B200CV_TM_SQDIFF_NORMED 1
#define B200CV_TM_CCORR 2
#define B200CV_TM_CCORR_NORMED 3
#define B200CV_TM_CCOEFF 4
#define B200CV_TM_CCOEFF_NORMED 5

/* A (batch of) device image(s).  frames<=1 means a single frame (frame_step ignored). */
typedef struct b200cvMat {
    void*  data;        /* device pointer to pixel (0,0) of frame 0 */
    size_t step;        /* bytes per row */
    int    cols;        /* width in pixels */
    int    rows;        /* height in pixels */
    int    type;        /* CV_MAKETYPE(depth, cn) */
    int    frames;      /* number of frames in the batch (>=1) */
    size_t frame_step;  /* bytes between consecutive frames */
} b200cvMat;

/* ---- runtime ---------------------------------------------------------------------------------------------- */
/* replaces: cv::cuda::setDevice / getCudaEnabledDeviceCount (core/include/opencv2/core/cuda.hpp:1040-1060) */
B200CV_API int b200cv_init(int device);
B200CV_API int b200cv_device_count(void);
B200CV_API const char* b200cv_last_error(void);
B200CV_API const char* b200cv_version(void);
/* number of b200cv kernels launched by this process so far (bench.py's gpu_launches) */
B200CV_API unsigned long long b200cv_launch_count(void);

/* replaces: cv::cuda::GpuMat::Allocator::allocate/free (cuda.hpp:108-115; default = cudaMallocPitch, core/src/cuda/gpu_mat.cu:116).
 * Pitch is rounded up to 256 B so every row is TMA-addressable. */
B200CV_API int b200cv_malloc_pitch(void** dptr, size_t* step, size_t width_bytes, size_t rows);
B200CV_API int b200cv_free(void* dptr);
/* replaces: cv::cuda::HostMem (cuda.hpp:791-870): page-locked host allocation */
B200CV_API int b200cv_host_alloc(void** hptr, size_t bytes);
B200CV_API int b200cv_host_free(void* hptr);
/* replaces: GpuMat::upload / download (cuda.hpp:160-190; core/src/cuda/gpu_mat.cu:228-288) */
B200CV_API int b200cv_upload(const void* hsrc, size_t hstep, void* ddst, size_t dstep, size_t width_bytes, size_t rows, void* stream);
B200CV_API int b200cv_download(const void* dsrc, size_t dstep, void* hdst, size_t hstep, size_t width_bytes, size_t rows, void* stream);

/* replaces: cv::cuda::Stream (cuda.hpp:909-975) and cv::cuda::Event (cuda.hpp:984-1016) */
B200CV_API int b200cv_stream_create(void** stream);
B200CV_API int b200cv_stream_destroy(void* stream);
B200CV_API int b200cv_stream_query(void* stream);              /* 0 = complete, 1 = still running (Stream::queryIfComplete) */
B200CV_API int b200cv_stream_synchronize(void* stream);        /* Stream::waitForCompletion */
B200CV_API int b200cv_stream_wait_event(void* stream, void* event); /* Stream::waitEvent */
B200CV_API int b200cv_stream_add_callback(void* stream, void (*fn)(int status, void* user), void* user); /* enqueueHostCallback */
B200CV_API int b200cv_event_create(void** event);
B200CV_API int b200cv_event_destroy(void* event);
B200CV_API int b200cv_event_record(void* event, void* stream);
B200CV_API int b200cv_event_synchronize(void* event);
B200CV_API int b200cv_event_elapsed_ms(void* start, void* end, float* ms);

/* ---- host-side exact tables (pure host code; exported so callers/tests can inspect them) ----------------------- */
/* cv::getGaussianKernel (imgproc/src/smooth.dispatch.cpp:81-221): n taps as double, bit-exact softdouble arithmetic */
B200CV_API int b200cv_get_gaussian_kernel(int n, double sigma, double* out);
/* 8.8 fixed-point taps with error diffusion (smooth.dispatch.cpp:224-277) */
/* the same taps with 8 (8-bit images) or 16 (16-bit images) fractional bits: getGaussianKernelFixedPoint_ED, smooth.dispatch.cpp:224-258 */
B200CV_API int b200cv_get_gaussian_kernel_fixed(int ksize, double sigma, int bits, unsigned int* out);
B200CV_API int b200cv_get_gaussian_kernel_fixed8(int n, double sigma, uint16_t* out);

/* ---- device ops ------------------------------------------------------------------------------------------------
 * All take b200cvMat descriptors over DEVICE memory; small operands (taps, matrices) are HOST pointers, copied at
 * call time into kernel parameters.  dst must be pre-allocated with the right size/type (as the HAL guarantees). */

/* replaces cv::GaussianBlur (imgproc.hpp:1544; smooth.dispatch.cpp:609-826). u8: bit-exact 8.8 fixed point; f32: float. */
B200CV_API int b200cv_gaussian_blur(const b200cvMat* src, const b200cvMat* dst, int ksize_w, int ksize_h,
                                    double sigma_x, double sigma_y, int border, void* stream);
/* replaces cv::sepFilter2D (imgproc.hpp:1723; filter.dispatch.cpp:1555-1594). kx/ky: float taps on the host. */
B200CV_API int b200cv_sep_filter2d(const b200cvMat* src, const b200cvMat* dst, const float* kx, int kx_len,
                                   const float* ky, int ky_len, int anchor_x, int anchor_y, double delta,
                                   int border, void* stream);
/* replaces cv::filter2D (imgproc.hpp:1702; filter.dispatch.cpp:1521-1553). kernel: kh x kw float taps (correlation). */
B200CV_API int b200cv_filter2d(const b200cvMat* src, const b200cvMat* dst, const float* kernel, int kw, int kh,
                               int anchor_x, int anchor_y, double delta, int border, void* stream);
/* replaces cv::Sobel (imgproc.hpp:1862; deriv.cpp:414-465) for ksize 1/3/5/7 */
B200CV_API int b200cv_sobel(const b200cvMat* src, const b200cvMat* dst, int dx, int dy, int ksize, double scale,
                            double delta, int border, void* stream);
/* replaces cv::boxFilter / cv::blur (imgproc.hpp:1603, :1659; box_filter.dispatch.cpp:440-498).  dst depth picks ddepth:
 * 8U->8U, 8U->32F, 32F->32F; anchor (-1,-1) = centre; borders CONSTANT (zeros), REPLICATE, REFLECT, REFLECT_101; ksize <= 128x128. */
B200CV_API int b200cv_box_filter(const b200cvMat* src, const b200cvMat* dst, int ksize_w, int ksize_h, int anchor_x, int anchor_y,
                                 int normalize, int border, void* stream);
/* replaces cv::integral (imgproc.hpp; sumpixels.dispatch.cpp:415-451) for 8UC1 sources: sum is 32SC1 of (W+1) x (H+1); sqsum is NULL or
 * 64FC1 of the same size.  Tilted sums and other depth combinations: B200CV_NOT_IMPLEMENTED. */
B200CV_API int b200cv_integral(const b200cvMat* src, const b200cvMat* sum, const b200cvMat* sqsum, void* stream);
/* replaces cv::resize (imgproc.hpp:2422; resize.cpp:4201-4246).  Scale factors are dst/src sizes (fx=fy=0 form). */
B200CV_API int b200cv_resize(const b200cvMat* src, const b200cvMat* dst, int interpolation, void* stream);
/* cv::resize(src, dst, Size(), fx, fy) (imgproc.hpp:2422, resize.cpp:4214-4228): dst must be round(cols*fx) x round(rows*fy); the sampling
   scale is fx, fy themselves (not dst/src).  NEAREST / LINEAR / CUBIC; other modes return NOT_IMPLEMENTED when fx, fy differ from the size ratio. */
B200CV_API int b200cv_resize_scaled(const b200cvMat* src, const b200cvMat* dst, int interpolation, double fx, double fy, void* stream);
/* replaces cv::warpAffine (imgproc.hpp:2450; imgwarp.cpp:2788-2902). M: 2x3 doubles; inverted unless WARP_INVERSE_MAP. */
B200CV_API int b200cv_warp_affine(const b200cvMat* src, const b200cvMat* dst, const double* M, int flags,
                                  int border, const double* border_value, void* stream);
/* replaces cv::warpPerspective (imgproc.hpp:2482; imgwarp.cpp:3370-3466). M: 3x3 doubles. */
B200CV_API int b200cv_warp_perspective(const b200cvMat* src, const b200cvMat* dst, const double* M, int flags,
                                       int border, const double* border_value, void* stream);
/* replaces cv::remap (imgproc.hpp:2531; imgwarp.cpp:1762-1900, RemapInvoker :1096-1330) -- the caller of the
 * sampling code the warps already use.  dst has the size of the maps and the type of src.  Maps (one set for the whole batch):
 *   map1 CV_32FC1 + map2 CV_32FC1 (x and y planes), map1 CV_32FC2 (map2 NULL), or the fixed-point pair of cv::convertMaps
 *   map1 CV_16SC2 + map2 CV_16UC1 (map2 may be NULL for INTER_NEAREST).  WARP_RELATIVE_MAP is not implemented. */
B200CV_API int b200cv_remap(const b200cvMat* src, const b200cvMat* dst, const b200cvMat* map1, const b200cvMat* map2, int interpolation,
                            int border, const double* border_value, void* stream);
/* replace cv::pyrDown / cv::pyrUp (imgproc.hpp:3325, :3351; pyramids.cpp:1348-1400, :1459-1505) for the default destination sizes
 * ((W+1)/2 x (H+1)/2 and 2W x 2H), 8-bit and float, 1/3/4 channels */
B200CV_API int b200cv_pyr_down(const b200cvMat* src, const b200cvMat* dst, int border, void* stream);
B200CV_API int b200cv_pyr_up(const b200cvMat* src, const b200cvMat* dst, int border, void* stream);
/* replaces cv::cvtColor (imgproc.hpp:3736; color.cpp:192-400) for BGR/RGB(A) <-> GRAY / YUV / YCrCb / HSV(_FULL) / BGR(A), and for the
 * subsampled-YUV wire formats (codes 90-108, 111-112, 115-124, 127-134: NV12 / NV21 / YV12 / IYUV / UYVY / YUY2 / YVYU; color.cpp:323-380),
 * whose source and destination sizes differ: a 4:2:0 image of W x H pixels is one 8-bit plane of H*3/2 rows.
 * CV_16U and CV_32F images: the channel reorders (codes 0-5), BGR/RGB(A) <-> GRAY (6-11), BGR/RGB <-> XYZ (32-35), BGR/RGB <-> YCrCb / YUV (36-39, 82-85) and, float only, BGR/RGB <-> HSV (40-41, 54-55, 66-67, 70-71)
 * (color_rgb.simd.hpp:608-841, color_yuv.simd.hpp:134-396,616-1013, color_lab.cpp:172-700), bit-exact incl. float; other codes at those depths: NOT_IMPLEMENTED */
B200CV_API int b200cv_cvt_color(const b200cvMat* src, const b200cvMat* dst, int code, void* stream);
/* replaces cv::cvtColorTwoPlane (imgproc.hpp; color.cpp:171-185): NV12 / NV21 (codes 90-97) with the luma plane (8UC1, W x H) and the
 * interleaved chroma plane (8UC2, W/2 x H/2) in separate buffers with their own pitches, as hardware decoders hand them out */
B200CV_API int b200cv_cvt_color_two_plane(const b200cvMat* src_y, const b200cvMat* src_uv, const b200cvMat* dst, int code, void* stream);
/* replaces cv::matchTemplate (imgproc.hpp:3916; templmatch.cpp:1158-1194), 1-channel u8/f32, all six methods.
 * result: CV_32FC1 (W-w+1) x (H-h+1).  The CCORR numerator of u8 images runs on the tensor cores (wgmma). */
B200CV_API int b200cv_match_template(const b200cvMat* image, const b200cvMat* templ, const b200cvMat* result,
                                     int method, void* stream);
/* cv::matchTemplate with a mask (templmatch.cpp:762-905): mask = 8UC1 (non-zero = 1) or 32FC1 (weights) of the template's size, one channel */
B200CV_API int b200cv_match_template_masked(const b200cvMat* image, const b200cvMat* templ, const b200cvMat* mask, const b200cvMat* result, int method,
                                            void* stream);
/* replaces cv::cornerHarris / cv::cornerMinEigenVal (imgproc.hpp:1948,1921; corner.cpp:634-654,610-632) */
B200CV_API int b200cv_corner_harris(const b200cvMat* src, const b200cvMat* dst, int block_size, int ksize, double k,
                                    int border, void* stream);
B200CV_API int b200cv_corner_min_eigen_val(const b200cvMat* src, const b200cvMat* dst, int block_size, int ksize,
                                           int border, void* stream);
/* replaces cv::goodFeaturesToTrack (imgproc.hpp:2096; featureselect.cpp:382-548).  Synchronous (returns host data).
 * corners: host array of 2*max_out floats (x,y pairs) per frame, laid out frame after frame; counts[f] = corners found
 * in frame f (may exceed max_out; only the first max_out are stored). */
B200CV_API int b200cv_good_features_to_track(const b200cvMat* src, float* corners, float* quality, int max_out,
                                             int* counts, int max_corners, double quality_level, double min_distance,
                                             int block_size, int gradient_size, int use_harris, double k, void* stream);
/* SIFT Gaussian pyramid + DoG (features2d/src/sift.dispatch.cpp:176-310).
 * src: 8UC1 batch.  gauss / dog: device float buffers, per frame packed image after image, octave-major
 * (n_octaves*(n_layers+3) Gaussian images, n_octaves*(n_layers+2) DoG images); per-frame strides in floats.
 * Query sizes first with b200cv_sift_pyramid_layout. dog may be NULL (Gaussian only).
 * upscale: 0 = first octave at the image size; 1 = doubled with the precise up-scaling (SIFT::create(..., enable_precise_upscale = true):
 * warpAffine, sift.dispatch.cpp:196-202); 2 = doubled as SIFT::create's default does it (cv::resize INTER_LINEAR, :203-208). */
B200CV_API int b200cv_sift_pyramid_layout(int width, int height, int n_octave_layers, int upscale,
                                          int* n_octaves, size_t* gauss_elems, size_t* dog_elems, int* dims /*2*n_octaves or NULL*/);
/* the SIFT front end after the pyramid (cv::SIFT::detectAndCompute, sift.dispatch.cpp:501-580): scale-space extrema,
 * sub-pixel refinement, orientation assignment, duplicate removal, first-octave rescaling and, if descriptors != NULL, the 128-float
 * descriptors.  gauss / dog: DEVICE pointers to ONE frame's packed pyramids as b200cv_sift_pyramid writes them; dims: the per-octave (w, h)
 * table of b200cv_sift_pyramid_layout (host); keypoints: HOST, 6 floats each (x, y, size, angle, response, packed octave as int bits);
 * descriptors: HOST, 128 floats each; n_features > 0 keeps the strongest responses (KeyPointsFilter::retainBest, ties included); mask: NULL or a HOST 8-bit image
 * of the input frame's size, keypoints on zero bytes are dropped before the descriptors are computed (runByPixelsMask); at most
 * max_keypoints are written, *n_keypoints receives the number found.  Synchronises the stream. */
B200CV_API int b200cv_sift_detect_and_compute(const float* gauss, const float* dog, const int* dims, int n_octaves, int n_octave_layers,
                                              double contrast_threshold, double edge_threshold, double sigma, int first_octave, int n_features,
                                              const unsigned char* mask, size_t mask_step, int mask_width, int mask_height,
                                              int max_keypoints, float* keypoints, float* descriptors, int* n_keypoints, void* stream);
B200CV_API int b200cv_sift_pyramid(const b200cvMat* src, int n_octave_layers, double sigma, int upscale,
                                   float* gauss, size_t gauss_frame_elems, float* dog, size_t dog_frame_elems, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200CV_H */
