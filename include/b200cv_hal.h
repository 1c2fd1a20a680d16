/*
 * b200cv_hal.h -- HOST-pointer entry points of the hot path.
 *
 * (1) b200cv_hal_*  : exactly the argument lists of the reference's imgproc HAL seam
 *     (modules/imgproc/src/hal_replacement.hpp; each prototype cites the hal_ni_* it replaces), so a stock OpenCV
 *     rebuilt with `-DOpenCV_HAL_DIR=<this repo>/hal` routes its host cv::Mat calls here:
 *         #undef  cv_hal_resize
 *         #define cv_hal_resize b200cv_hal_resize          (see INTEGRATION.md and hal/b200cv_hal_replacement.hpp)
 *     Calls are synchronous (result in dst on return), thread-safe (per-thread stream + staging buffers), return
 *     CV_HAL_ERROR_OK (0) / CV_HAL_ERROR_NOT_IMPLEMENTED (1: OpenCV silently uses its own code) / other = error
 *     (hal_replacement.hpp:1342-1357).  Inside: H2D copy, the same sm_90a kernels as the device API, D2H copy.
 *
 * (2) b200cv_host_* : the device API of b200cv.h over HOST b200cvMat descriptors (data = host pointer, ideally
 *     page-locked: b200cv_host_alloc), for BATCHES of frames: frames are cut into chunks that flow through a
 *     3-stream upload -> kernel -> download pipeline so PCIe transfers in both directions overlap the kernels.
 *     This is the end-to-end path bench.py times as `e2e`.
 */
#ifndef B200CV_HAL_H
#define B200CV_HAL_H
#include "b200cv.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef unsigned char b200cv_uchar;
struct b200cvFilterCtx;   /* stands in for cvhalFilter2D (opaque context), hal_replacement.hpp:90 */

/* hal_ni_gaussianBlur, hal_replacement.hpp:1146 */
B200CV_API int b200cv_hal_gaussianBlur(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                       int depth, int cn, size_t margin_left, size_t margin_top, size_t margin_right, size_t margin_bottom,
                                       size_t ksize_width, size_t ksize_height, double sigmaX, double sigmaY, int border_type);
/* hal_ni_gaussianBlurBinomial, hal_replacement.hpp:1169 */
B200CV_API int b200cv_hal_gaussianBlurBinomial(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width,
                                               int height, int depth, int cn, size_t margin_left, size_t margin_top, size_t margin_right,
                                               size_t margin_bottom, size_t ksize, int border_type);
/* hal_ni_sepFilterInit / sepFilter / sepFilterFree, hal_replacement.hpp:155,171,177 */
B200CV_API int b200cv_hal_sepFilterInit(struct b200cvFilterCtx** context, int src_type, int dst_type, int kernel_type, b200cv_uchar* kernelx_data,
                                        int kernelx_length, b200cv_uchar* kernely_data, int kernely_length, int anchor_x, int anchor_y,
                                        double delta, int borderType);
B200CV_API int b200cv_hal_sepFilter(struct b200cvFilterCtx* context, b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step,
                                    int width, int height, int full_width, int full_height, int offset_x, int offset_y);
B200CV_API int b200cv_hal_sepFilterFree(struct b200cvFilterCtx* context);
/* hal_ni_filterInit / filter / filterFree, hal_replacement.hpp:109,125,131 */
B200CV_API int b200cv_hal_filterInit(struct b200cvFilterCtx** context, b200cv_uchar* kernel_data, size_t kernel_step, int kernel_type, int kernel_width,
                                     int kernel_height, int max_width, int max_height, int src_type, int dst_type, int borderType, double delta,
                                     int anchor_x, int anchor_y, bool allowSubmatrix, bool allowInplace);
B200CV_API int b200cv_hal_filter(struct b200cvFilterCtx* context, b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step,
                                 int width, int height, int full_width, int full_height, int offset_x, int offset_y);
B200CV_API int b200cv_hal_filterFree(struct b200cvFilterCtx* context);
/* hal_ni_sobel, hal_replacement.hpp:1197 */
B200CV_API int b200cv_hal_sobel(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                int src_depth, int dst_depth, int cn, int margin_left, int margin_top, int margin_right, int margin_bottom,
                                int dx, int dy, int ksize, double scale, double delta, int border_type);
/* hal_ni_scharr, hal_replacement.hpp:1224 */
B200CV_API int b200cv_hal_scharr(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                 int src_depth, int dst_depth, int cn, int margin_left, int margin_top, int margin_right, int margin_bottom,
                                 int dx, int dy, double scale, double delta, int border_type);
/* hal_ni_boxFilter, hal_replacement.hpp:1105 (cv::boxFilter / cv::blur, box_filter.dispatch.cpp:474) */
B200CV_API int b200cv_hal_boxFilter(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                    int src_depth, int dst_depth, int cn, int margin_left, int margin_top, int margin_right, int margin_bottom,
                                    size_t ksize_width, size_t ksize_height, int anchor_x, int anchor_y, bool normalize, int border_type);
/* hal_ni_integral, hal_replacement.hpp:977 (cv::integral, sumpixels.dispatch.cpp:375): 8UC1 -> 32S sum (+ 64F sqsum); no tilted sums */
B200CV_API int b200cv_hal_integral(int depth, int sdepth, int sqdepth, const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* sum_data, size_t sum_step,
                                   b200cv_uchar* sqsum_data, size_t sqsum_step, b200cv_uchar* tilted_data, size_t tilted_step, int width, int height, int cn);
/* hal_ni_resize, hal_replacement.hpp:257 */
B200CV_API int b200cv_hal_resize(int src_type, const b200cv_uchar* src_data, size_t src_step, int src_width, int src_height, b200cv_uchar* dst_data,
                                 size_t dst_step, int dst_width, int dst_height, double inv_scale_x, double inv_scale_y, int interpolation);
/* hal_ni_warpAffine :275 / hal_ni_warpPerspective :316 -- M is already the inverse (dst -> src) map */
B200CV_API int b200cv_hal_warpAffine(int src_type, const b200cv_uchar* src_data, size_t src_step, int src_width, int src_height, b200cv_uchar* dst_data,
                                     size_t dst_step, int dst_width, int dst_height, const double M[6], int interpolation, int borderType,
                                     const double borderValue[4]);
B200CV_API int b200cv_hal_warpPerspective(int src_type, const b200cv_uchar* src_data, size_t src_step, int src_width, int src_height,
                                          b200cv_uchar* dst_data, size_t dst_step, int dst_width, int dst_height, const double M[9],
                                          int interpolation, int borderType, const double borderValue[4]);
/* hal_ni_remap32f, hal_replacement.hpp:371 (called from cv::remap for CV_32FC1 map pairs, imgwarp.cpp:1818-1822) */
B200CV_API int b200cv_hal_remap32f(int src_type, const b200cv_uchar* src_data, size_t src_step, int src_width, int src_height, b200cv_uchar* dst_data,
                                   size_t dst_step, int dst_width, int dst_height, float* mapx, size_t mapx_step, float* mapy, size_t mapy_step,
                                   int interpolation, int border_type, const double border_value[4]);
/* hal_ni_pyrdown, hal_replacement.hpp:1244 (cv::pyrDown on a whole Mat, pyramids.cpp:1377) */
B200CV_API int b200cv_hal_pyrdown(const b200cv_uchar* src_data, size_t src_step, int src_width, int src_height, b200cv_uchar* dst_data, size_t dst_step,
                                  int dst_width, int dst_height, int depth, int cn, int border_type);
/* colour: hal_ni_cvtBGRtoBGR :395, cvtBGRtoGray :442, cvtGraytoBGR :456, cvtBGRtoYUV :500, cvtYUVtoBGR :533, cvtBGRtoHSV :596, cvtHSVtoBGR :613.
 * depth: CV_8U for all; CV_16U and CV_32F for BGRtoBGR / BGRtoGray / GraytoBGR / BGRtoYUV / YUVtoBGR / XYZ; CV_32F for HSV (HLS: not implemented) */
B200CV_API int b200cv_hal_cvtBGRtoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int scn, int dcn, bool swapBlue);
B200CV_API int b200cv_hal_cvtBGRtoGray(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                       int depth, int scn, bool swapBlue);
B200CV_API int b200cv_hal_cvtGraytoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                       int depth, int dcn);
B200CV_API int b200cv_hal_cvtBGRtoYUV(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int scn, bool swapBlue, bool isCbCr);
B200CV_API int b200cv_hal_cvtYUVtoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int dcn, bool swapBlue, bool isCbCr);
B200CV_API int b200cv_hal_cvtBGRtoHSV(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int scn, bool swapBlue, bool isFullRange, bool isHSV);
B200CV_API int b200cv_hal_cvtHSVtoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int dcn, bool swapBlue, bool isFullRange, bool isHSV);
/* hal_ni_cvtBGRtoXYZ / hal_ni_cvtXYZtoBGR (hal_replacement.hpp:564, :579): 8-bit, 16-bit, float */
B200CV_API int b200cv_hal_cvtBGRtoXYZ(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int scn, bool swapBlue);
B200CV_API int b200cv_hal_cvtXYZtoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int dcn, bool swapBlue);
/* hal_ni_cvtBGRtoLab / hal_ni_cvtLabtoBGR (hal_replacement.hpp:630, :647): 8-bit Lab only (isLab; Luv and float data are declined) */
B200CV_API int b200cv_hal_cvtBGRtoLab(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int scn, bool swapBlue, bool isLab, bool srgb);
B200CV_API int b200cv_hal_cvtLabtoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                      int depth, int dcn, bool swapBlue, bool isLab, bool srgb);
/* subsampled YUV wire formats: hal_ni_cvtTwoPlaneYUVtoBGR :664 (NV12 uIdx 0 / NV21 uIdx 1, one buffer), cvtThreePlaneYUVtoBGR :763
 * (IYUV uIdx 0 / YV12 uIdx 1), cvtBGRtoThreePlaneYUV :797 (IYUV uIdx 1 / YV12 uIdx 2: color.hpp:162-176), cvtOnePlaneYUVtoBGR :833
 * (YUY2 uIdx 0 ycn 0, YVYU uIdx 1 ycn 0, UYVY uIdx 0 ycn 1) */
B200CV_API int b200cv_hal_cvtTwoPlaneYUVtoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int dst_width, int dst_height,
                                              int dcn, bool swapBlue, int uIdx);
B200CV_API int b200cv_hal_cvtThreePlaneYUVtoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int dst_width, int dst_height,
                                                int dcn, bool swapBlue, int uIdx);
B200CV_API int b200cv_hal_cvtBGRtoThreePlaneYUV(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                                int scn, bool swapBlue, int uIdx);
B200CV_API int b200cv_hal_cvtOnePlaneBGRtoYUV(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                              int scn, bool swapBlue, int uIdx, int ycn);      /* hal_ni_cvtOnePlaneBGRtoYUV :866 */
B200CV_API int b200cv_hal_cvtOnePlaneYUVtoBGR(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                              int dcn, bool swapBlue, int uIdx, int ycn);

/* hal_ni_canny, hal_replacement.hpp:1291 (cv::Canny, canny.cpp:864): 8-bit, 1-4 channels.  The thresholds arrive already divided by 16
 * for aperture 7 and swapped (canny.cpp:848-856 runs before the call) and are used as given; ksize 3 / 5 / 7 or -1 (Scharr) */
B200CV_API int b200cv_hal_canny(const b200cv_uchar* src_data, size_t src_step, b200cv_uchar* dst_data, size_t dst_step, int width, int height,
                                int cn, double lowThreshold, double highThreshold, int ksize, bool L2gradient);

/* ---- batched host API (what cv::-signature wrappers over cv::Mat call; pipelined over 3 streams) ----------------------- */
B200CV_API int b200cv_host_gaussian_blur(const b200cvMat* src, const b200cvMat* dst, int ksize_w, int ksize_h, double sigma_x, double sigma_y, int border);
B200CV_API int b200cv_host_sep_filter2d(const b200cvMat* src, const b200cvMat* dst, const float* kx, int kx_len, const float* ky, int ky_len,
                                        int anchor_x, int anchor_y, double delta, int border);
B200CV_API int b200cv_host_filter2d(const b200cvMat* src, const b200cvMat* dst, const float* kernel, int kw, int kh, int anchor_x, int anchor_y,
                                    double delta, int border);
B200CV_API int b200cv_host_sobel(const b200cvMat* src, const b200cvMat* dst, int dx, int dy, int ksize, double scale, double delta, int border);
B200CV_API int b200cv_host_laplacian(const b200cvMat* src, const b200cvMat* dst, int ksize, double scale, double delta, int border);
/* cv::erode / cv::dilate / cv::morphologyEx over host frames; arguments as b200cv_morphology takes them.  No cv_hal_morph hook is
 * registered (see INTEGRATION.md), so there is no hal_ni_* counterpart. */
B200CV_API int b200cv_host_morphology(const b200cvMat* src, const b200cvMat* dst, int op, const unsigned char* kernel_data, size_t kernel_step,
                                      int kw, int kh, int anchor_x, int anchor_y, int iterations, int border, const double border_value[4]);
B200CV_API int b200cv_host_box_filter(const b200cvMat* src, const b200cvMat* dst, int ksize_w, int ksize_h, int anchor_x, int anchor_y, int normalize, int border);
B200CV_API int b200cv_host_integral(const b200cvMat* src, const b200cvMat* sum, const b200cvMat* sqsum);
B200CV_API int b200cv_host_resize(const b200cvMat* src, const b200cvMat* dst, int interpolation);
B200CV_API int b200cv_host_resize_scaled(const b200cvMat* src, const b200cvMat* dst, int interpolation, double fx, double fy);
B200CV_API int b200cv_host_warp_affine(const b200cvMat* src, const b200cvMat* dst, const double* M, int flags, int border, const double* border_value);
B200CV_API int b200cv_host_warp_perspective(const b200cvMat* src, const b200cvMat* dst, const double* M, int flags, int border, const double* border_value);
B200CV_API int b200cv_host_pyr_down(const b200cvMat* src, const b200cvMat* dst, int border);
B200CV_API int b200cv_host_pyr_up(const b200cvMat* src, const b200cvMat* dst, int border);
/* maps are host arrays too (one set for the whole batch); they are uploaded once per call */
B200CV_API int b200cv_host_remap(const b200cvMat* src, const b200cvMat* dst, const b200cvMat* map1, const b200cvMat* map2, int interpolation, int border,
                                 const double* border_value);
B200CV_API int b200cv_host_cvt_color(const b200cvMat* src, const b200cvMat* dst, int code);
B200CV_API int b200cv_host_match_template(const b200cvMat* image, const b200cvMat* templ, const b200cvMat* result, int method);
B200CV_API int b200cv_host_corner_harris(const b200cvMat* src, const b200cvMat* dst, int block_size, int ksize, double k, int border);
B200CV_API int b200cv_host_corner_min_eigen_val(const b200cvMat* src, const b200cvMat* dst, int block_size, int ksize, int border);
/* cv::Canny over host frames; thresholds and aperture as b200cv_canny takes them */
B200CV_API int b200cv_host_canny(const b200cvMat* src, const b200cvMat* dst, double threshold1, double threshold2, int aperture_size, int l2gradient);
/* cv::distanceTransform over host frames; arguments as b200cv_distance_transform takes them (the type of dst selects the 8-bit L1 call).
 * The reference has no HAL hook for it, so there is no hal_ni_* counterpart. */
B200CV_API int b200cv_host_distance_transform(const b200cvMat* src, const b200cvMat* dst, int distance_type, int mask_size);

#ifdef __cplusplus
}
#endif
#endif
