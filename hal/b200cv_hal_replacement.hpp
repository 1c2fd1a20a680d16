// b200cv_hal_replacement.hpp -- OpenCV imgproc HAL replacement header.
//
// Registered through OpenCV's own mechanism (CMakeLists.txt:927-1040, samples/hal/README.md):
//     cmake -DOpenCV_HAL_DIR=<repo>/hal  ...        (hal/b200cv_halConfig.cmake names this header + libb200cv.so)
// modules/imgproc/src/hal_replacement.hpp then includes it via custom_hal.hpp (:1339) and every `cv_hal_X` below stops being
// the NOT_IMPLEMENTED stub (`hal_ni_X`) and becomes the GPU path.  Semantics of the return value are the seam's
// (hal_replacement.hpp:1342-1357): 0 = done, 1 = not implemented -> OpenCV runs its own code, anything else -> cv::Error.
#ifndef B200CV_HAL_REPLACEMENT_HPP
#define B200CV_HAL_REPLACEMENT_HPP
#include "b200cv_hal.h"

#undef cv_hal_gaussianBlur
#define cv_hal_gaussianBlur b200cv_hal_gaussianBlur
#undef cv_hal_gaussianBlurBinomial
#define cv_hal_gaussianBlurBinomial b200cv_hal_gaussianBlurBinomial
#undef cv_hal_sepFilterInit
#define cv_hal_sepFilterInit(ctx, ...) b200cv_hal_sepFilterInit((struct b200cvFilterCtx**)(ctx), __VA_ARGS__)
#undef cv_hal_sepFilter
#define cv_hal_sepFilter(ctx, ...) b200cv_hal_sepFilter((struct b200cvFilterCtx*)(ctx), __VA_ARGS__)
#undef cv_hal_sepFilterFree
#define cv_hal_sepFilterFree(ctx) b200cv_hal_sepFilterFree((struct b200cvFilterCtx*)(ctx))
#undef cv_hal_filterInit
#define cv_hal_filterInit(ctx, ...) b200cv_hal_filterInit((struct b200cvFilterCtx**)(ctx), __VA_ARGS__)
#undef cv_hal_filter
#define cv_hal_filter(ctx, ...) b200cv_hal_filter((struct b200cvFilterCtx*)(ctx), __VA_ARGS__)
#undef cv_hal_filterFree
#define cv_hal_filterFree(ctx) b200cv_hal_filterFree((struct b200cvFilterCtx*)(ctx))
#undef cv_hal_sobel
#define cv_hal_sobel b200cv_hal_sobel
#undef cv_hal_resize
#define cv_hal_resize b200cv_hal_resize
#undef cv_hal_warpAffine
#define cv_hal_warpAffine b200cv_hal_warpAffine
#undef cv_hal_warpPerspective
#define cv_hal_warpPerspective b200cv_hal_warpPerspective
#undef cv_hal_remap32f
#define cv_hal_remap32f b200cv_hal_remap32f
#undef cv_hal_pyrdown
#define cv_hal_pyrdown b200cv_hal_pyrdown
#undef cv_hal_scharr
#define cv_hal_scharr b200cv_hal_scharr
#undef cv_hal_cvtTwoPlaneYUVtoBGR
#define cv_hal_cvtTwoPlaneYUVtoBGR b200cv_hal_cvtTwoPlaneYUVtoBGR
#undef cv_hal_cvtThreePlaneYUVtoBGR
#define cv_hal_cvtThreePlaneYUVtoBGR b200cv_hal_cvtThreePlaneYUVtoBGR
#undef cv_hal_cvtBGRtoThreePlaneYUV
#define cv_hal_cvtBGRtoThreePlaneYUV b200cv_hal_cvtBGRtoThreePlaneYUV
#undef cv_hal_cvtOnePlaneYUVtoBGR
#define cv_hal_cvtOnePlaneYUVtoBGR b200cv_hal_cvtOnePlaneYUVtoBGR
#undef cv_hal_cvtOnePlaneBGRtoYUV
#define cv_hal_cvtOnePlaneBGRtoYUV b200cv_hal_cvtOnePlaneBGRtoYUV
#undef cv_hal_integral
#define cv_hal_integral b200cv_hal_integral
#undef cv_hal_cvtBGRtoXYZ
#define cv_hal_cvtBGRtoXYZ b200cv_hal_cvtBGRtoXYZ
#undef cv_hal_cvtXYZtoBGR
#define cv_hal_cvtXYZtoBGR b200cv_hal_cvtXYZtoBGR
#undef cv_hal_cvtBGRtoLab
#define cv_hal_cvtBGRtoLab b200cv_hal_cvtBGRtoLab
#undef cv_hal_cvtLabtoBGR
#define cv_hal_cvtLabtoBGR b200cv_hal_cvtLabtoBGR
#undef cv_hal_boxFilter
#define cv_hal_boxFilter b200cv_hal_boxFilter
#undef cv_hal_cvtBGRtoBGR
#define cv_hal_cvtBGRtoBGR b200cv_hal_cvtBGRtoBGR
#undef cv_hal_cvtBGRtoGray
#define cv_hal_cvtBGRtoGray b200cv_hal_cvtBGRtoGray
#undef cv_hal_cvtGraytoBGR
#define cv_hal_cvtGraytoBGR b200cv_hal_cvtGraytoBGR
#undef cv_hal_cvtBGRtoYUV
#define cv_hal_cvtBGRtoYUV b200cv_hal_cvtBGRtoYUV
#undef cv_hal_cvtYUVtoBGR
#define cv_hal_cvtYUVtoBGR b200cv_hal_cvtYUVtoBGR
#undef cv_hal_cvtBGRtoHSV
#define cv_hal_cvtBGRtoHSV b200cv_hal_cvtBGRtoHSV
#undef cv_hal_cvtHSVtoBGR
#define cv_hal_cvtHSVtoBGR b200cv_hal_cvtHSVtoBGR
#endif
