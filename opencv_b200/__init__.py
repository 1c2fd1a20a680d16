"""opencv_b200 -- Python face of the H100-native dense-imgproc hot path (libb200cv.so, sm_90a).

The functions mirror the cv2 / cv:: names and argument meaning of the reference
(modules/imgproc/include/opencv2/imgproc.hpp) for the calls on the hot path:

    GaussianBlur, sepFilter2D, filter2D, Sobel, Laplacian, erode, dilate, morphologyEx, resize, warpAffine, warpPerspective, cvtColor,
    matchTemplate, cornerHarris, cornerMinEigenVal, goodFeaturesToTrack, Canny, distanceTransform, sift_pyramid

Inputs are torch CUDA tensors laid out like a cv::Mat -- (H, W) or (H, W, C), or a batch
(N, H, W[, C]) of independent frames -- and go to the device C ABI (include/b200cv.h) without a
copy; numpy arrays go through the synchronous host C ABI (include/b200cv_hal.h), which uploads,
runs the same kernels and downloads.  There is NO CPU fallback: if the CUDA library is missing or
no H100 is visible every call raises.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "lib", "libb200cv.so")
_lib = None

# ---- OpenCV-compatible constants -------------------------------------------------------------------------------
CV_8U, CV_16S, CV_32F = 0, 3, 5
BORDER_CONSTANT, BORDER_REPLICATE, BORDER_REFLECT, BORDER_WRAP, BORDER_REFLECT_101 = 0, 1, 2, 3, 4
BORDER_DEFAULT = BORDER_REFLECT_101
BORDER_REFLECT101 = BORDER_REFLECT_101
BORDER_TRANSPARENT, BORDER_ISOLATED = 5, 16
INTER_NEAREST, INTER_LINEAR, INTER_CUBIC, INTER_AREA = 0, 1, 2, 3
INTER_LANCZOS4, INTER_LINEAR_EXACT, INTER_NEAREST_EXACT = 4, 5, 6
WARP_INVERSE_MAP = 16
TM_SQDIFF, TM_SQDIFF_NORMED, TM_CCORR, TM_CCORR_NORMED, TM_CCOEFF, TM_CCOEFF_NORMED = range(6)
# cv::DistanceTypes and cv::DistanceTransformMasks
DIST_USER, DIST_L1, DIST_L2, DIST_C, DIST_L12, DIST_FAIR, DIST_WELSCH, DIST_HUBER = -1, 1, 2, 3, 4, 5, 6, 7
DIST_MASK_3, DIST_MASK_5, DIST_MASK_PRECISE = 3, 5, 0
# cv::MorphTypes and cv::MorphShapes
MORPH_ERODE, MORPH_DILATE, MORPH_OPEN, MORPH_CLOSE, MORPH_GRADIENT, MORPH_TOPHAT, MORPH_BLACKHAT, MORPH_HITMISS = range(8)
MORPH_RECT, MORPH_CROSS, MORPH_ELLIPSE = 0, 1, 2
COLOR_BGR2BGRA, COLOR_BGRA2BGR, COLOR_BGR2RGBA, COLOR_RGBA2BGR, COLOR_BGR2RGB, COLOR_BGRA2RGBA = range(6)
COLOR_RGB2BGRA, COLOR_BGRA2RGB, COLOR_RGB2BGR, COLOR_RGBA2BGRA = COLOR_BGR2RGBA, COLOR_RGBA2BGR, COLOR_BGR2RGB, COLOR_BGRA2RGBA
COLOR_BGR2GRAY, COLOR_RGB2GRAY, COLOR_GRAY2BGR, COLOR_GRAY2BGRA, COLOR_BGRA2GRAY, COLOR_RGBA2GRAY = 6, 7, 8, 9, 10, 11
COLOR_GRAY2RGB, COLOR_GRAY2RGBA = COLOR_GRAY2BGR, COLOR_GRAY2BGRA
COLOR_BGR2YCrCb, COLOR_RGB2YCrCb, COLOR_YCrCb2BGR, COLOR_YCrCb2RGB = 36, 37, 38, 39
COLOR_BGR2HSV, COLOR_RGB2HSV, COLOR_HSV2BGR, COLOR_HSV2RGB = 40, 41, 54, 55
COLOR_BGR2XYZ, COLOR_RGB2XYZ, COLOR_XYZ2BGR, COLOR_XYZ2RGB = 32, 33, 34, 35
COLOR_BGR2Lab, COLOR_RGB2Lab, COLOR_Lab2BGR, COLOR_Lab2RGB = 44, 45, 56, 57
COLOR_LBGR2Lab, COLOR_LRGB2Lab, COLOR_Lab2LBGR, COLOR_Lab2LRGB = 74, 75, 78, 79
COLOR_BGR2HSV_FULL, COLOR_RGB2HSV_FULL, COLOR_HSV2BGR_FULL, COLOR_HSV2RGB_FULL = 66, 67, 70, 71
COLOR_BGR2YUV, COLOR_RGB2YUV, COLOR_YUV2BGR, COLOR_YUV2RGB = 82, 83, 84, 85
# Bayer mosaics, bilinear demosaicing (imgproc.hpp: 46-49, 139-142; the 2RGB names are the 2BGR numbers of the mirrored pattern)
COLOR_BayerBG2BGR, COLOR_BayerGB2BGR, COLOR_BayerRG2BGR, COLOR_BayerGR2BGR = 46, 47, 48, 49
COLOR_BayerBG2RGB, COLOR_BayerGB2RGB, COLOR_BayerRG2RGB, COLOR_BayerGR2RGB = 48, 49, 46, 47
COLOR_BayerBG2BGRA, COLOR_BayerGB2BGRA, COLOR_BayerRG2BGRA, COLOR_BayerGR2BGRA = 139, 140, 141, 142
COLOR_BayerBG2RGBA, COLOR_BayerGB2RGBA, COLOR_BayerRG2RGBA, COLOR_BayerGR2RGBA = 141, 142, 139, 140
# edge-aware demosaicing (demosaicing.cpp:1592-1737), 3-channel destinations
COLOR_BayerBG2BGR_EA, COLOR_BayerGB2BGR_EA, COLOR_BayerRG2BGR_EA, COLOR_BayerGR2BGR_EA = 135, 136, 137, 138
COLOR_BayerBG2RGB_EA, COLOR_BayerGB2RGB_EA, COLOR_BayerRG2RGB_EA, COLOR_BayerGR2RGB_EA = 137, 138, 135, 136
# Variable Number of Gradients (demosaicing.cpp:1059-1587), 8-bit mosaics, 3-channel destinations
COLOR_BayerBG2BGR_VNG, COLOR_BayerGB2BGR_VNG, COLOR_BayerRG2BGR_VNG, COLOR_BayerGR2BGR_VNG = 62, 63, 64, 65
COLOR_BayerBG2RGB_VNG, COLOR_BayerGB2RGB_VNG, COLOR_BayerRG2RGB_VNG, COLOR_BayerGR2RGB_VNG = 64, 65, 62, 63
# Bayer mosaic to luma (demosaicing.cpp:652-792), 8- and 16-bit
COLOR_BayerBG2GRAY, COLOR_BayerGB2GRAY, COLOR_BayerRG2GRAY, COLOR_BayerGR2GRAY = 86, 87, 88, 89
# subsampled-YUV wire formats (imgproc.hpp: ColorConversionCodes 90-134)
COLOR_YUV2RGB_NV12, COLOR_YUV2BGR_NV12, COLOR_YUV2RGB_NV21, COLOR_YUV2BGR_NV21 = 90, 91, 92, 93
COLOR_YUV2RGBA_NV12, COLOR_YUV2BGRA_NV12, COLOR_YUV2RGBA_NV21, COLOR_YUV2BGRA_NV21 = 94, 95, 96, 97
COLOR_YUV2RGB_YV12, COLOR_YUV2BGR_YV12, COLOR_YUV2RGB_IYUV, COLOR_YUV2BGR_IYUV = 98, 99, 100, 101
COLOR_YUV2RGBA_YV12, COLOR_YUV2BGRA_YV12, COLOR_YUV2RGBA_IYUV, COLOR_YUV2BGRA_IYUV = 102, 103, 104, 105
COLOR_YUV2RGB_I420, COLOR_YUV2BGR_I420, COLOR_YUV2RGBA_I420, COLOR_YUV2BGRA_I420 = 100, 101, 104, 105
COLOR_YUV2GRAY_420 = COLOR_YUV2GRAY_NV12 = COLOR_YUV2GRAY_NV21 = COLOR_YUV2GRAY_I420 = COLOR_YUV2GRAY_YV12 = 106
COLOR_YUV2RGB_UYVY, COLOR_YUV2BGR_UYVY, COLOR_YUV2RGBA_UYVY, COLOR_YUV2BGRA_UYVY = 107, 108, 111, 112
COLOR_YUV2RGB_YUY2, COLOR_YUV2BGR_YUY2, COLOR_YUV2RGB_YVYU, COLOR_YUV2BGR_YVYU = 115, 116, 117, 118
COLOR_YUV2RGBA_YUY2, COLOR_YUV2BGRA_YUY2, COLOR_YUV2RGBA_YVYU, COLOR_YUV2BGRA_YVYU = 119, 120, 121, 122
COLOR_YUV2GRAY_UYVY, COLOR_YUV2GRAY_YUY2 = 123, 124
COLOR_RGB2YUV_I420, COLOR_BGR2YUV_I420, COLOR_RGBA2YUV_I420, COLOR_BGRA2YUV_I420 = 127, 128, 129, 130
COLOR_RGB2YUV_IYUV, COLOR_BGR2YUV_IYUV, COLOR_RGBA2YUV_IYUV, COLOR_BGRA2YUV_IYUV = 127, 128, 129, 130
COLOR_RGB2YUV_YV12, COLOR_BGR2YUV_YV12, COLOR_RGBA2YUV_YV12, COLOR_BGRA2YUV_YV12 = 131, 132, 133, 134
COLOR_RGB2YUV_UYVY, COLOR_BGR2YUV_UYVY, COLOR_RGBA2YUV_UYVY, COLOR_BGRA2YUV_UYVY = 143, 144, 145, 146
COLOR_RGB2YUV_YUY2, COLOR_BGR2YUV_YUY2, COLOR_RGB2YUV_YVYU, COLOR_BGR2YUV_YVYU = 147, 148, 149, 150
COLOR_RGBA2YUV_YUY2, COLOR_BGRA2YUV_YUY2, COLOR_RGBA2YUV_YVYU, COLOR_BGRA2YUV_YVYU = 151, 152, 153, 154

OK, NOT_IMPLEMENTED = 0, 1


class B200cvError(RuntimeError):
    pass


class NotImplementedOnDevice(B200cvError):
    """The C ABI returned CV_HAL_ERROR_NOT_IMPLEMENTED (unsupported type/border/size combination)."""


class Mat(ctypes.Structure):
    """struct b200cvMat (include/b200cv.h)"""
    _fields_ = [("data", ctypes.c_void_p), ("step", ctypes.c_size_t), ("cols", ctypes.c_int), ("rows", ctypes.c_int),
                ("type", ctypes.c_int), ("frames", ctypes.c_int), ("frame_step", ctypes.c_size_t)]


def lib_path():
    return _LIB_PATH


def lib():
    """Load libb200cv.so (built in-tree by `python -m opencv_b200.build`); fail loudly if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise B200cvError("libb200cv.so not built (%s): run `python -m opencv_b200.build`; "
                              "there is no CPU fallback for this path" % _LIB_PATH)
        L = ctypes.CDLL(_LIB_PATH)
        L.b200cv_last_error.restype = ctypes.c_char_p
        L.b200cv_version.restype = ctypes.c_char_p
        L.b200cv_launch_count.restype = ctypes.c_ulonglong
        _lib = L
    return _lib


def _check(rc, what):
    if rc == OK:
        return
    if rc == NOT_IMPLEMENTED:
        raise NotImplementedOnDevice("%s: combination not implemented on the device path" % what)
    raise B200cvError("%s failed (%d): %s" % (what, rc, lib().b200cv_last_error().decode()))


def init(device=0):
    _check(lib().b200cv_init(int(device)), "b200cv_init")


def launch_count():
    return int(lib().b200cv_launch_count())


CV_32S, CV_64F = 4, 6
_DEPTH_OF = {"torch.uint8": CV_8U, "torch.uint16": 2, "uint16": 2, "torch.int16": CV_16S, "torch.float32": CV_32F, "torch.int32": CV_32S, "torch.float64": CV_64F,
             "uint8": CV_8U, "int16": CV_16S, "float32": CV_32F, "int32": CV_32S, "float64": CV_64F}
_ESZ = {CV_8U: 1, 2: 2, CV_16S: 2, CV_32F: 4, CV_32S: 4, CV_64F: 8}


def make_type(depth, cn):
    return (depth & 7) + ((cn - 1) << 3)


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _stream_ptr(stream):
    if stream is None:
        import torch
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if hasattr(stream, "cuda_stream"):
        return ctypes.c_void_p(stream.cuda_stream)
    return ctypes.c_void_p(int(stream))


def describe(t):
    """b200cvMat over a torch CUDA tensor laid out like a cv::Mat / GpuMat:
    (H,W) single channel, (H,W,C) interleaved channels, or (N,H,W,C) a batch of N independent frames.
    Rows may be padded (stride(-3) >= W*C); pixels and channels must be dense."""
    assert _is_torch(t) and t.is_cuda, "device API needs a torch CUDA tensor"
    depth = _DEPTH_OF[str(t.dtype)]
    esz = _ESZ[depth]
    nd = t.dim()
    if nd == 2:
        n, h, w, c = 1, t.shape[0], t.shape[1], 1
        fs, rs = 0, t.stride(0)
        assert t.stride(1) == 1 or w == 1
    elif nd == 3:
        n, (h, w, c) = 1, t.shape
        fs, rs = 0, t.stride(0)
        assert (t.stride(2) == 1 or c == 1) and (t.stride(1) == c or w == 1)
    elif nd == 4:
        n, h, w, c = t.shape
        fs, rs = t.stride(0), t.stride(1)
        assert (t.stride(3) == 1 or c == 1) and (t.stride(2) == c or w == 1)
    else:
        raise ValueError("unsupported tensor rank %d" % nd)
    return Mat(t.data_ptr(), rs * esz, w, h, make_type(depth, c), n, fs * esz)


def _cn(m):
    return ((m.type >> 3) & 511) + 1


def _new(src, dtype=None, channels=None, size=None):
    """output tensor for `src`: same rank convention, optionally other dtype / channel count / (w, h)"""
    import torch
    m = describe(src)
    c = _cn(m) if channels is None else channels
    w, h = (m.cols, m.rows) if size is None else size
    if src.dim() == 4:
        shape = [max(m.frames, 1), h, w, c]
    elif c == 1:
        shape = [h, w]
    else:
        shape = [h, w, c]
    return torch.empty(shape, dtype=dtype or src.dtype, device=src.device)


def _pair(src, dst):
    return describe(src), describe(dst)


# ---- ops -----------------------------------------------------------------------------------------------------------
def GaussianBlur(src, ksize, sigmaX, sigmaY=0, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::GaussianBlur (imgproc.hpp:1544)"""
    if not _is_torch(src):
        from . import hal
        return hal.GaussianBlur(src, ksize, sigmaX, sigmaY, borderType)
    dst = dst if dst is not None else _new(src)
    ms, md = _pair(src, dst)
    _check(lib().b200cv_gaussian_blur(ctypes.byref(ms), ctypes.byref(md), int(ksize[0]), int(ksize[1]),
                                      ctypes.c_double(sigmaX), ctypes.c_double(sigmaY), int(borderType), _stream_ptr(stream)),
           "GaussianBlur")
    return dst


def _f32(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(-1))
    return a, a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _f64(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1))
    return a, a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _ddepth_dtype(src, ddepth):
    import torch
    if ddepth is None or ddepth < 0:
        return src.dtype
    return {CV_8U: torch.uint8, CV_16S: torch.int16, CV_32F: torch.float32}[ddepth]


def sepFilter2D(src, ddepth, kernelX, kernelY, anchor=(-1, -1), delta=0.0, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::sepFilter2D (imgproc.hpp:1723)"""
    dst = dst if dst is not None else _new(src, dtype=_ddepth_dtype(src, ddepth))
    ms, md = _pair(src, dst)
    kx, pkx = _f32(kernelX)
    ky, pky = _f32(kernelY)
    _check(lib().b200cv_sep_filter2d(ctypes.byref(ms), ctypes.byref(md), pkx, len(kx), pky, len(ky), int(anchor[0]), int(anchor[1]),
                                     ctypes.c_double(delta), int(borderType), _stream_ptr(stream)), "sepFilter2D")
    return dst


def filter2D(src, ddepth, kernel, anchor=(-1, -1), delta=0.0, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::filter2D (imgproc.hpp:1702)"""
    dst = dst if dst is not None else _new(src, dtype=_ddepth_dtype(src, ddepth))
    ms, md = _pair(src, dst)
    k = np.asarray(kernel, dtype=np.float32)
    kh, kw = k.shape
    kk, pk = _f32(k)
    _check(lib().b200cv_filter2d(ctypes.byref(ms), ctypes.byref(md), pk, kw, kh, int(anchor[0]), int(anchor[1]),
                                 ctypes.c_double(delta), int(borderType), _stream_ptr(stream)), "filter2D")
    return dst


def Sobel(src, ddepth, dx, dy, ksize=3, scale=1.0, delta=0.0, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::Sobel (imgproc.hpp:1862)"""
    if not _is_torch(src):
        from . import hal
        return hal.Sobel(src, ddepth, dx, dy, ksize, scale, delta, borderType, dst)
    dst = dst if dst is not None else _new(src, dtype=_ddepth_dtype(src, ddepth))
    ms, md = _pair(src, dst)
    _check(lib().b200cv_sobel(ctypes.byref(ms), ctypes.byref(md), int(dx), int(dy), int(ksize), ctypes.c_double(scale),
                              ctypes.c_double(delta), int(borderType), _stream_ptr(stream)), "Sobel")
    return dst


def Laplacian(src, ddepth, ksize=1, scale=1, delta=0, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::Laplacian (imgproc.hpp): 8U -> 8U / 16S / 32F and 32F -> 32F, 1 to 4 channels, odd ksize 1..31; ddepth -1 keeps the source
    depth.  A 64F destination (the cv2.Laplacian(gray, cv2.CV_64F) focus-measure idiom) is not offered."""
    if not _is_torch(src):
        from . import hal
        return hal.Laplacian(src, ddepth, ksize, scale, delta, borderType, dst)
    dst = dst if dst is not None else _new(src, dtype=_ddepth_dtype(src, ddepth))
    ms, md = _pair(src, dst)
    _check(lib().b200cv_laplacian(ctypes.byref(ms), ctypes.byref(md), int(ksize), ctypes.c_double(scale), ctypes.c_double(delta),
                                  int(borderType), _stream_ptr(stream)), "Laplacian")
    return dst


def getStructuringElement(shape, ksize, anchor=(-1, -1)):
    """cv::getStructuringElement (morph.dispatch.cpp), computed on the host: a (h, w) uint8 array of 0 / 1 for MORPH_RECT, MORPH_CROSS
    or MORPH_ELLIPSE; a 1x1 size is always a rectangle.  Ellipse rows span c +- round(c * sqrt((r^2 - dy^2) / r^2)), half to even."""
    import math
    import numpy as np
    w, h = int(ksize[0]), int(ksize[1])
    if shape not in (MORPH_RECT, MORPH_CROSS, MORPH_ELLIPSE):
        raise B200cvError("getStructuringElement: unknown shape %r" % (shape,))
    ax = w // 2 if anchor[0] == -1 else int(anchor[0])
    ay = h // 2 if anchor[1] == -1 else int(anchor[1])
    if not (0 <= ax < w and 0 <= ay < h):
        raise B200cvError("getStructuringElement: the anchor must lie inside the element")
    if (w, h) == (1, 1):
        shape = MORPH_RECT
    r, c = h // 2, w // 2
    inv_r2 = 1.0 / (float(r) * r) if r else 0.0
    elem = np.zeros((h, w), np.uint8)
    for i in range(h):
        j1 = j2 = 0
        if shape == MORPH_RECT or (shape == MORPH_CROSS and i == ay):
            j2 = w
        elif shape == MORPH_CROSS:
            j1, j2 = ax, ax + 1
        elif abs(i - r) <= r:
            dx = int(round(c * math.sqrt((r * r - (i - r) * (i - r)) * inv_r2)))
            j1, j2 = max(c - dx, 0), min(c + dx + 1, w)
        elem[i, j1:j2] = 1
    return elem


def _morph_args(kernel, borderValue, entry_ex):
    """(k, kp, kw, kh, bv) for b200cv_morphology / b200cv_host_morphology: k is the element as a contiguous 0 / 1 byte mask (None for
    the empty element: None or any array, list or tensor of size 0) and kp its pointer, kw / kh its size, bv the double[4] border value
    (None: the reference's default, four DBL_MAX).  entry_ex (morphologyEx) turns the empty element into the 3x3 rectangle for every op,
    as the reference's morphologyEx does; erode / dilate keep it empty, their own (1 + 2 * iterations)^2 rule."""
    import numpy as np
    if kernel is not None and _is_torch(kernel):
        kernel = kernel.cpu().numpy()
    if (kernel is None or np.asarray(kernel).size == 0) and entry_ex:
        kernel = np.ones((3, 3), np.uint8)
    if kernel is None or np.asarray(kernel).size == 0:
        k, kw, kh = None, 0, 0
    else:
        k = np.ascontiguousarray(np.asarray(kernel) != 0, dtype=np.uint8)
        if k.ndim == 1:
            k = k.reshape(1, -1)
        kh, kw = k.shape
    if borderValue is None:
        bv = [1.7976931348623157e308] * 4
    else:
        vals = [float(v) for v in (borderValue if hasattr(borderValue, "__len__") else (borderValue,))]
        bv = (vals + [0.0] * 4)[:4]
    kp = None if k is None else k.ctypes.data_as(ctypes.POINTER(ctypes.c_ubyte))
    return k, kp, kw, kh, (ctypes.c_double * 4)(*bv)


def morphologyEx(src, op, kernel, dst=None, anchor=(-1, -1), iterations=1, borderType=BORDER_CONSTANT, borderValue=None, stream=None):
    """cv::morphologyEx (imgproc.hpp): MORPH_ERODE .. MORPH_BLACKHAT over 8U / 16U / 16S / 32F images of 1 to 4 channels, or (N, H, W, C)
    batches.  kernel: any 2-D array, non-zero meaning "in the element"; None or an empty array, list or tensor is the 3x3 rectangle.  borderValue None is the
    reference's morphologyDefaultBorderValue().  MORPH_HITMISS is not offered."""
    return _morphology(src, op, kernel, dst, anchor, iterations, borderType, borderValue, stream, True)


def erode(src, kernel, dst=None, anchor=(-1, -1), iterations=1, borderType=BORDER_CONSTANT, borderValue=None, stream=None):
    """cv::erode (imgproc.hpp); kernel None is the reference's empty element, a (1+2*iterations)^2 rectangle applied once"""
    return _morphology(src, MORPH_ERODE, kernel, dst, anchor, iterations, borderType, borderValue, stream)


def dilate(src, kernel, dst=None, anchor=(-1, -1), iterations=1, borderType=BORDER_CONSTANT, borderValue=None, stream=None):
    """cv::dilate (imgproc.hpp); kernel None is the reference's empty element, a (1+2*iterations)^2 rectangle applied once"""
    return _morphology(src, MORPH_DILATE, kernel, dst, anchor, iterations, borderType, borderValue, stream)


def _morphology(src, op, kernel, dst, anchor, iterations, borderType, borderValue, stream, entry_ex=False):
    if not _is_torch(src):
        from . import hal
        return hal._morphology(src, op, kernel, dst, anchor, iterations, borderType, borderValue, entry_ex)
    dst = dst if dst is not None else _new(src)
    ms, md = _pair(src, dst)
    k, kp, kw, kh, bv = _morph_args(kernel, borderValue, entry_ex)
    _check(lib().b200cv_morphology(ctypes.byref(ms), ctypes.byref(md), int(op), kp, ctypes.c_size_t(kw), int(kw), int(kh), int(anchor[0]),
                                   int(anchor[1]), int(iterations), int(borderType), bv, _stream_ptr(stream)), "morphology")
    return dst


def boxFilter(src, ddepth, ksize, anchor=(-1, -1), normalize=True, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::boxFilter (imgproc.hpp:1603)"""
    if not _is_torch(src):
        from . import hal
        return hal.boxFilter(src, ddepth, ksize, anchor, normalize, borderType, dst)
    dst = dst if dst is not None else _new(src, dtype=_ddepth_dtype(src, ddepth))
    ms, md = _pair(src, dst)
    _check(lib().b200cv_box_filter(ctypes.byref(ms), ctypes.byref(md), int(ksize[0]), int(ksize[1]), int(anchor[0]), int(anchor[1]),
                                   int(bool(normalize)), int(borderType), _stream_ptr(stream)), "boxFilter")
    return dst


def blur(src, ksize, anchor=(-1, -1), borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::blur (imgproc.hpp:1659) = boxFilter(src, -1, ksize, anchor, true, borderType)"""
    return boxFilter(src, -1, ksize, anchor, True, borderType, dst, stream)


def Scharr(src, ddepth, dx, dy, scale=1.0, delta=0.0, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::Scharr (imgproc.hpp:1928) = cv::Sobel with ksize = FILTER_SCHARR (deriv.cpp:468-510)"""
    return Sobel(src, ddepth, dx, dy, -1, scale, delta, borderType, dst, stream)


_CVT_DCN = {COLOR_BGR2BGRA: 4, COLOR_BGRA2BGR: 3, COLOR_BGR2RGBA: 4, COLOR_RGBA2BGR: 3, COLOR_BGR2RGB: 3, COLOR_BGRA2RGBA: 4,
            COLOR_BGR2GRAY: 1, COLOR_RGB2GRAY: 1, COLOR_BGRA2GRAY: 1, COLOR_RGBA2GRAY: 1, COLOR_GRAY2BGR: 3, COLOR_GRAY2BGRA: 4,
            139: 4, 140: 4, 141: 4, 142: 4, 86: 1, 87: 1, 88: 1, 89: 1}


def _cvt_dst_geometry(code, cols, rows, dstCn=0):
    """(width, height, channels) of cv::cvtColor's destination (color.cpp:323-372 for the subsampled-YUV codes)"""
    if 90 <= code <= 105:
        return cols, rows * 2 // 3, (4 if code in (94, 95, 96, 97, 102, 103, 104, 105) else 3)
    if code == 106:
        return cols, rows * 2 // 3, 1
    if 107 <= code <= 122:
        return cols, rows, (4 if code in (111, 112, 119, 120, 121, 122) else 3)
    if code in (123, 124):
        return cols, rows, 1
    if 127 <= code <= 134:
        return cols, rows * 3 // 2, 1
    if 143 <= code <= 154:
        return cols, rows, 2
    return cols, rows, (dstCn if dstCn > 0 else _CVT_DCN.get(code, 3))


def cvtColor(src, code, dstCn=0, dst=None, stream=None):
    """cv::cvtColor (imgproc.hpp:3736)"""
    if not _is_torch(src):
        from . import hal
        return hal.cvtColor(src, code, dstCn)
    m = describe(src)
    w, h, dcn = _cvt_dst_geometry(int(code), m.cols, m.rows, dstCn)
    dst = dst if dst is not None else _new(src, channels=dcn, size=(w, h))
    ms, md = _pair(src, dst)
    _check(lib().b200cv_cvt_color(ctypes.byref(ms), ctypes.byref(md), int(code), _stream_ptr(stream)), "cvtColor")
    return dst


def cvtColorTwoPlane(src1, src2, code, dst=None, stream=None):
    """cv::cvtColorTwoPlane: NV12 / NV21 with separate luma (H,W) and chroma (H/2,W/2,2) tensors (batches: (N,H,W,1) and (N,H/2,W/2,2))"""
    m = describe(src1)
    dcn = 4 if int(code) in (94, 95, 96, 97) else 3
    dst = dst if dst is not None else _new(src1, channels=dcn)
    my, muv, md = describe(src1), describe(src2), describe(dst)
    _check(lib().b200cv_cvt_color_two_plane(ctypes.byref(my), ctypes.byref(muv), ctypes.byref(md), int(code), _stream_ptr(stream)), "cvtColorTwoPlane")
    return dst


def integral(src, with_sqsum=False, stream=None):
    """cv::integral for 8UC1 frames: the (H+1) x (W+1) int32 sum, and with with_sqsum=True also the float64 sum of squares.
    (H,W) or (N,H,W,1) torch CUDA tensors; numpy arrays take the host path."""
    if not _is_torch(src):
        from . import hal
        return hal.integral(src, with_sqsum)
    import torch
    m = describe(src)
    s = _new(src, dtype=torch.int32, channels=1, size=(m.cols + 1, m.rows + 1))
    q = _new(src, dtype=torch.float64, channels=1, size=(m.cols + 1, m.rows + 1)) if with_sqsum else None
    ms, md = describe(src), describe(s)
    mq = describe(q) if with_sqsum else None
    _check(lib().b200cv_integral(ctypes.byref(ms), ctypes.byref(md), ctypes.byref(mq) if with_sqsum else None, _stream_ptr(stream)), "integral")
    return (s, q) if with_sqsum else s


def getGaussianKernel(ksize, sigma):
    """cv::getGaussianKernel as float64 (bit-exact softdouble arithmetic on the host)"""
    out = np.zeros(ksize, np.float64)
    _check(lib().b200cv_get_gaussian_kernel(int(ksize), ctypes.c_double(sigma), out.ctypes.data_as(ctypes.POINTER(ctypes.c_double))),
           "getGaussianKernel")
    return out


def getGaussianKernelFixed(ksize, sigma, bits):
    """the fixed-point taps GaussianBlur uses for 8-bit (bits = 8) and 16-bit (bits = 16) images"""
    out = np.zeros(ksize, np.uint32)
    _check(lib().b200cv_get_gaussian_kernel_fixed(int(ksize), ctypes.c_double(sigma), int(bits), out.ctypes.data_as(ctypes.c_void_p)), "getGaussianKernelFixed")
    return out


def getGaussianKernelFixed8(ksize, sigma):
    out = np.zeros(ksize, np.uint16)
    _check(lib().b200cv_get_gaussian_kernel_fixed8(int(ksize), ctypes.c_double(sigma), out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16))),
           "getGaussianKernelFixed8")
    return out


def resize(src, dsize, fx=0, fy=0, interpolation=INTER_LINEAR, dst=None, stream=None):
    """cv::resize (imgproc.hpp:2422).  dsize=(w,h); or dsize=None and fx, fy."""
    if not _is_torch(src):
        from . import hal
        return hal.resize(src, dsize, fx, fy, interpolation)
    m = describe(src)
    by_factor = not dsize or dsize[0] <= 0
    if by_factor:
        dsize = (int(round(m.cols * fx)), int(round(m.rows * fy)))    # saturate_cast<int>(cols*fx): round-half-even like Python's round
    dst = dst if dst is not None else _new(src, size=(int(dsize[0]), int(dsize[1])))
    ms, md = _pair(src, dst)
    if by_factor:      # the sampling scale is fx, fy themselves, not dst / src (resize.cpp:4214-4228)
        _check(lib().b200cv_resize_scaled(ctypes.byref(ms), ctypes.byref(md), int(interpolation), ctypes.c_double(fx), ctypes.c_double(fy), _stream_ptr(stream)), "resize")
    else:
        _check(lib().b200cv_resize(ctypes.byref(ms), ctypes.byref(md), int(interpolation), _stream_ptr(stream)), "resize")
    return dst


def _warp(fn, name, src, M, dsize, flags, borderMode, borderValue, dst, stream, n):
    dst = dst if dst is not None else _new(src, size=(int(dsize[0]), int(dsize[1])))
    ms, md = _pair(src, dst)
    m, pm = _f64(M)
    assert len(m) == n
    bv = np.zeros(4, np.float64)
    b = np.atleast_1d(np.asarray(borderValue, np.float64))
    bv[:len(b)] = b
    _check(fn(ctypes.byref(ms), ctypes.byref(md), pm, int(flags), int(borderMode), bv.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
              _stream_ptr(stream)), name)
    return dst


def warpAffine(src, M, dsize, flags=INTER_LINEAR, borderMode=BORDER_CONSTANT, borderValue=0, dst=None, stream=None):
    """cv::warpAffine (imgproc.hpp:2450)"""
    return _warp(lib().b200cv_warp_affine, "warpAffine", src, M, dsize, flags, borderMode, borderValue, dst, stream, 6)


def warpPerspective(src, M, dsize, flags=INTER_LINEAR, borderMode=BORDER_CONSTANT, borderValue=0, dst=None, stream=None):
    """cv::warpPerspective (imgproc.hpp:2482)"""
    return _warp(lib().b200cv_warp_perspective, "warpPerspective", src, M, dsize, flags, borderMode, borderValue, dst, stream, 9)


def remap(src, map1, map2, interpolation, borderMode=BORDER_CONSTANT, borderValue=0, dst=None, stream=None):
    """cv::remap (imgproc.hpp:2531).  map1/map2: float32 (H,W) planes, map1 float32 (H,W,2) with map2=None, or the fixed-point pair of
    cv::convertMaps: map1 int16 (H,W,2) + map2 int16/None (H,W).  dst takes the size of the maps."""
    m1 = describe(map1)
    dst = dst if dst is not None else _new(src, size=(m1.cols, m1.rows))
    ms, md = _pair(src, dst)
    m2 = describe(map2) if map2 is not None else None
    bv = np.zeros(4, np.float64)
    b = np.atleast_1d(np.asarray(borderValue, np.float64))
    bv[:len(b)] = b
    _check(lib().b200cv_remap(ctypes.byref(ms), ctypes.byref(md), ctypes.byref(m1), ctypes.byref(m2) if m2 is not None else None, int(interpolation),
                              int(borderMode), bv.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), _stream_ptr(stream)), "remap")
    return dst


def pyrDown(src, dst=None, borderType=BORDER_DEFAULT, stream=None):
    """cv::pyrDown (imgproc.hpp:3325), default destination size ((W+1)/2, (H+1)/2)"""
    m = describe(src)
    dst = dst if dst is not None else _new(src, size=((m.cols + 1) // 2, (m.rows + 1) // 2))
    ms, md = _pair(src, dst)
    _check(lib().b200cv_pyr_down(ctypes.byref(ms), ctypes.byref(md), int(borderType), _stream_ptr(stream)), "pyrDown")
    return dst


def pyrUp(src, dst=None, stream=None):
    """cv::pyrUp (imgproc.hpp:3351), destination 2W x 2H"""
    m = describe(src)
    dst = dst if dst is not None else _new(src, size=(m.cols * 2, m.rows * 2))
    ms, md = _pair(src, dst)
    _check(lib().b200cv_pyr_up(ctypes.byref(ms), ctypes.byref(md), int(BORDER_DEFAULT), _stream_ptr(stream)), "pyrUp")
    return dst


def matchTemplate(image, templ, method, result=None, stream=None, mask=None):
    """cv::matchTemplate (imgproc.hpp:3916): image (H,W) / (N,H,W,1), templ (h,w); result float32 (H-h+1, W-w+1); mask: uint8 / float32 (h,w)"""
    import torch
    mi, mt = describe(image), describe(templ)
    ow, oh = mi.cols - mt.cols + 1, mi.rows - mt.rows + 1
    if result is None:
        shape = [max(mi.frames, 1), oh, ow, 1] if image.dim() == 4 else [oh, ow]
        result = torch.empty(shape, dtype=torch.float32, device=image.device)
    mr = describe(result)
    if mask is not None:
        mm = describe(mask)
        _check(lib().b200cv_match_template_masked(ctypes.byref(mi), ctypes.byref(mt), ctypes.byref(mm), ctypes.byref(mr), int(method), _stream_ptr(stream)),
               "matchTemplate(mask)")
        return result
    _check(lib().b200cv_match_template(ctypes.byref(mi), ctypes.byref(mt), ctypes.byref(mr), int(method), _stream_ptr(stream)), "matchTemplate")
    return result


def cornerHarris(src, blockSize, ksize, k, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::cornerHarris (imgproc.hpp:1948)"""
    import torch
    dst = dst if dst is not None else _new(src, dtype=torch.float32)
    ms, md = _pair(src, dst)
    _check(lib().b200cv_corner_harris(ctypes.byref(ms), ctypes.byref(md), int(blockSize), int(ksize), ctypes.c_double(k), int(borderType),
                                      _stream_ptr(stream)), "cornerHarris")
    return dst


def cornerMinEigenVal(src, blockSize, ksize=3, borderType=BORDER_DEFAULT, dst=None, stream=None):
    """cv::cornerMinEigenVal (imgproc.hpp:1921)"""
    import torch
    dst = dst if dst is not None else _new(src, dtype=torch.float32)
    ms, md = _pair(src, dst)
    _check(lib().b200cv_corner_min_eigen_val(ctypes.byref(ms), ctypes.byref(md), int(blockSize), int(ksize), int(borderType),
                                             _stream_ptr(stream)), "cornerMinEigenVal")
    return dst


def _int32(v):
    """a Python int as the C int of the same bits (cv2 passes CV_CANNY_L2_GRADIENT = 1 << 31 inside apertureSize)"""
    return ((int(v) + (1 << 31)) % (1 << 32)) - (1 << 31)


def _is_array(x):
    return _is_torch(x) or isinstance(x, np.ndarray)


def Canny(*args, **kwargs):
    """cv::Canny (imgproc.hpp:1889, :1907), both of cv2's overloads:
        Canny(image, threshold1, threshold2, edges=None, apertureSize=3, L2gradient=False, stream=None)
        Canny(dx, dy, threshold1, threshold2, edges=None, L2gradient=False, stream=None)
    chosen by whether the second argument is an array.  Returns 8-bit edges (0 / 255), one channel, of the input's size."""
    if (len(args) > 1 and _is_array(args[1])) or "dy" in kwargs:
        return _canny_derivs(*args, **kwargs)
    return _canny_image(*args, **kwargs)


def _canny_image(image, threshold1, threshold2, edges=None, apertureSize=3, L2gradient=False, stream=None):
    if not _is_torch(image):
        from . import hal
        return hal.Canny(image, threshold1, threshold2, edges, apertureSize, L2gradient)
    import torch
    edges = edges if edges is not None else _new(image, dtype=torch.uint8, channels=1)
    ms, md = _pair(image, edges)
    _check(lib().b200cv_canny(ctypes.byref(ms), ctypes.byref(md), ctypes.c_double(threshold1), ctypes.c_double(threshold2), _int32(apertureSize),
                              int(bool(L2gradient)), _stream_ptr(stream)), "Canny")
    return edges


def _canny_derivs(dx, dy, threshold1, threshold2, edges=None, L2gradient=False, stream=None):
    if not _is_torch(dx):
        from . import hal
        return hal.Canny(dx, dy, threshold1, threshold2, edges, L2gradient)
    import torch
    edges = edges if edges is not None else _new(dx, dtype=torch.uint8, channels=1)
    mx, my, md = describe(dx), describe(dy), describe(edges)
    _check(lib().b200cv_canny_derivs(ctypes.byref(mx), ctypes.byref(my), ctypes.byref(md), ctypes.c_double(threshold1), ctypes.c_double(threshold2),
                                     int(bool(L2gradient)), _stream_ptr(stream)), "Canny")
    return edges


def distanceTransform(src, distanceType, maskSize, dst=None, dstType=CV_32F, stream=None):
    """cv::distanceTransform(src, distanceType, maskSize, dst, dstType) over an 8UC1 image or (N, H, W, 1) batch: the distance of every
    pixel to the nearest zero pixel.  The result is 8UC1 for DIST_L1 with dstType CV_8U (the saturating city-block call, which may run
    in place: dst=src) and 32FC1 otherwise, as in the reference.  DIST_C and DIST_L1 always use the 3x3 mask; maskSize 0
    (DIST_MASK_PRECISE) gives the exact Euclidean distance for every other type."""
    if not _is_torch(src):
        from . import hal
        return hal.distanceTransform(src, distanceType, maskSize, dst, dstType)
    import torch
    if dst is None:
        u8 = distanceType == DIST_L1 and dstType == CV_8U
        dst = _new(src, dtype=torch.uint8 if u8 else torch.float32, channels=1)
    ms, md = _pair(src, dst)
    _check(lib().b200cv_distance_transform(ctypes.byref(ms), ctypes.byref(md), int(distanceType), int(maskSize), _stream_ptr(stream)),
           "distanceTransform")
    return dst


def goodFeaturesToTrack(image, maxCorners, qualityLevel, minDistance, blockSize=3, gradientSize=3, useHarrisDetector=False, k=0.04,
                        max_out=None, stream=None, with_quality=False):
    """cv::goodFeaturesToTrack (imgproc.hpp:2096).  Returns an (n,2) float32 array of (x,y) for a single frame, or a list of
    such arrays for an (N,H,W,1) batch."""
    ms = describe(image)
    frames = max(ms.frames, 1)
    cap = int(max_out or (maxCorners if maxCorners > 0 else ms.cols * ms.rows))
    pts = np.zeros((frames, cap, 2), np.float32)
    q = np.zeros((frames, cap), np.float32)
    cnt = np.zeros(frames, np.int32)
    _check(lib().b200cv_good_features_to_track(ctypes.byref(ms), pts.ctypes.data_as(ctypes.c_void_p), q.ctypes.data_as(ctypes.c_void_p), cap,
                                               cnt.ctypes.data_as(ctypes.c_void_p), int(maxCorners), ctypes.c_double(qualityLevel),
                                               ctypes.c_double(minDistance), int(blockSize), int(gradientSize), int(bool(useHarrisDetector)),
                                               ctypes.c_double(k), _stream_ptr(stream)), "goodFeaturesToTrack")
    out = [(pts[f, :min(cnt[f], cap)].copy(), q[f, :min(cnt[f], cap)].copy()) for f in range(frames)]
    if not with_quality:
        out = [o[0] for o in out]
    return out if image.dim() == 4 else out[0]


def sift_detectAndCompute(gray, nfeatures=0, nOctaveLayers=3, contrastThreshold=0.04, edgeThreshold=10, sigma=1.6, max_keypoints=200000,
                          with_descriptors=True, stream=None, enable_precise_upscale=True, mask=None):
    """cv::SIFT::create(nfeatures, nOctaveLayers, contrastThreshold, edgeThreshold, sigma, enable_precise_upscale)->detectAndCompute(gray) for one
    (H,W) CV_8U frame: pyramid, extrema, refinement, orientation and descriptors all on the device.
    Returns (keypoints[n,5] = x, y, size, angle, response; octave[n] int32; descriptors[n,128] float32 or None) as numpy arrays."""
    if gray.dim() == 4:           # a batch: frame by frame (the detector returns host data and synchronises per frame)
        return [sift_detectAndCompute(gray[f, :, :, 0], nfeatures, nOctaveLayers, contrastThreshold, edgeThreshold, sigma, max_keypoints, with_descriptors,
                                      stream, enable_precise_upscale, None if mask is None else (mask if mask.ndim == 2 else mask[f])) for f in range(gray.shape[0])]
    assert gray.dim() == 2
    m8 = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    G, D, dims = sift_pyramid(gray, nOctaveLayers, sigma, 1 if enable_precise_upscale else 2, True, stream)
    dims32 = np.ascontiguousarray(dims, np.int32).reshape(-1)
    kp = np.zeros((max_keypoints, 6), np.float32)
    desc = np.zeros((max_keypoints, 128), np.float32) if with_descriptors else None
    n = ctypes.c_int(0)
    _check(lib().b200cv_sift_detect_and_compute(ctypes.c_void_p(G.data_ptr()), ctypes.c_void_p(D.data_ptr()), dims32.ctypes.data_as(ctypes.c_void_p),
                                                len(dims32) // 2, int(nOctaveLayers), ctypes.c_double(contrastThreshold), ctypes.c_double(edgeThreshold),
                                                ctypes.c_double(sigma), -1, int(nfeatures),
                                                m8.ctypes.data_as(ctypes.c_void_p) if m8 is not None else None, ctypes.c_size_t(m8.strides[0] if m8 is not None else 0),
                                                int(m8.shape[1]) if m8 is not None else 0, int(m8.shape[0]) if m8 is not None else 0,
                                                int(max_keypoints), kp.ctypes.data_as(ctypes.c_void_p),
                                                desc.ctypes.data_as(ctypes.c_void_p) if with_descriptors else None, ctypes.byref(n), _stream_ptr(stream)),
           "sift_detectAndCompute")
    m = min(n.value, max_keypoints)
    return kp[:m, :5].copy(), kp[:m, 5].copy().view(np.int32), (desc[:m].copy() if with_descriptors else None)


class GFTTDetector:
    """cv::GFTTDetector (features2d.hpp; features2d/src/gftt.cpp:44-157): the Feature2D face of goodFeaturesToTrack.  detect() returns an
    (n, 4) float32 array per frame: x, y, size (= blockSize, gftt.cpp:147), response (the corner quality); angle / octave are unset
    in the reference (-1 / 0).  3- and 4-channel frames are converted with COLOR_BGR2GRAY first, as the reference does (gftt.cpp:139-140)."""

    def __init__(self, maxCorners=1000, qualityLevel=0.01, minDistance=1, blockSize=3, gradientSize=3, useHarrisDetector=False, k=0.04):
        self.maxCorners, self.qualityLevel, self.minDistance = int(maxCorners), float(qualityLevel), float(minDistance)
        self.blockSize, self.gradientSize, self.useHarrisDetector, self.k = int(blockSize), int(gradientSize), bool(useHarrisDetector), float(k)

    @staticmethod
    def create(maxCorners=1000, qualityLevel=0.01, minDistance=1, blockSize=3, gradientSize=3, useHarrisDetector=False, k=0.04):
        return GFTTDetector(maxCorners, qualityLevel, minDistance, blockSize, gradientSize, useHarrisDetector, k)

    def setMaxFeatures(self, v): self.maxCorners = int(v)
    def getMaxFeatures(self): return self.maxCorners
    def setQualityLevel(self, v): self.qualityLevel = float(v)
    def getQualityLevel(self): return self.qualityLevel
    def setMinDistance(self, v): self.minDistance = float(v)
    def getMinDistance(self): return self.minDistance
    def setBlockSize(self, v): self.blockSize = int(v)
    def getBlockSize(self): return self.blockSize
    def setGradientSize(self, v): self.gradientSize = int(v)
    def getGradientSize(self): return self.gradientSize
    def setHarrisDetector(self, v): self.useHarrisDetector = bool(v)
    def getHarrisDetector(self): return self.useHarrisDetector
    def setK(self, v): self.k = float(v)
    def getK(self): return self.k

    def detect(self, image, stream=None):
        m = describe(image)
        if _cn(m) != 1:
            image = cvtColor(image, COLOR_BGR2GRAY if _cn(m) == 3 else COLOR_BGRA2GRAY, stream=stream)
        res = goodFeaturesToTrack(image, self.maxCorners, self.qualityLevel, self.minDistance, self.blockSize, self.gradientSize,
                                  self.useHarrisDetector, self.k, stream=stream, with_quality=True)
        def pack(r):
            pts, q = r
            return np.concatenate([pts, np.full((len(pts), 1), float(self.blockSize), np.float32), q[:, None]], axis=1).astype(np.float32)
        return [pack(r) for r in res] if image.dim() == 4 else pack(res)


def sift_pyramid_layout(width, height, nOctaveLayers=3, upscale=True):
    no = ctypes.c_int(0)
    ge, de = ctypes.c_size_t(0), ctypes.c_size_t(0)
    dims = np.zeros(64, np.int32)
    _check(lib().b200cv_sift_pyramid_layout(int(width), int(height), int(nOctaveLayers), int(bool(upscale)), ctypes.byref(no), ctypes.byref(ge),
                                            ctypes.byref(de), dims.ctypes.data_as(ctypes.c_void_p)), "sift_pyramid_layout")
    return no.value, ge.value, de.value, dims[:2 * no.value].reshape(-1, 2).copy()


def sift_pyramid(gray, nOctaveLayers=3, sigma=1.6, upscale=True, with_dog=True, stream=None):
    """SIFT Gaussian + DoG pyramids (sift.dispatch.cpp:176-310) of a (H,W) frame or (N,H,W,1) batch of CV_8U frames.
    Returns (gauss, dog, dims): flat float32 CUDA tensors of shape (N, elems) packed image after image, octave-major,
    and the per-octave (w,h) table."""
    import torch
    ms = describe(gray)
    frames = max(ms.frames, 1)
    no, ge, de, dims = sift_pyramid_layout(ms.cols, ms.rows, nOctaveLayers, upscale)
    gstride = (ge + 3) & ~3
    dstride = (de + 3) & ~3
    G = torch.empty((frames, gstride), dtype=torch.float32, device=gray.device)
    D = torch.empty((frames, dstride), dtype=torch.float32, device=gray.device) if with_dog else None
    _check(lib().b200cv_sift_pyramid(ctypes.byref(ms), int(nOctaveLayers), ctypes.c_double(sigma), int(upscale),      # 2: SIFT::create's default first octave
                                     ctypes.c_void_p(G.data_ptr()), ctypes.c_size_t(gstride),
                                     ctypes.c_void_p(D.data_ptr() if with_dog else 0), ctypes.c_size_t(dstride), _stream_ptr(stream)), "sift_pyramid")
    return G, D, dims
