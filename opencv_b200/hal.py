"""opencv_b200.hal -- the HOST-memory face: numpy arrays (cv::Mat layout) in, numpy arrays out.

Each function is the cv2-named call over host memory; it goes through the batched host C ABI
(b200cv_host_*, include/b200cv_hal.h): frames are uploaded, processed by the same sm_90a kernels and
downloaded through a 3-stream pipeline.  Arrays: (H,W), (H,W,C) or a batch (N,H,W,C).
`pinned_empty` allocates page-locked numpy arrays (b200cv_host_alloc) for full PCIe speed.
"""
import ctypes

import numpy as np

from . import (BORDER_CONSTANT, BORDER_DEFAULT, INTER_LINEAR, CV_8U, CV_16S, CV_32F, Mat, _check, lib, make_type, _CVT_DCN, _cvt_dst_geometry)

_DEPTH = {np.dtype(np.uint8): CV_8U, np.dtype(np.uint16): 2, np.dtype(np.int16): CV_16S, np.dtype(np.float32): CV_32F,
          np.dtype(np.int32): 4, np.dtype(np.float64): 6}
_NP = {CV_8U: np.uint8, CV_16S: np.int16, CV_32F: np.float32}


def describe(a):
    assert isinstance(a, np.ndarray)
    depth = _DEPTH[a.dtype]
    es = a.itemsize
    if a.ndim == 2:
        n, h, w, c = 1, a.shape[0], a.shape[1], 1
        fs, rs = 0, a.strides[0]
        assert a.strides[1] == es and a.strides[0] > 0, "rows must be dense and ascending (a[:, ::2], a.T and flipped views are not cv::Mat layouts)"
    elif a.ndim == 3:
        n, (h, w, c) = 1, a.shape
        fs, rs = 0, a.strides[0]
        assert a.strides[2] == es and a.strides[1] == es * c
    elif a.ndim == 4:
        n, h, w, c = a.shape
        fs, rs = a.strides[0], a.strides[1]
        assert a.strides[3] == es and a.strides[2] == es * c
    else:
        raise ValueError("unsupported rank")
    return Mat(a.ctypes.data, rs, w, h, make_type(depth, c), n, fs)


def _new(src, dtype=None, channels=None, size=None):
    m = describe(src)
    c = (((m.type >> 3) & 511) + 1) if channels is None else channels
    w, h = (m.cols, m.rows) if size is None else size
    if src.ndim == 4:
        shape = (max(m.frames, 1), h, w, c)
    elif c == 1:
        shape = (h, w)
    else:
        shape = (h, w, c)
    return np.empty(shape, dtype or src.dtype)


_pinned = []


def pinned_empty(shape, dtype):
    """page-locked numpy array (kept alive for the life of the process)"""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = ctypes.c_void_p()
    _check(lib().b200cv_host_alloc(ctypes.byref(p), ctypes.c_size_t(max(n, 1))), "host_alloc")
    buf = (ctypes.c_ubyte * n).from_address(p.value)
    a = np.frombuffer(buf, dtype=dtype).reshape(shape)
    _pinned.append((p, buf))
    return a


def _ddt(src, ddepth):
    return src.dtype if ddepth is None or ddepth < 0 else _NP[ddepth]


def GaussianBlur(src, ksize, sigmaX, sigmaY=0, borderType=BORDER_DEFAULT, dst=None):
    dst = dst if dst is not None else _new(src)
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_gaussian_blur(ctypes.byref(ms), ctypes.byref(md), int(ksize[0]), int(ksize[1]), ctypes.c_double(sigmaX),
                                           ctypes.c_double(sigmaY), int(borderType)), "GaussianBlur")
    return dst


def sepFilter2D(src, ddepth, kernelX, kernelY, anchor=(-1, -1), delta=0.0, borderType=BORDER_DEFAULT, dst=None):
    dst = dst if dst is not None else _new(src, dtype=_ddt(src, ddepth))
    kx = np.ascontiguousarray(kernelX, np.float32).reshape(-1)
    ky = np.ascontiguousarray(kernelY, np.float32).reshape(-1)
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_sep_filter2d(ctypes.byref(ms), ctypes.byref(md), kx.ctypes.data_as(ctypes.c_void_p), len(kx),
                                          ky.ctypes.data_as(ctypes.c_void_p), len(ky), int(anchor[0]), int(anchor[1]), ctypes.c_double(delta),
                                          int(borderType)), "sepFilter2D")
    return dst


def filter2D(src, ddepth, kernel, anchor=(-1, -1), delta=0.0, borderType=BORDER_DEFAULT, dst=None):
    dst = dst if dst is not None else _new(src, dtype=_ddt(src, ddepth))
    k = np.ascontiguousarray(kernel, np.float32)
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_filter2d(ctypes.byref(ms), ctypes.byref(md), k.ctypes.data_as(ctypes.c_void_p), k.shape[1], k.shape[0],
                                      int(anchor[0]), int(anchor[1]), ctypes.c_double(delta), int(borderType)), "filter2D")
    return dst


def Sobel(src, ddepth, dx, dy, ksize=3, scale=1.0, delta=0.0, borderType=BORDER_DEFAULT, dst=None):
    dst = dst if dst is not None else _new(src, dtype=_ddt(src, ddepth))
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_sobel(ctypes.byref(ms), ctypes.byref(md), int(dx), int(dy), int(ksize), ctypes.c_double(scale), ctypes.c_double(delta),
                                   int(borderType)), "Sobel")
    return dst


def Scharr(src, ddepth, dx, dy, scale=1.0, delta=0.0, borderType=BORDER_DEFAULT, dst=None):
    return Sobel(src, ddepth, dx, dy, -1, scale, delta, borderType, dst)


def cvtColor(src, code, dstCn=0, dst=None):
    m = describe(src)
    w, h, dcn = _cvt_dst_geometry(int(code), m.cols, m.rows, dstCn)
    dst = dst if dst is not None else _new(src, channels=dcn, size=(w, h))
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_cvt_color(ctypes.byref(ms), ctypes.byref(md), int(code)), "cvtColor")
    return dst


def resize(src, dsize, fx=0, fy=0, interpolation=INTER_LINEAR, dst=None):
    m = describe(src)
    by_factor = not dsize or dsize[0] <= 0
    if by_factor:
        dsize = (int(round(m.cols * fx)), int(round(m.rows * fy)))
    dst = dst if dst is not None else _new(src, size=(int(dsize[0]), int(dsize[1])))
    ms, md = describe(src), describe(dst)
    if by_factor:      # the sampling scale is fx, fy themselves, not dst / src (resize.cpp:4214-4228)
        _check(lib().b200cv_host_resize_scaled(ctypes.byref(ms), ctypes.byref(md), int(interpolation), ctypes.c_double(fx), ctypes.c_double(fy)), "resize")
    else:
        _check(lib().b200cv_host_resize(ctypes.byref(ms), ctypes.byref(md), int(interpolation)), "resize")
    return dst


def _warp(fn, name, src, M, dsize, flags, borderMode, borderValue, dst):
    dst = dst if dst is not None else _new(src, size=(int(dsize[0]), int(dsize[1])))
    m = np.ascontiguousarray(M, np.float64).reshape(-1)
    bv = np.zeros(4, np.float64)
    b = np.atleast_1d(np.asarray(borderValue, np.float64))
    bv[:len(b)] = b
    ms, md = describe(src), describe(dst)
    _check(fn(ctypes.byref(ms), ctypes.byref(md), m.ctypes.data_as(ctypes.c_void_p), int(flags), int(borderMode), bv.ctypes.data_as(ctypes.c_void_p)), name)
    return dst


def warpAffine(src, M, dsize, flags=INTER_LINEAR, borderMode=BORDER_CONSTANT, borderValue=0, dst=None):
    return _warp(lib().b200cv_host_warp_affine, "warpAffine", src, M, dsize, flags, borderMode, borderValue, dst)


def warpPerspective(src, M, dsize, flags=INTER_LINEAR, borderMode=BORDER_CONSTANT, borderValue=0, dst=None):
    return _warp(lib().b200cv_host_warp_perspective, "warpPerspective", src, M, dsize, flags, borderMode, borderValue, dst)


def boxFilter(src, ddepth, ksize, anchor=(-1, -1), normalize=True, borderType=BORDER_DEFAULT, dst=None):
    dd = src.dtype if ddepth is None or ddepth < 0 else {0: np.uint8, 5: np.float32}[int(ddepth)]
    dst = dst if dst is not None else _new(src, dtype=dd)
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_box_filter(ctypes.byref(ms), ctypes.byref(md), int(ksize[0]), int(ksize[1]), int(anchor[0]), int(anchor[1]),
                                        int(bool(normalize)), int(borderType)), "boxFilter")
    return dst


def blur(src, ksize, anchor=(-1, -1), borderType=BORDER_DEFAULT, dst=None):
    return boxFilter(src, -1, ksize, anchor, True, borderType, dst)


def integral(src, with_sqsum=False):
    m = describe(src)
    s = _new(src, dtype=np.int32, channels=1, size=(m.cols + 1, m.rows + 1))
    q = _new(src, dtype=np.float64, channels=1, size=(m.cols + 1, m.rows + 1)) if with_sqsum else None
    ms, md = describe(src), describe(s)
    mq = describe(q) if with_sqsum else None
    _check(lib().b200cv_host_integral(ctypes.byref(ms), ctypes.byref(md), ctypes.byref(mq) if with_sqsum else None), "integral")
    return (s, q) if with_sqsum else s


def pyrDown(src, dst=None, borderType=BORDER_DEFAULT):
    m = describe(src)
    dst = dst if dst is not None else _new(src, size=((m.cols + 1) // 2, (m.rows + 1) // 2))
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_pyr_down(ctypes.byref(ms), ctypes.byref(md), int(borderType)), "pyrDown")
    return dst


def pyrUp(src, dst=None):
    m = describe(src)
    dst = dst if dst is not None else _new(src, size=(m.cols * 2, m.rows * 2))
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_pyr_up(ctypes.byref(ms), ctypes.byref(md), int(BORDER_DEFAULT)), "pyrUp")
    return dst


def remap(src, map1, map2, interpolation, borderMode=BORDER_CONSTANT, borderValue=0, dst=None):
    m1 = describe(map1)
    dst = dst if dst is not None else _new(src, size=(m1.cols, m1.rows))
    ms, md = describe(src), describe(dst)
    m2 = describe(map2) if map2 is not None else None
    bv = np.zeros(4, np.float64)
    b = np.atleast_1d(np.asarray(borderValue, np.float64))
    bv[:len(b)] = b
    _check(lib().b200cv_host_remap(ctypes.byref(ms), ctypes.byref(md), ctypes.byref(m1), ctypes.byref(m2) if m2 is not None else None, int(interpolation),
                                   int(borderMode), bv.ctypes.data_as(ctypes.POINTER(ctypes.c_double))), "remap")
    return dst


def cornerHarris(src, blockSize, ksize, k, borderType=BORDER_DEFAULT, dst=None):
    dst = dst if dst is not None else _new(src, dtype=np.float32)
    ms, md = describe(src), describe(dst)
    _check(lib().b200cv_host_corner_harris(ctypes.byref(ms), ctypes.byref(md), int(blockSize), int(ksize), ctypes.c_double(k), int(borderType)), "cornerHarris")
    return dst


def matchTemplate(image, templ, method, result=None):
    mi, mt = describe(image), describe(templ)
    ow, oh = mi.cols - mt.cols + 1, mi.rows - mt.rows + 1
    if result is None:
        result = np.empty((max(mi.frames, 1), oh, ow, 1) if image.ndim == 4 else (oh, ow), np.float32)
    mr = describe(result)
    _check(lib().b200cv_host_match_template(ctypes.byref(mi), ctypes.byref(mt), ctypes.byref(mr), int(method)), "matchTemplate")
    return result
