// b200cv.hpp -- C++ host-side mirror of the reference's operator surface for the hot path (header only, over the C ABI).
//
//   b200cv::GpuMat / Stream / Event / HostMem   the method sets of cv::cuda::GpuMat (create/upload/download/release, cuda.hpp:105-340),
//                                               cv::cuda::Stream (cuda.hpp:909-975), Event (:984-1016), HostMem (:791-870)
//   b200cv::Filter + create*Filter               the cv::cuda::Filter shape used by samples/cpp/tutorial_code/gpu/gpu-basics-similarity
//                                               (createGaussianFilter(type, type, ksize, sigma) -> apply(src, dst, stream))
//   b200cv::GaussianBlur, sepFilter2D, filter2D, Sobel, resize, warpAffine, warpPerspective, cvtColor, matchTemplate, cornerHarris,
//   cornerMinEigenVal, goodFeaturesToTrack,     same argument order and meaning as imgproc.hpp:1544,1723,1702,1862,2422,2450,2482,3736,
//   Canny, distanceTransform, Laplacian,        3916,1948,1921,2096,1889,1907, cv::distanceTransform, cv::Laplacian and cv::erode / dilate /
//   erode, dilate, morphologyEx                 morphologyEx (the element as a byte mask and its Size), with a trailing Stream& like the
//                                               cv::cuda:: functions
// With -DB200CV_WITH_OPENCV (OpenCV headers on the include path) b200cv_opencv.hpp adds namespace b200cv::cuda: the same operations over
// cv::InputArray / cv::OutputArray (cv::Mat, cv::cuda::GpuMat, cv::cuda::HostMem) with cv::cuda's Filter / Stream& shapes.
// Errors: the C ABI status is turned into b200cv::Error (std::runtime_error); NOT_IMPLEMENTED is b200cv::NotImplemented.
#pragma once
#ifdef B200CV_WITH_OPENCV
#include <opencv2/core.hpp>
#endif
#include <cfloat>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>
#include "../../include/b200cv.h"
#include "../../include/b200cv_hal.h"

namespace b200cv {

struct Error : std::runtime_error { int code; Error(int c, const std::string& m) : std::runtime_error(m), code(c) {} };
struct NotImplemented : Error { using Error::Error; };
inline void check(int rc, const char* what)
{
    if (rc == B200CV_OK) return;
    if (rc == B200CV_NOT_IMPLEMENTED) throw NotImplemented(rc, std::string(what) + ": not implemented on the device path");
    throw Error(rc, std::string(what) + ": " + b200cv_last_error());
}

struct Size { int width = 0, height = 0; Size() {} Size(int w, int h) : width(w), height(h) {} };
struct Point { int x = -1, y = -1; Point() {} Point(int x_, int y_) : x(x_), y(y_) {} };
struct Point2f { float x, y; };
struct Scalar { double val[4] = {0, 0, 0, 0}; Scalar() {} Scalar(double a, double b = 0, double c = 0, double d = 0) { val[0] = a; val[1] = b; val[2] = c; val[3] = d; } };

#ifndef CV_8U      // OpenCV's own depth macros when its headers came first (B200CV_WITH_OPENCV)
enum { CV_8U = 0, CV_16S = 3, CV_32F = 5 };
#endif
inline int makeType(int depth, int cn) { return B200CV_MAKETYPE(depth, cn); }
enum { BORDER_CONSTANT = 0, BORDER_REPLICATE = 1, BORDER_REFLECT = 2, BORDER_WRAP = 3, BORDER_REFLECT_101 = 4, BORDER_DEFAULT = 4 };
enum { INTER_NEAREST = 0, INTER_LINEAR = 1, INTER_CUBIC = 2, INTER_AREA = 3, INTER_LANCZOS4 = 4, INTER_LINEAR_EXACT = 5, INTER_NEAREST_EXACT = 6, WARP_INVERSE_MAP = 16 };

class Event;
class Stream {
public:
    Stream() { check(b200cv_stream_create(&s_), "Stream"); own_ = true; }
    explicit Stream(void* cuda_stream) : s_(cuda_stream), own_(false) {}
    ~Stream() { if (own_ && s_) b200cv_stream_destroy(s_); }
    Stream(const Stream&) = delete;
    Stream& operator=(const Stream&) = delete;
    bool queryIfComplete() const { int r = b200cv_stream_query(s_); if (r < 0) check(r, "queryIfComplete"); return r == 0; }
    void waitForCompletion() { check(b200cv_stream_synchronize(s_), "waitForCompletion"); }
    void waitEvent(const Event& e);
    typedef void (*StreamCallback)(int status, void* userData);
    void enqueueHostCallback(StreamCallback cb, void* userData) { check(b200cv_stream_add_callback(s_, cb, userData), "enqueueHostCallback"); }
    static Stream& Null() { static Stream n(nullptr); return n; }
    void* cudaPtr() const { return s_; }
private:
    void* s_ = nullptr; bool own_ = false;
};

class Event {
public:
    Event() { check(b200cv_event_create(&e_), "Event"); }
    ~Event() { if (e_) b200cv_event_destroy(e_); }
    void record(Stream& s = Stream::Null()) { check(b200cv_event_record(e_, s.cudaPtr()), "Event::record"); }
    void waitForCompletion() { check(b200cv_event_synchronize(e_), "Event::waitForCompletion"); }
    static float elapsedTime(const Event& a, const Event& b) { float ms = 0; check(b200cv_event_elapsed_ms(a.e_, b.e_, &ms), "elapsedTime"); return ms; }
    void* ptr() const { return e_; }
private:
    void* e_ = nullptr;
};
inline void Stream::waitEvent(const Event& e) { check(b200cv_stream_wait_event(s_, e.ptr()), "waitEvent"); }

// device image: cv::cuda::GpuMat fields (rows, cols, step, data, type) + an optional batch of frames
class GpuMat {
public:
    int rows = 0, cols = 0, frames = 1; size_t step = 0, frame_step = 0; unsigned char* data = nullptr;
    GpuMat() {}
    GpuMat(int r, int c, int t, int nframes = 1) { create(r, c, t, nframes); }
    GpuMat(int r, int c, int t, void* ptr, size_t stp) : rows(r), cols(c), step(stp), data((unsigned char*)ptr), type_(t) {}   // wraps user memory (cuda_gpu_mat.cpp:56-78)
    int type() const { return type_; }
    int channels() const { return B200CV_CN(type_); }
    bool empty() const { return !data; }
    Size size() const { return Size(cols, rows); }
    void create(int r, int c, int t, int nframes = 1)
    {
        if (data && r == rows && c == cols && t == type_ && nframes == frames) return;
        release();
        size_t es = (size_t)B200CV_CN(t) * (B200CV_DEPTH(t) <= 1 ? 1 : B200CV_DEPTH(t) <= 3 ? 2 : B200CV_DEPTH(t) == 6 ? 8 : 4);
        void* p = nullptr;
        check(b200cv_malloc_pitch(&p, &step, (size_t)c * es, (size_t)r * nframes), "GpuMat::create");
        own_.reset((unsigned char*)p, [](unsigned char* q) { b200cv_free(q); });
        data = (unsigned char*)p; rows = r; cols = c; type_ = t; frames = nframes; frame_step = step * r;
    }
    void release() { own_.reset(); data = nullptr; rows = cols = 0; }
    void upload(const void* host, size_t host_step, Stream& s = Stream::Null())
    { check(b200cv_upload(host, host_step, data, step, rowBytes(), (size_t)rows * frames, s.cudaPtr()), "upload"); if (!s.cudaPtr()) b200cv_stream_synchronize(nullptr); }
    void download(void* host, size_t host_step, Stream& s = Stream::Null()) const
    { check(b200cv_download(data, step, host, host_step, rowBytes(), (size_t)rows * frames, s.cudaPtr()), "download"); if (!s.cudaPtr()) b200cv_stream_synchronize(nullptr); }
    b200cvMat desc() const { b200cvMat m = {data, step, cols, rows, type_, frames, frame_step}; return m; }
private:
    size_t rowBytes() const { return (size_t)cols * B200CV_CN(type_) * (B200CV_DEPTH(type_) <= 1 ? 1 : B200CV_DEPTH(type_) <= 3 ? 2 : 4); }
    int type_ = 0; std::shared_ptr<unsigned char> own_;
};

class HostMem {   // page-locked host buffer (cv::cuda::HostMem::PAGE_LOCKED)
public:
    HostMem(size_t bytes) { check(b200cv_host_alloc(&p_, bytes), "HostMem"); }
    ~HostMem() { if (p_) b200cv_host_free(p_); }
    void* data() const { return p_; }
private:
    void* p_ = nullptr;
};

#define B200CV_DST(dst, src, t) (dst).create((src).rows, (src).cols, (t), (src).frames)

inline void GaussianBlur(const GpuMat& src, GpuMat& dst, Size ksize, double sigmaX, double sigmaY = 0, int borderType = BORDER_DEFAULT, Stream& s = Stream::Null())
{ B200CV_DST(dst, src, src.type()); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_gaussian_blur(&a, &b, ksize.width, ksize.height, sigmaX, sigmaY, borderType, s.cudaPtr()), "GaussianBlur"); }
inline void sepFilter2D(const GpuMat& src, GpuMat& dst, int ddepth, const std::vector<float>& kx, const std::vector<float>& ky, Point anchor = Point(), double delta = 0,
                        int borderType = BORDER_DEFAULT, Stream& s = Stream::Null())
{ B200CV_DST(dst, src, makeType(ddepth < 0 ? B200CV_DEPTH(src.type()) : ddepth, src.channels())); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_sep_filter2d(&a, &b, kx.data(), (int)kx.size(), ky.data(), (int)ky.size(), anchor.x, anchor.y, delta, borderType, s.cudaPtr()), "sepFilter2D"); }
inline void filter2D(const GpuMat& src, GpuMat& dst, int ddepth, const float* kernel, Size ksz, Point anchor = Point(), double delta = 0, int borderType = BORDER_DEFAULT,
                     Stream& s = Stream::Null())
{ B200CV_DST(dst, src, makeType(ddepth < 0 ? B200CV_DEPTH(src.type()) : ddepth, src.channels())); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_filter2d(&a, &b, kernel, ksz.width, ksz.height, anchor.x, anchor.y, delta, borderType, s.cudaPtr()), "filter2D"); }
inline void Sobel(const GpuMat& src, GpuMat& dst, int ddepth, int dx, int dy, int ksize = 3, double scale = 1, double delta = 0, int borderType = BORDER_DEFAULT,
                  Stream& s = Stream::Null())
{ B200CV_DST(dst, src, makeType(ddepth < 0 ? B200CV_DEPTH(src.type()) : ddepth, src.channels())); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_sobel(&a, &b, dx, dy, ksize, scale, delta, borderType, s.cudaPtr()), "Sobel"); }
// cv::Laplacian: 8U -> 8U / 16S / 32F and 32F -> 32F, odd ksize 1..31
inline void Laplacian(const GpuMat& src, GpuMat& dst, int ddepth, int ksize = 1, double scale = 1, double delta = 0, int borderType = BORDER_DEFAULT,
                      Stream& s = Stream::Null())
{ B200CV_DST(dst, src, makeType(ddepth < 0 ? B200CV_DEPTH(src.type()) : ddepth, src.channels())); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_laplacian(&a, &b, ksize, scale, delta, borderType, s.cudaPtr()), "Laplacian"); }
// cv::erode / cv::dilate / cv::morphologyEx: 8U / 16U / 16S / 32F, 1 to 4 channels.  The element is a host byte mask of ksize.height rows
// of ksize.width bytes (non-zero = in the element); nullptr is the empty element (erode / dilate: a (1+2*iterations)^2 rectangle;
// morphologyEx: 3x3).  The default borderValue is morphologyDefaultBorderValue() (four DBL_MAX).
inline Scalar morphologyDefaultBorderValue() { return Scalar(DBL_MAX, DBL_MAX, DBL_MAX, DBL_MAX); }
inline void morphologyEx(const GpuMat& src, GpuMat& dst, int op, const unsigned char* kernel, Size ksize, Point anchor = Point(-1, -1),
                         int iterations = 1, int borderType = BORDER_CONSTANT, const Scalar& borderValue = morphologyDefaultBorderValue(),
                         Stream& s = Stream::Null())
{ static const unsigned char k3[9] = {1, 1, 1, 1, 1, 1, 1, 1, 1};
  if (!kernel || ksize.width <= 0 || ksize.height <= 0) { kernel = k3; ksize = Size(3, 3); }
  B200CV_DST(dst, src, src.type()); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_morphology(&a, &b, op, kernel, (size_t)ksize.width, ksize.width, ksize.height, anchor.x, anchor.y, iterations, borderType,
                          borderValue.val, s.cudaPtr()), "morphologyEx"); }
inline void erode(const GpuMat& src, GpuMat& dst, const unsigned char* kernel, Size ksize, Point anchor = Point(-1, -1), int iterations = 1,
                  int borderType = BORDER_CONSTANT, const Scalar& borderValue = morphologyDefaultBorderValue(), Stream& s = Stream::Null())
{ B200CV_DST(dst, src, src.type()); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_morphology(&a, &b, B200CV_MORPH_ERODE, kernel, (size_t)ksize.width, ksize.width, ksize.height, anchor.x, anchor.y, iterations,
                          borderType, borderValue.val, s.cudaPtr()), "erode"); }
inline void dilate(const GpuMat& src, GpuMat& dst, const unsigned char* kernel, Size ksize, Point anchor = Point(-1, -1), int iterations = 1,
                   int borderType = BORDER_CONSTANT, const Scalar& borderValue = morphologyDefaultBorderValue(), Stream& s = Stream::Null())
{ B200CV_DST(dst, src, src.type()); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_morphology(&a, &b, B200CV_MORPH_DILATE, kernel, (size_t)ksize.width, ksize.width, ksize.height, anchor.x, anchor.y, iterations,
                          borderType, borderValue.val, s.cudaPtr()), "dilate"); }
// cv::integral (8UC1 -> 32SC1 sum of (rows+1) x (cols+1); optional 64FC1 sum of squares) and cv::cvtColorTwoPlane (NV12 / NV21, separate planes)
inline void integral(const GpuMat& src, GpuMat& sum, Stream& s = Stream::Null())
{ sum.create(src.rows + 1, src.cols + 1, makeType(B200CV_32S, 1), src.frames); b200cvMat a = src.desc(), b = sum.desc();
  check(b200cv_integral(&a, &b, nullptr, s.cudaPtr()), "integral"); }
inline void integral(const GpuMat& src, GpuMat& sum, GpuMat& sqsum, Stream& s = Stream::Null())
{ sum.create(src.rows + 1, src.cols + 1, makeType(B200CV_32S, 1), src.frames); sqsum.create(src.rows + 1, src.cols + 1, makeType(B200CV_64F, 1), src.frames);
  b200cvMat a = src.desc(), b = sum.desc(), q = sqsum.desc(); check(b200cv_integral(&a, &b, &q, s.cudaPtr()), "integral"); }
inline void cvtColorTwoPlane(const GpuMat& src1, const GpuMat& src2, GpuMat& dst, int code, Stream& s = Stream::Null())
{ dst.create(src1.rows, src1.cols, makeType(B200CV_8U, code >= 94 ? 4 : 3), src1.frames); b200cvMat y = src1.desc(), uv = src2.desc(), d = dst.desc();
  check(b200cv_cvt_color_two_plane(&y, &uv, &d, code, s.cudaPtr()), "cvtColorTwoPlane"); }
// cv::boxFilter / cv::blur (imgproc.hpp:1603, :1659)
inline void boxFilter(const GpuMat& src, GpuMat& dst, int ddepth, Size ksize, Point anchor = Point(-1, -1), bool normalize = true, int borderType = BORDER_DEFAULT,
                      Stream& s = Stream::Null())
{ B200CV_DST(dst, src, makeType(ddepth < 0 ? B200CV_DEPTH(src.type()) : ddepth, src.channels())); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_box_filter(&a, &b, ksize.width, ksize.height, anchor.x, anchor.y, normalize ? 1 : 0, borderType, s.cudaPtr()), "boxFilter"); }
inline void blur(const GpuMat& src, GpuMat& dst, Size ksize, Point anchor = Point(-1, -1), int borderType = BORDER_DEFAULT, Stream& s = Stream::Null())
{ boxFilter(src, dst, -1, ksize, anchor, true, borderType, s); }
inline void resize(const GpuMat& src, GpuMat& dst, Size dsize, double fx = 0, double fy = 0, int interpolation = INTER_LINEAR, Stream& s = Stream::Null())
{ if (dsize.width <= 0) dsize = Size((int)(src.cols * fx + 0.5), (int)(src.rows * fy + 0.5));
  dst.create(dsize.height, dsize.width, src.type(), src.frames); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_resize(&a, &b, interpolation, s.cudaPtr()), "resize"); }
inline void warpAffine(const GpuMat& src, GpuMat& dst, const double M[6], Size dsize, int flags = INTER_LINEAR, int borderMode = BORDER_CONSTANT, Scalar bv = Scalar(),
                       Stream& s = Stream::Null())
{ dst.create(dsize.height, dsize.width, src.type(), src.frames); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_warp_affine(&a, &b, M, flags, borderMode, bv.val, s.cudaPtr()), "warpAffine"); }
inline void warpPerspective(const GpuMat& src, GpuMat& dst, const double M[9], Size dsize, int flags = INTER_LINEAR, int borderMode = BORDER_CONSTANT, Scalar bv = Scalar(),
                            Stream& s = Stream::Null())
{ dst.create(dsize.height, dsize.width, src.type(), src.frames); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_warp_perspective(&a, &b, M, flags, borderMode, bv.val, s.cudaPtr()), "warpPerspective"); }
// cv::pyrDown / cv::pyrUp (imgproc.hpp:3325, :3351), default destination sizes
inline void pyrDown(const GpuMat& src, GpuMat& dst, int borderType = BORDER_DEFAULT, Stream& s = Stream::Null())
{ dst.create((src.rows + 1) / 2, (src.cols + 1) / 2, src.type(), src.frames); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_pyr_down(&a, &b, borderType, s.cudaPtr()), "pyrDown"); }
inline void pyrUp(const GpuMat& src, GpuMat& dst, Stream& s = Stream::Null())
{ dst.create(src.rows * 2, src.cols * 2, src.type(), src.frames); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_pyr_up(&a, &b, BORDER_DEFAULT, s.cudaPtr()), "pyrUp"); }
// cv::remap (imgproc.hpp:2531): map1/map2 as cv::remap takes them (CV_32FC1 pair, CV_32FC2, or CV_16SC2 + CV_16UC1); one set of maps per batch
inline void remap(const GpuMat& src, GpuMat& dst, const GpuMat& map1, const GpuMat& map2, int interpolation, int borderMode = BORDER_CONSTANT, Scalar bv = Scalar(),
                  Stream& s = Stream::Null())
{
    dst.create(map1.rows, map1.cols, src.type(), src.frames);
    b200cvMat a = src.desc(), b = dst.desc(), m1 = map1.desc(), m2 = map2.desc();
    check(b200cv_remap(&a, &b, &m1, map2.data ? &m2 : nullptr, interpolation, borderMode, bv.val, s.cudaPtr()), "remap");
}
// destination geometry of cv::cvtColor (color.cpp:323-372): the subsampled-YUV wire formats change the size, everything else keeps it
inline void cvtColorGeometry(int code, int cols, int rows, int dcn, int& w, int& h, int& cn)
{
    w = cols; h = rows; cn = dcn;
    if (code >= 90 && code <= 105) { h = rows * 2 / 3; cn = (code >= 94 && code <= 97) || code >= 102 ? 4 : 3; }
    else if (code == 106) { h = rows * 2 / 3; cn = 1; }
    else if (code >= 107 && code <= 122) cn = (code == 111 || code == 112 || code >= 119) ? 4 : 3;
    else if (code == 123 || code == 124) cn = 1;
    else if (code >= 127 && code <= 134) { h = rows * 3 / 2; cn = 1; }
    else if (code >= 143 && code <= 154) cn = 2;
    else if (code >= 139 && code <= 142) cn = 4;
    else if (code >= 86 && code <= 89) cn = 1;
    else if (cn <= 0) cn = (code == 0 || code == 2 || code == 5 || code == 9) ? 4 : (code == 6 || code == 7 || code == 10 || code == 11) ? 1 : 3;
}
inline void cvtColor(const GpuMat& src, GpuMat& dst, int code, int dcn = 0, Stream& s = Stream::Null())
{ int w, h, cn; cvtColorGeometry(code, src.cols, src.rows, dcn, w, h, cn);
  dst.create(h, w, makeType(B200CV_DEPTH(src.type()), cn), src.frames); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_cvt_color(&a, &b, code, s.cudaPtr()), "cvtColor"); }
inline void matchTemplate(const GpuMat& image, const GpuMat& templ, GpuMat& result, int method, Stream& s = Stream::Null())
{ result.create(image.rows - templ.rows + 1, image.cols - templ.cols + 1, makeType(CV_32F, 1), image.frames); b200cvMat a = image.desc(), t = templ.desc(), r = result.desc();
  check(b200cv_match_template(&a, &t, &r, method, s.cudaPtr()), "matchTemplate"); }
inline void cornerHarris(const GpuMat& src, GpuMat& dst, int blockSize, int ksize, double k, int borderType = BORDER_DEFAULT, Stream& s = Stream::Null())
{ B200CV_DST(dst, src, makeType(CV_32F, 1)); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_corner_harris(&a, &b, blockSize, ksize, k, borderType, s.cudaPtr()), "cornerHarris"); }
inline void cornerMinEigenVal(const GpuMat& src, GpuMat& dst, int blockSize, int ksize = 3, int borderType = BORDER_DEFAULT, Stream& s = Stream::Null())
{ B200CV_DST(dst, src, makeType(CV_32F, 1)); b200cvMat a = src.desc(), b = dst.desc(); check(b200cv_corner_min_eigen_val(&a, &b, blockSize, ksize, borderType, s.cudaPtr()), "cornerMinEigenVal"); }
// cv::Canny (imgproc.hpp:1889, :1907): 8-bit image -> 8UC1 edges; or 16S derivatives dx, dy -> 8UC1 edges
inline void Canny(const GpuMat& image, GpuMat& edges, double threshold1, double threshold2, int apertureSize = 3, bool L2gradient = false, Stream& s = Stream::Null())
{ B200CV_DST(edges, image, makeType(CV_8U, 1)); b200cvMat a = image.desc(), b = edges.desc();
  check(b200cv_canny(&a, &b, threshold1, threshold2, apertureSize, L2gradient ? 1 : 0, s.cudaPtr()), "Canny"); }
inline void Canny(const GpuMat& dx, const GpuMat& dy, GpuMat& edges, double threshold1, double threshold2, bool L2gradient = false, Stream& s = Stream::Null())
{ B200CV_DST(edges, dx, makeType(CV_8U, 1)); b200cvMat a = dx.desc(), b = dy.desc(), c = edges.desc();
  check(b200cv_canny_derivs(&a, &b, &c, threshold1, threshold2, L2gradient ? 1 : 0, s.cudaPtr()), "Canny"); }
// cv::distanceTransform(src, dst, distanceType, maskSize, dstType): 8UC1 -> 32FC1, or 8UC1 for DIST_L1 with dstType CV_8U (src == dst allowed)
inline void distanceTransform(const GpuMat& src, GpuMat& dst, int distanceType, int maskSize, int dstType = CV_32F, Stream& s = Stream::Null())
{ B200CV_DST(dst, src, makeType(distanceType == B200CV_DIST_L1 && dstType == CV_8U ? CV_8U : CV_32F, 1)); b200cvMat a = src.desc(), b = dst.desc();
  check(b200cv_distance_transform(&a, &b, distanceType, maskSize, s.cudaPtr()), "distanceTransform"); }
inline void goodFeaturesToTrack(const GpuMat& image, std::vector<Point2f>& corners, int maxCorners, double qualityLevel, double minDistance, int blockSize = 3,
                                int gradientSize = 3, bool useHarrisDetector = false, double k = 0.04, Stream& s = Stream::Null())
{ int cap = maxCorners > 0 ? maxCorners : image.rows * image.cols; std::vector<float> pts((size_t)2 * cap * image.frames); std::vector<int> cnt(image.frames);
  b200cvMat a = image.desc();
  check(b200cv_good_features_to_track(&a, pts.data(), nullptr, cap, cnt.data(), maxCorners, qualityLevel, minDistance, blockSize, gradientSize, useHarrisDetector, k, s.cudaPtr()), "goodFeaturesToTrack");
  corners.clear(); for (int i = 0; i < cnt[0] && i < cap; i++) corners.push_back(Point2f{pts[2 * i], pts[2 * i + 1]}); }

// ---- cv::cuda::Filter-shaped objects ---------------------------------------------------------------------------------------
class Filter {
public:
    virtual ~Filter() {}
    virtual void apply(const GpuMat& src, GpuMat& dst, Stream& stream = Stream::Null()) = 0;
};
typedef std::shared_ptr<Filter> FilterPtr;

inline FilterPtr createGaussianFilter(int srcType, int dstType, Size ksize, double sigma1, double sigma2 = 0, int rowBorderMode = BORDER_DEFAULT, int = -1)
{
    struct F : Filter { Size k; double s1, s2; int b;
        void apply(const GpuMat& src, GpuMat& dst, Stream& st) override { GaussianBlur(src, dst, k, s1, s2, b, st); } };
    (void)srcType; (void)dstType;
    auto f = std::make_shared<F>(); f->k = ksize; f->s1 = sigma1; f->s2 = sigma2; f->b = rowBorderMode; return f;
}
inline FilterPtr createSeparableLinearFilter(int srcType, int dstType, const std::vector<float>& rowKernel, const std::vector<float>& columnKernel, Point anchor = Point(),
                                             int rowBorderMode = BORDER_DEFAULT, int = -1)
{
    struct F : Filter { int dd; std::vector<float> kx, ky; Point a; int b;
        void apply(const GpuMat& src, GpuMat& dst, Stream& st) override { sepFilter2D(src, dst, dd, kx, ky, a, 0, b, st); } };
    (void)srcType;
    auto f = std::make_shared<F>(); f->dd = B200CV_DEPTH(dstType); f->kx = rowKernel; f->ky = columnKernel; f->a = anchor; f->b = rowBorderMode; return f;
}
inline FilterPtr createLinearFilter(int srcType, int dstType, const std::vector<float>& kernel, Size ksz, Point anchor = Point(), int borderMode = BORDER_DEFAULT)
{
    struct F : Filter { int dd; std::vector<float> k; Size sz; Point a; int b;
        void apply(const GpuMat& src, GpuMat& dst, Stream& st) override { filter2D(src, dst, dd, k.data(), sz, a, 0, b, st); } };
    (void)srcType;
    auto f = std::make_shared<F>(); f->dd = B200CV_DEPTH(dstType); f->k = kernel; f->sz = ksz; f->a = anchor; f->b = borderMode; return f;
}
inline FilterPtr createSobelFilter(int srcType, int dstType, int dx, int dy, int ksize = 3, double scale = 1, int rowBorderMode = BORDER_DEFAULT, int = -1)
{
    struct F : Filter { int dd, dx, dy, ks; double sc; int b;
        void apply(const GpuMat& src, GpuMat& dst, Stream& st) override { Sobel(src, dst, dd, dx, dy, ks, sc, 0, b, st); } };
    (void)srcType;
    auto f = std::make_shared<F>(); f->dd = B200CV_DEPTH(dstType); f->dx = dx; f->dy = dy; f->ks = ksize; f->sc = scale; f->b = rowBorderMode; return f;
}



}  // namespace b200cv

#ifdef B200CV_WITH_OPENCV
#include "b200cv_opencv.hpp"     // cv::InputArray / cv::OutputArray face (b200cv::cuda::*), DeviceMat, PinnedMat, DeviceAllocator
#endif
