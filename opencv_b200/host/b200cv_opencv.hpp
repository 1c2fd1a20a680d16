// b200cv_opencv.hpp -- the cv::-typed face of the hot path: the reference's own argument types (cv::InputArray / cv::OutputArray, cv::Size,
// cv::Scalar, cv::Point) with the cv::cuda operator surface (trailing Stream&, Filter objects), compiled against the REAL OpenCV headers
// (-I<opencv>/modules/core/include).  Included by b200cv.hpp under -DB200CV_WITH_OPENCV.
//
//   namespace b200cv::cuda   what a user of cv::cuda:: switches to (rename the namespace, keep the code): the reference signatures of
//       GaussianBlur / sepFilter2D / filter2D / Sobel / resize / warpAffine / warpPerspective / cvtColor / matchTemplate / cornerHarris /
//       cornerMinEigenVal / goodFeaturesToTrack / Canny / distanceTransform (imgproc.hpp:1544,1723,1702,1862,2422,2450,2482,3736,3916,1948,1921,2096,1889,1907) + Stream&, and
//       GFTTDetector (features2d/src/gftt.cpp), createGaussianFilter / createSeparableLinearFilter / createLinearFilter / createSobelFilter -> Ptr<Filter>, Filter::apply(InputArray,
//       OutputArray, Stream&) -- the usage of samples/cpp/tutorial_code/gpu/gpu-basics-similarity/gpu-basics-similarity.cpp:392-404.
//   Array kinds accepted (core/include/opencv2/core/mat.hpp:163-188):
//       CUDA_GPU_MAT   cv::cuda::GpuMat (fields read directly: data, step, rows, cols, flags) -> device path, asynchronous on the Stream
//       MAT, MATX, STD_VECTOR, ...  host memory -> host path (b200cv_host_*: upload, kernel, download; synchronous)
//       CUDA_HOST_MEM  cv::cuda::HostMem (page-locked host memory) -> host path at full PCIe speed
//   DeviceMat  IS-A cv::cuda::GpuMat that owns a b200cv allocation (create / upload / download / release work in an OpenCV build WITHOUT CUDA,
//              where cv::cuda::GpuMat::create throws, core/src/cuda_gpu_mat.cpp:428-434); binds to InputArray / OutputArray as CUDA_GPU_MAT.
//   PinnedMat  IS-A cv::cuda::HostMem over b200cv_host_alloc.
//   DeviceAllocator  cv::cuda::GpuMat::Allocator {allocate, free} (cuda.hpp:108-115) over the b200cv runtime: in a CUDA-enabled OpenCV build
//              cv::cuda::GpuMat::setDefaultAllocator(&b200cv::deviceAllocator()) makes every plain GpuMat use it.
//   Output GpuMats of the wrong size / type are (re)allocated by the library, as cv::cuda functions do (getOutputMat, cuda_gpu_mat.cpp:367-391);
//   the allocation belongs to a registry keyed by the data pointer and is released when that GpuMat is re-created or by releaseOutputs().
//   b200cv::Stream has the method set of cv::cuda::Stream (cuda.hpp:909-975); the reference's own Stream needs HAVE_CUDA -- with it,
//   b200cv::Stream(cv_stream.cudaPtr()) wraps one.
#pragma once
#include <mutex>
#include <unordered_map>
#include <opencv2/core.hpp>
#include <opencv2/core/cuda.hpp>
#include <opencv2/imgproc.hpp>       // the cv:: enums (interpolation, border, colour codes) the signatures default to

namespace b200cv {

// ---- cv::cuda::GpuMat::Allocator over the b200cv runtime -----------------------------------------------------------------------------------
class DeviceAllocator : public cv::cuda::GpuMat::Allocator {
public:
    bool allocate(cv::cuda::GpuMat* mat, int rows, int cols, size_t elemSize) override
    {
        void* p = nullptr; size_t step = 0;
        if (b200cv_malloc_pitch(&p, &step, (size_t)cols * elemSize, (size_t)rows) != B200CV_OK) return false;
        mat->data = (uchar*)p; mat->step = step; mat->refcount = new int(1);
        return true;
    }
    void free(cv::cuda::GpuMat* mat) override
    {
        b200cv_free(mat->datastart ? mat->datastart : mat->data);
        delete mat->refcount;
    }
};
inline DeviceAllocator& deviceAllocator() { static DeviceAllocator a; return a; }

// ---- device matrix: a cv::cuda::GpuMat header over memory this object owns --------------------------------------------------------------------
class DeviceMat : public cv::cuda::GpuMat {
public:
    DeviceMat() : cv::cuda::GpuMat((cv::cuda::GpuMat::Allocator*)nullptr) {}
    DeviceMat(int r, int c, int t) : cv::cuda::GpuMat((cv::cuda::GpuMat::Allocator*)nullptr) { create(r, c, t); }
    DeviceMat(cv::Size s, int t) : cv::cuda::GpuMat((cv::cuda::GpuMat::Allocator*)nullptr) { create(s.height, s.width, t); }
    void create(int r, int c, int t)
    {
        t &= cv::Mat::TYPE_MASK;
        if (data && r == rows && c == cols && t == type()) return;
        release();
        void* p = nullptr; size_t stp = 0;
        check(b200cv_malloc_pitch(&p, &stp, (size_t)c * CV_ELEM_SIZE(t), (size_t)r), "DeviceMat::create");
        own_.reset(p, [](void* q) { b200cv_free(q); });
        static_cast<cv::cuda::GpuMat&>(*this) = cv::cuda::GpuMat(r, c, t, p, stp);          // the reference's wrapping constructor (cuda_gpu_mat.cpp:56-78)
    }
    void create(cv::Size s, int t) { create(s.height, s.width, t); }
    void release() { own_.reset(); static_cast<cv::cuda::GpuMat&>(*this) = cv::cuda::GpuMat((cv::cuda::GpuMat::Allocator*)nullptr); }
    void upload(cv::InputArray arr, Stream& s = Stream::Null())
    {
        cv::Mat m = arr.getMat();
        create(m.rows, m.cols, m.type());
        check(b200cv_upload(m.data, m.step, data, step, (size_t)m.cols * m.elemSize(), (size_t)m.rows, s.cudaPtr()), "DeviceMat::upload");
        if (!s.cudaPtr()) b200cv_stream_synchronize(nullptr);
    }
    void download(cv::OutputArray dst, Stream& s = Stream::Null()) const
    {
        dst.create(rows, cols, type());
        cv::Mat m = dst.getMat();
        check(b200cv_download(data, step, m.data, m.step, (size_t)cols * elemSize(), (size_t)rows, s.cudaPtr()), "DeviceMat::download");
        if (!s.cudaPtr()) b200cv_stream_synchronize(nullptr);
    }
private:
    std::shared_ptr<void> own_;
};

// ---- page-locked host matrix: a cv::cuda::HostMem header over b200cv_host_alloc ---------------------------------------------------------------
class PinnedMat : public cv::cuda::HostMem {
public:
    PinnedMat(int r, int c, int t) : cv::cuda::HostMem(cv::cuda::HostMem::PAGE_LOCKED)
    {
        t &= cv::Mat::TYPE_MASK;
        void* p = nullptr;
        const size_t stp = (size_t)c * CV_ELEM_SIZE(t);
        check(b200cv_host_alloc(&p, stp * r), "PinnedMat");
        own_.reset(p, [](void* q) { b200cv_host_free(q); });
        flags = cv::Mat::MAGIC_VAL + t + cv::Mat::CONTINUOUS_FLAG; rows = r; cols = c; step = stp;
        data = datastart = (uchar*)p; dataend = data + stp * r; refcount = nullptr;
    }
    cv::Mat mat() const { return cv::Mat(rows, cols, type(), data, step); }     // HostMem::createMatHeader (cuda.hpp:845)
private:
    std::shared_ptr<void> own_;
};

namespace cuda {

using b200cv::Stream;
using b200cv::Event;

// ---- InputArray / OutputArray -> b200cvMat ------------------------------------------------------------------------------------------------------
struct Arr { b200cvMat m; bool device; cv::Mat keep; };

inline Arr input(cv::InputArray a, const char* what)
{
    Arr r = {};
    const int k = a.kind();
    if (k == cv::_InputArray::CUDA_GPU_MAT) {
        const cv::cuda::GpuMat* g = (const cv::cuda::GpuMat*)a.getObj();
        if (!g || !g->data) throw Error(B200CV_ERR_BAD_ARG, std::string(what) + ": empty GpuMat");
        r.m = b200cvMat{g->data, g->step, g->cols, g->rows, g->type(), 1, 0};
        r.device = true;
    } else if (k == cv::_InputArray::CUDA_HOST_MEM) {
        const cv::cuda::HostMem* h = (const cv::cuda::HostMem*)a.getObj();
        if (!h || !h->data) throw Error(B200CV_ERR_BAD_ARG, std::string(what) + ": empty HostMem");
        r.m = b200cvMat{h->data, h->step, h->cols, h->rows, h->type(), 1, 0};
    } else if (k == cv::_InputArray::UMAT || k == cv::_InputArray::OPENGL_BUFFER) {
        throw NotImplemented(B200CV_NOT_IMPLEMENTED, std::string(what) + ": UMat / OpenGL arrays are not on the device path");
    } else {
        r.keep = a.getMat();
        if (r.keep.empty() || r.keep.dims > 2) throw Error(B200CV_ERR_BAD_ARG, std::string(what) + ": empty or n-dimensional array");
        r.m = b200cvMat{r.keep.data, r.keep.step, r.keep.cols, r.keep.rows, r.keep.type(), 1, 0};
    }
    return r;
}

// allocations made for output GpuMats (see the header comment)
struct OutputRegistry {
    std::mutex m;
    std::unordered_map<void*, std::shared_ptr<void>> owned;
    static OutputRegistry& get() { static OutputRegistry r; return r; }
};
inline void releaseOutputs() { std::lock_guard<std::mutex> g(OutputRegistry::get().m); OutputRegistry::get().owned.clear(); }

inline Arr output(cv::OutputArray d, int rows, int cols, int type, bool device, const char* what)
{
    Arr r = {};
    const int k = d.kind();
    type &= cv::Mat::TYPE_MASK;
    if (device) {
        if (k != cv::_InputArray::CUDA_GPU_MAT) throw Error(B200CV_ERR_BAD_ARG, std::string(what) + ": device source needs a cv::cuda::GpuMat destination");
        cv::cuda::GpuMat* g = (cv::cuda::GpuMat*)d.getObj();
        if (!g->data || g->rows != rows || g->cols != cols || g->type() != type) {
            OutputRegistry& reg = OutputRegistry::get();
            void* p = nullptr; size_t stp = 0;
            check(b200cv_malloc_pitch(&p, &stp, (size_t)cols * CV_ELEM_SIZE(type), (size_t)rows), what);
            std::lock_guard<std::mutex> lk(reg.m);
            if (g->data) reg.owned.erase(g->data);                       // this GpuMat's previous output buffer, if it was ours
            reg.owned[p] = std::shared_ptr<void>(p, [](void* q) { b200cv_free(q); });
            *g = cv::cuda::GpuMat(rows, cols, type, p, stp);
        }
        r.m = b200cvMat{g->data, g->step, g->cols, g->rows, g->type(), 1, 0};
        r.device = true;
    } else if (k == cv::_InputArray::CUDA_HOST_MEM) {
        cv::cuda::HostMem* h = (cv::cuda::HostMem*)d.getObj();
        if (!h->data || h->rows != rows || h->cols != cols || h->type() != type)
            throw Error(B200CV_ERR_BAD_ARG, std::string(what) + ": a HostMem destination must be allocated with the result's size and type");
        r.m = b200cvMat{h->data, h->step, h->cols, h->rows, h->type(), 1, 0};
    } else if (k == cv::_InputArray::CUDA_GPU_MAT) {
        throw Error(B200CV_ERR_BAD_ARG, std::string(what) + ": host source with a GpuMat destination (upload first: DeviceMat::upload)");
    } else {
        d.create(rows, cols, type);
        r.keep = d.getMat();
        r.m = b200cvMat{r.keep.data, r.keep.step, r.keep.cols, r.keep.rows, r.keep.type(), 1, 0};
    }
    return r;
}

inline std::vector<float> floatTaps(cv::InputArray k)
{
    cv::Mat m = k.getMat(), f;
    m.convertTo(f, CV_32F);
    f = f.isContinuous() ? f : f.clone();
    return std::vector<float>((const float*)f.datastart, (const float*)f.datastart + f.total());
}
inline int dstType(int ddepth, int srcType) { return CV_MAKETYPE(ddepth < 0 ? CV_MAT_DEPTH(srcType) : ddepth, CV_MAT_CN(srcType)); }
inline void hostSync(const Arr& a, Stream& s) { (void)a; (void)s; }

// ---- the reference signatures + Stream& -------------------------------------------------------------------------------------------------------
inline void GaussianBlur(cv::InputArray src, cv::OutputArray dst, cv::Size ksize, double sigmaX, double sigmaY = 0, int borderType = cv::BORDER_DEFAULT, Stream& s = Stream::Null())
{
    Arr a = input(src, "GaussianBlur"), b = output(dst, a.m.rows, a.m.cols, a.m.type, a.device, "GaussianBlur");
    check(a.device ? b200cv_gaussian_blur(&a.m, &b.m, ksize.width, ksize.height, sigmaX, sigmaY, borderType, s.cudaPtr())
                   : b200cv_host_gaussian_blur(&a.m, &b.m, ksize.width, ksize.height, sigmaX, sigmaY, borderType), "GaussianBlur");
}
inline void sepFilter2D(cv::InputArray src, cv::OutputArray dst, int ddepth, cv::InputArray kernelX, cv::InputArray kernelY, cv::Point anchor = cv::Point(-1, -1), double delta = 0,
                        int borderType = cv::BORDER_DEFAULT, Stream& s = Stream::Null())
{
    Arr a = input(src, "sepFilter2D"), b = output(dst, a.m.rows, a.m.cols, dstType(ddepth, a.m.type), a.device, "sepFilter2D");
    const std::vector<float> kx = floatTaps(kernelX), ky = floatTaps(kernelY);
    check(a.device ? b200cv_sep_filter2d(&a.m, &b.m, kx.data(), (int)kx.size(), ky.data(), (int)ky.size(), anchor.x, anchor.y, delta, borderType, s.cudaPtr())
                   : b200cv_host_sep_filter2d(&a.m, &b.m, kx.data(), (int)kx.size(), ky.data(), (int)ky.size(), anchor.x, anchor.y, delta, borderType), "sepFilter2D");
}
inline void filter2D(cv::InputArray src, cv::OutputArray dst, int ddepth, cv::InputArray kernel, cv::Point anchor = cv::Point(-1, -1), double delta = 0,
                     int borderType = cv::BORDER_DEFAULT, Stream& s = Stream::Null())
{
    Arr a = input(src, "filter2D"), b = output(dst, a.m.rows, a.m.cols, dstType(ddepth, a.m.type), a.device, "filter2D");
    const cv::Size ks = kernel.size();
    const std::vector<float> k = floatTaps(kernel);
    check(a.device ? b200cv_filter2d(&a.m, &b.m, k.data(), ks.width, ks.height, anchor.x, anchor.y, delta, borderType, s.cudaPtr())
                   : b200cv_host_filter2d(&a.m, &b.m, k.data(), ks.width, ks.height, anchor.x, anchor.y, delta, borderType), "filter2D");
}
inline void Sobel(cv::InputArray src, cv::OutputArray dst, int ddepth, int dx, int dy, int ksize = 3, double scale = 1, double delta = 0, int borderType = cv::BORDER_DEFAULT,
                  Stream& s = Stream::Null())
{
    Arr a = input(src, "Sobel"), b = output(dst, a.m.rows, a.m.cols, dstType(ddepth, a.m.type), a.device, "Sobel");
    check(a.device ? b200cv_sobel(&a.m, &b.m, dx, dy, ksize, scale, delta, borderType, s.cudaPtr()) : b200cv_host_sobel(&a.m, &b.m, dx, dy, ksize, scale, delta, borderType), "Sobel");
}
// cv::Laplacian: a stock OpenCV built with the HAL already sends ksize 1 / 3 here through filter2D; ksize 5..31 only through this call
inline void Laplacian(cv::InputArray src, cv::OutputArray dst, int ddepth, int ksize = 1, double scale = 1, double delta = 0, int borderType = cv::BORDER_DEFAULT,
                      Stream& s = Stream::Null())
{
    Arr a = input(src, "Laplacian"), b = output(dst, a.m.rows, a.m.cols, dstType(ddepth, a.m.type), a.device, "Laplacian");
    check(a.device ? b200cv_laplacian(&a.m, &b.m, ksize, scale, delta, borderType, s.cudaPtr()) : b200cv_host_laplacian(&a.m, &b.m, ksize, scale, delta, borderType),
          "Laplacian");
}
// cv::erode / cv::dilate / cv::morphologyEx (MORPH_ERODE .. MORPH_BLACKHAT): no cv_hal_morph hook is registered (INTEGRATION.md), so a
// stock OpenCV keeps its own morphology; call these instead.  kernel: any 8-bit single-channel mask, or empty.
inline void morphology_(int op, cv::InputArray src, cv::OutputArray dst, cv::InputArray kernel, cv::Point anchor, int iterations, int borderType,
                        const cv::Scalar& borderValue, Stream& s, const char* what)
{
    Arr a = input(src, what), b = output(dst, a.m.rows, a.m.cols, a.m.type, a.device, what);
    cv::Mat k = kernel.getMat();
    if (!k.empty()) { CV_Assert(k.type() == CV_8UC1); k = k.isContinuous() ? k : k.clone(); }
    const unsigned char* kp = k.empty() ? nullptr : k.ptr();
    const size_t kstep = k.empty() ? 0 : k.step[0];
    check(a.device ? b200cv_morphology(&a.m, &b.m, op, kp, kstep, k.cols, k.rows, anchor.x, anchor.y, iterations, borderType, borderValue.val, s.cudaPtr())
                   : b200cv_host_morphology(&a.m, &b.m, op, kp, kstep, k.cols, k.rows, anchor.x, anchor.y, iterations, borderType, borderValue.val),
          what);
}
inline void erode(cv::InputArray src, cv::OutputArray dst, cv::InputArray kernel, cv::Point anchor = cv::Point(-1, -1), int iterations = 1,
                  int borderType = cv::BORDER_CONSTANT, const cv::Scalar& borderValue = cv::morphologyDefaultBorderValue(), Stream& s = Stream::Null())
{ morphology_(cv::MORPH_ERODE, src, dst, kernel, anchor, iterations, borderType, borderValue, s, "erode"); }
inline void dilate(cv::InputArray src, cv::OutputArray dst, cv::InputArray kernel, cv::Point anchor = cv::Point(-1, -1), int iterations = 1,
                   int borderType = cv::BORDER_CONSTANT, const cv::Scalar& borderValue = cv::morphologyDefaultBorderValue(), Stream& s = Stream::Null())
{ morphology_(cv::MORPH_DILATE, src, dst, kernel, anchor, iterations, borderType, borderValue, s, "dilate"); }
inline void morphologyEx(cv::InputArray src, cv::OutputArray dst, int op, cv::InputArray kernel, cv::Point anchor = cv::Point(-1, -1), int iterations = 1,
                         int borderType = cv::BORDER_CONSTANT, const cv::Scalar& borderValue = cv::morphologyDefaultBorderValue(), Stream& s = Stream::Null())
{
    cv::Mat k = kernel.getMat();
    if (k.empty()) k = cv::getStructuringElement(cv::MORPH_RECT, cv::Size(3, 3));
    morphology_(op, src, dst, k, anchor, iterations, borderType, borderValue, s, "morphologyEx");
}
inline void resize(cv::InputArray src, cv::OutputArray dst, cv::Size dsize, double fx = 0, double fy = 0, int interpolation = cv::INTER_LINEAR, Stream& s = Stream::Null())
{
    Arr a = input(src, "resize");
    const bool by_factor = dsize.width <= 0 || dsize.height <= 0;
    if (by_factor) dsize = cv::Size(cv::saturate_cast<int>(a.m.cols * fx), cv::saturate_cast<int>(a.m.rows * fy));      // resize.cpp:4214-4228
    else fx = fy = 0;
    Arr b = output(dst, dsize.height, dsize.width, a.m.type, a.device, "resize");
    check(a.device ? b200cv_resize_scaled(&a.m, &b.m, interpolation, fx, fy, s.cudaPtr()) : b200cv_host_resize_scaled(&a.m, &b.m, interpolation, fx, fy), "resize");
}
inline void warpAffine(cv::InputArray src, cv::OutputArray dst, cv::InputArray M, cv::Size dsize, int flags = cv::INTER_LINEAR, int borderMode = cv::BORDER_CONSTANT,
                       const cv::Scalar& borderValue = cv::Scalar(), Stream& s = Stream::Null())
{
    Arr a = input(src, "warpAffine"), b = output(dst, dsize.height, dsize.width, a.m.type, a.device, "warpAffine");
    cv::Mat m; M.getMat().convertTo(m, CV_64F);
    if (m.total() != 6) throw Error(B200CV_ERR_BAD_ARG, "warpAffine: M must be 2x3");
    m = m.isContinuous() ? m : m.clone();
    check(a.device ? b200cv_warp_affine(&a.m, &b.m, m.ptr<double>(), flags, borderMode, borderValue.val, s.cudaPtr())
                   : b200cv_host_warp_affine(&a.m, &b.m, m.ptr<double>(), flags, borderMode, borderValue.val), "warpAffine");
}
inline void warpPerspective(cv::InputArray src, cv::OutputArray dst, cv::InputArray M, cv::Size dsize, int flags = cv::INTER_LINEAR, int borderMode = cv::BORDER_CONSTANT,
                            const cv::Scalar& borderValue = cv::Scalar(), Stream& s = Stream::Null())
{
    Arr a = input(src, "warpPerspective"), b = output(dst, dsize.height, dsize.width, a.m.type, a.device, "warpPerspective");
    cv::Mat m; M.getMat().convertTo(m, CV_64F);
    if (m.total() != 9) throw Error(B200CV_ERR_BAD_ARG, "warpPerspective: M must be 3x3");
    m = m.isContinuous() ? m : m.clone();
    check(a.device ? b200cv_warp_perspective(&a.m, &b.m, m.ptr<double>(), flags, borderMode, borderValue.val, s.cudaPtr())
                   : b200cv_host_warp_perspective(&a.m, &b.m, m.ptr<double>(), flags, borderMode, borderValue.val), "warpPerspective");
}
inline void cvtColor(cv::InputArray src, cv::OutputArray dst, int code, int dstCn = 0, Stream& s = Stream::Null())
{
    Arr a = input(src, "cvtColor");
    int w, h, cn; cvtColorGeometry(code, a.m.cols, a.m.rows, dstCn, w, h, cn);
    Arr b = output(dst, h, w, CV_MAKETYPE(CV_MAT_DEPTH(a.m.type), cn), a.device, "cvtColor");
    check(a.device ? b200cv_cvt_color(&a.m, &b.m, code, s.cudaPtr()) : b200cv_host_cvt_color(&a.m, &b.m, code), "cvtColor");
}
inline void matchTemplate(cv::InputArray image, cv::InputArray templ, cv::OutputArray result, int method, Stream& s = Stream::Null())
{
    Arr a = input(image, "matchTemplate"), t = input(templ, "matchTemplate templ");
    if (a.device != t.device) throw Error(B200CV_ERR_BAD_ARG, "matchTemplate: image and templ must live on the same side");
    Arr r = output(result, a.m.rows - t.m.rows + 1, a.m.cols - t.m.cols + 1, CV_32FC1, a.device, "matchTemplate");
    check(a.device ? b200cv_match_template(&a.m, &t.m, &r.m, method, s.cudaPtr()) : b200cv_host_match_template(&a.m, &t.m, &r.m, method), "matchTemplate");
}
inline void cornerHarris(cv::InputArray src, cv::OutputArray dst, int blockSize, int ksize, double k, int borderType = cv::BORDER_DEFAULT, Stream& s = Stream::Null())
{
    Arr a = input(src, "cornerHarris"), b = output(dst, a.m.rows, a.m.cols, CV_32FC1, a.device, "cornerHarris");
    check(a.device ? b200cv_corner_harris(&a.m, &b.m, blockSize, ksize, k, borderType, s.cudaPtr()) : b200cv_host_corner_harris(&a.m, &b.m, blockSize, ksize, k, borderType), "cornerHarris");
}
inline void Canny(cv::InputArray image, cv::OutputArray edges, double threshold1, double threshold2, int apertureSize = 3, bool L2gradient = false,
                  Stream& s = Stream::Null())
{
    Arr a = input(image, "Canny"), b = output(edges, a.m.rows, a.m.cols, CV_8UC1, a.device, "Canny");
    const int l2 = L2gradient ? 1 : 0;
    check(a.device ? b200cv_canny(&a.m, &b.m, threshold1, threshold2, apertureSize, l2, s.cudaPtr())
                   : b200cv_host_canny(&a.m, &b.m, threshold1, threshold2, apertureSize, l2), "Canny");
}
// cv::distanceTransform(src, dst, distanceType, maskSize, dstType): the reference has no HAL hook for it, so a stock cv::distanceTransform
// never reaches the library; call this instead.  8UC1 for DIST_L1 with dstType CV_8U (in place allowed), 32FC1 otherwise.
inline void distanceTransform(cv::InputArray src, cv::OutputArray dst, int distanceType, int maskSize, int dstType = CV_32F, Stream& s = Stream::Null())
{
    Arr a = input(src, "distanceTransform");
    const int t = distanceType == cv::DIST_L1 && dstType == CV_8U ? CV_8UC1 : CV_32FC1;
    Arr b = output(dst, a.m.rows, a.m.cols, t, a.device, "distanceTransform");
    check(a.device ? b200cv_distance_transform(&a.m, &b.m, distanceType, maskSize, s.cudaPtr())
                   : b200cv_host_distance_transform(&a.m, &b.m, distanceType, maskSize), "distanceTransform");
}
// host derivatives are uploaded, the edges downloaded (there is no batched host path for this overload)
inline void Canny(cv::InputArray dx, cv::InputArray dy, cv::OutputArray edges, double threshold1, double threshold2, bool L2gradient = false,
                  Stream& s = Stream::Null())
{
    Arr a = input(dx, "Canny dx"), b = input(dy, "Canny dy");
    if (a.device != b.device) throw Error(B200CV_ERR_BAD_ARG, "Canny: dx and dy must live on the same side");
    const int l2 = L2gradient ? 1 : 0;
    if (a.device) {
        Arr e = output(edges, a.m.rows, a.m.cols, CV_8UC1, true, "Canny");
        check(b200cv_canny_derivs(&a.m, &b.m, &e.m, threshold1, threshold2, l2, s.cudaPtr()), "Canny");
        return;
    }
    DeviceMat ux, uy, ue(a.m.rows, a.m.cols, CV_8UC1);
    ux.upload(dx, s); uy.upload(dy, s);
    Arr da = input(ux, "Canny dx"), db = input(uy, "Canny dy"), de = input(ue, "Canny edges");
    check(b200cv_canny_derivs(&da.m, &db.m, &de.m, threshold1, threshold2, l2, s.cudaPtr()), "Canny");
    ue.download(edges, s);
}
inline void cornerMinEigenVal(cv::InputArray src, cv::OutputArray dst, int blockSize, int ksize = 3, int borderType = cv::BORDER_DEFAULT, Stream& s = Stream::Null())
{
    Arr a = input(src, "cornerMinEigenVal"), b = output(dst, a.m.rows, a.m.cols, CV_32FC1, a.device, "cornerMinEigenVal");
    check(a.device ? b200cv_corner_min_eigen_val(&a.m, &b.m, blockSize, ksize, borderType, s.cudaPtr()) : b200cv_host_corner_min_eigen_val(&a.m, &b.m, blockSize, ksize, borderType),
          "cornerMinEigenVal");
}
// corners: std::vector<cv::Point2f> or a Mat (N x 1 CV_32FC2), as cv::goodFeaturesToTrack writes it (featureselect.cpp:382-548).  The image is a GpuMat
// (a host image is uploaded first); the corner list comes back to the host.
inline void goodFeaturesToTrack(cv::InputArray image, cv::OutputArray corners, int maxCorners, double qualityLevel, double minDistance, cv::InputArray mask = cv::noArray(),
                                int blockSize = 3, bool useHarrisDetector = false, double k = 0.04, Stream& s = Stream::Null())
{
    if (!mask.empty()) throw NotImplemented(B200CV_NOT_IMPLEMENTED, "goodFeaturesToTrack: mask");
    Arr a = input(image, "goodFeaturesToTrack");
    DeviceMat up;
    if (!a.device) { up.upload(image, s); a = input(up, "goodFeaturesToTrack"); }
    const int cap = maxCorners > 0 ? maxCorners : a.m.rows * a.m.cols;
    std::vector<float> pts((size_t)2 * cap);
    int cnt = 0;
    check(b200cv_good_features_to_track(&a.m, pts.data(), nullptr, cap, &cnt, maxCorners, qualityLevel, minDistance, blockSize, 3, useHarrisDetector ? 1 : 0, k, s.cudaPtr()),
          "goodFeaturesToTrack");
    cnt = std::min(cnt, cap);
    cv::Mat(cnt, 1, CV_32FC2, pts.data()).copyTo(corners);
}

// ---- cv::cuda::Filter ----------------------------------------------------------------------------------------------------------------------------
class Filter : public cv::Algorithm {
public:
    virtual void apply(cv::InputArray src, cv::OutputArray dst, Stream& stream = Stream::Null()) = 0;
};

inline cv::Ptr<Filter> createGaussianFilter(int srcType, int dstType, cv::Size ksize, double sigma1, double sigma2 = 0, int rowBorderMode = cv::BORDER_DEFAULT, int columnBorderMode = -1)
{
    struct F : Filter { cv::Size k; double s1, s2; int b;
        void apply(cv::InputArray src, cv::OutputArray dst, Stream& st) override { b200cv::cuda::GaussianBlur(src, dst, k, s1, s2, b, st); } };
    if (dstType >= 0 && CV_MAT_DEPTH(dstType) != CV_MAT_DEPTH(srcType)) throw NotImplemented(B200CV_NOT_IMPLEMENTED, "createGaussianFilter: dstType != srcType");
    if (columnBorderMode >= 0 && columnBorderMode != rowBorderMode) throw NotImplemented(B200CV_NOT_IMPLEMENTED, "createGaussianFilter: different row / column borders");
    cv::Ptr<F> f = cv::makePtr<F>(); f->k = ksize; f->s1 = sigma1; f->s2 = sigma2; f->b = rowBorderMode; return f;
}
inline cv::Ptr<Filter> createSeparableLinearFilter(int srcType, int dstType, cv::InputArray rowKernel, cv::InputArray columnKernel, cv::Point anchor = cv::Point(-1, -1),
                                                   int rowBorderMode = cv::BORDER_DEFAULT, int columnBorderMode = -1)
{
    struct F : Filter { int dd; cv::Mat kx, ky; cv::Point a; int b;
        void apply(cv::InputArray src, cv::OutputArray dst, Stream& st) override { b200cv::cuda::sepFilter2D(src, dst, dd, kx, ky, a, 0, b, st); } };
    (void)srcType;
    if (columnBorderMode >= 0 && columnBorderMode != rowBorderMode) throw NotImplemented(B200CV_NOT_IMPLEMENTED, "createSeparableLinearFilter: different row / column borders");
    cv::Ptr<F> f = cv::makePtr<F>(); f->dd = dstType < 0 ? -1 : CV_MAT_DEPTH(dstType); f->kx = rowKernel.getMat().clone(); f->ky = columnKernel.getMat().clone(); f->a = anchor; f->b = rowBorderMode;
    return f;
}
inline cv::Ptr<Filter> createLinearFilter(int srcType, int dstType, cv::InputArray kernel, cv::Point anchor = cv::Point(-1, -1), int borderMode = cv::BORDER_DEFAULT,
                                          cv::Scalar borderVal = cv::Scalar::all(0))
{
    struct F : Filter { int dd; cv::Mat k; cv::Point a; int b;
        void apply(cv::InputArray src, cv::OutputArray dst, Stream& st) override { b200cv::cuda::filter2D(src, dst, dd, k, a, 0, b, st); } };
    (void)srcType; (void)borderVal;
    cv::Ptr<F> f = cv::makePtr<F>(); f->dd = dstType < 0 ? -1 : CV_MAT_DEPTH(dstType); f->k = kernel.getMat().clone(); f->a = anchor; f->b = borderMode; return f;
}
inline cv::Ptr<Filter> createSobelFilter(int srcType, int dstType, int dx, int dy, int ksize = 3, double scale = 1, int rowBorderMode = cv::BORDER_DEFAULT, int columnBorderMode = -1)
{
    struct F : Filter { int dd, dx, dy, ks; double sc; int b;
        void apply(cv::InputArray src, cv::OutputArray dst, Stream& st) override { b200cv::cuda::Sobel(src, dst, dd, dx, dy, ks, sc, 0, b, st); } };
    (void)srcType; (void)columnBorderMode;
    cv::Ptr<F> f = cv::makePtr<F>(); f->dd = dstType < 0 ? -1 : CV_MAT_DEPTH(dstType); f->dx = dx; f->dy = dy; f->ks = ksize; f->sc = scale; f->b = rowBorderMode; return f;
}

// ---- cv::GFTTDetector (features2d/include/opencv2/features2d.hpp; features2d/src/gftt.cpp:33-176): the Feature2D face of goodFeaturesToTrack ------
// create(...) with the reference's two argument lists, the set / get pairs, detect(image, keypoints, mask): colour images go through BGR2GRAY first,
// keypoints[i] = KeyPoint(corner, (float)blockSize, -1, quality) (gftt.cpp:131-151).  The image may be a cv::Mat or a cv::cuda::GpuMat.
class GFTTDetector : public cv::Algorithm {
public:
    static cv::Ptr<GFTTDetector> create(int maxCorners = 1000, double qualityLevel = 0.01, double minDistance = 1, int blockSize = 3, bool useHarrisDetector = false, double k = 0.04)
    { return create(maxCorners, qualityLevel, minDistance, blockSize, 3, useHarrisDetector, k); }
    static cv::Ptr<GFTTDetector> create(int maxCorners, double qualityLevel, double minDistance, int blockSize, int gradiantSize, bool useHarrisDetector = false, double k = 0.04)
    {
        cv::Ptr<GFTTDetector> d = cv::makePtr<GFTTDetector>();
        d->nfeatures = maxCorners; d->qualityLevel = qualityLevel; d->minDistance = minDistance; d->blockSize = blockSize; d->gradSize = gradiantSize;
        d->useHarrisDetector = useHarrisDetector; d->k = k;
        return d;
    }
    void setMaxFeatures(int v) { nfeatures = v; }            int getMaxFeatures() const { return nfeatures; }
    void setQualityLevel(double v) { qualityLevel = v; }     double getQualityLevel() const { return qualityLevel; }
    void setMinDistance(double v) { minDistance = v; }       double getMinDistance() const { return minDistance; }
    void setBlockSize(int v) { blockSize = v; }              int getBlockSize() const { return blockSize; }
    void setGradientSize(int v) { gradSize = v; }            int getGradientSize() { return gradSize; }
    void setHarrisDetector(bool v) { useHarrisDetector = v; } bool getHarrisDetector() const { return useHarrisDetector; }
    void setK(double v) { k = v; }                           double getK() const { return k; }
    cv::String getDefaultName() const override { return "Feature2D.GFTTDetector"; }

    void detect(cv::InputArray image, std::vector<cv::KeyPoint>& keypoints, cv::InputArray mask = cv::noArray(), Stream& s = Stream::Null())
    {
        keypoints.clear();
        if (image.empty()) return;
        if (!mask.empty()) throw NotImplemented(B200CV_NOT_IMPLEMENTED, "GFTTDetector::detect: mask");
        Arr a = input(image, "GFTTDetector::detect");
        DeviceMat up, gray;
        if (!a.device) { up.upload(image, s); a = input(up, "GFTTDetector::detect"); }
        if (a.m.type != CV_8UC1) {                      // gftt.cpp:138-140
            b200cv::cuda::cvtColor(a.device && up.empty() ? image : cv::InputArray(up), gray, cv::COLOR_BGR2GRAY, 0, s);
            a = input(gray, "GFTTDetector::detect");
        }
        const int cap = nfeatures > 0 ? nfeatures : a.m.rows * a.m.cols;
        std::vector<float> pts((size_t)2 * cap), q((size_t)cap);
        int cnt = 0;
        check(b200cv_good_features_to_track(&a.m, pts.data(), q.data(), cap, &cnt, nfeatures, qualityLevel, minDistance, blockSize, gradSize, useHarrisDetector ? 1 : 0, k, s.cudaPtr()),
              "GFTTDetector::detect");
        cnt = std::min(cnt, cap);
        keypoints.resize(cnt);
        for (int i = 0; i < cnt; i++) keypoints[i] = cv::KeyPoint(cv::Point2f(pts[2 * i], pts[2 * i + 1]), (float)blockSize, -1, q[i]);
    }
    int nfeatures = 1000, blockSize = 3, gradSize = 3;
    double qualityLevel = 0.01, minDistance = 1, k = 0.04;
    bool useHarrisDetector = false;
};

}  // namespace cuda
}  // namespace b200cv
