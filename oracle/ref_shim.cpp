// oracle/ref_shim.cpp -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
//
// extern "C" wrappers around the UNMODIFIED reference's public cv:: entry points for the
// dense-imgproc hot path, so that tests/ and bench.py's cpu_baseline leg can call the real
// reference (built by oracle/build_ref.py into oracle/_ref/libocvref.so) through ctypes.
// Every wrapper only builds cv::Mat headers over caller memory and forwards; no arithmetic
// lives here.  Reference entry points forwarded to:
//   cv::GaussianBlur        modules/imgproc/src/smooth.dispatch.cpp:609
//   cv::sepFilter2D         modules/imgproc/src/filter.dispatch.cpp:1555
//   cv::filter2D            modules/imgproc/src/filter.dispatch.cpp:1521
//   cv::resize              modules/imgproc/src/resize.cpp:4201
//   cv::warpAffine          modules/imgproc/src/imgwarp.cpp:2788
//   cv::warpPerspective     modules/imgproc/src/imgwarp.cpp:3370
//   cv::cvtColor            modules/imgproc/src/color.cpp:192
//   cv::matchTemplate       modules/imgproc/src/templmatch.cpp:1158
//   cv::cornerHarris        modules/imgproc/src/corner.cpp:634
//   cv::goodFeaturesToTrack modules/imgproc/src/featureselect.cpp:382
//   SIFT_Impl::{createInitialImage,buildGaussianPyramid,buildDoGPyramid}
//                           modules/features2d/src/sift.dispatch.cpp:176,224,302
#include <cstring>
#include <vector>
#include "opencv2/core.hpp"
#include "opencv2/core/softfloat.hpp"
#include "opencv2/imgproc.hpp"

// The SIFT pyramid builders live inside the reference's translation unit; compile that TU as
// part of this one (by path, nothing copied) so they can be called directly.
#include REF_SIFT_DISPATCH_CPP

#define API extern "C" __attribute__((visibility("default")))

using namespace cv;

static inline Mat hdr(const void* p, size_t step, int w, int h, int type)
{
    return Mat(h, w, type, const_cast<void*>(p), step);
}

#define GUARD_BEGIN try {
#define GUARD_END } catch (const cv::Exception& e) { std::fprintf(stderr, "ref_shim: %s\n", e.what()); return -1; } \
                    catch (...) { return -2; } return 0;

API int ref_set_num_threads(int n) { cv::setNumThreads(n); return cv::getNumThreads(); }
API int ref_get_num_threads(void) { return cv::getNumThreads(); }
API int ref_get_num_cpus(void) { return cv::getNumberOfCPUs(); }
API const char* ref_build_info(void) { static String s = cv::getBuildInformation(); return s.c_str(); }

// cv::RNG(seed).fill(UNIFORM, lo, hi) -- used to regenerate the reference tests' inputs
API int ref_rng_fill(void* p, size_t step, int w, int h, int type, unsigned long long seed, double lo, double hi)
{
    GUARD_BEGIN
    Mat m = hdr(p, step, w, h, type);
    RNG rng(seed);
    rng.fill(m, RNG::UNIFORM, lo, hi);
    GUARD_END
}

API int ref_gaussian_kernel(int n, double sigma, int ktype, void* out)
{
    GUARD_BEGIN
    Mat k = getGaussianKernel(n, sigma, ktype);
    std::memcpy(out, k.data, (size_t)n * k.elemSize());
    GUARD_END
}

API int ref_gaussian_blur(const void* src, size_t sstep, void* dst, size_t dstep, int w, int h, int type,
                          int kw, int kh, double sx, double sy, int border)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, w, h, type), d = hdr(dst, dstep, w, h, type);
    GaussianBlur(s, d, Size(kw, kh), sx, sy, border);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_sep_filter2d(const void* src, size_t sstep, void* dst, size_t dstep, int w, int h, int stype, int ddepth,
                         const float* kx, int kxlen, const float* ky, int kylen, int ax, int ay, double delta, int border)
{
    GUARD_BEGIN
    int dtype = CV_MAKETYPE(ddepth < 0 ? CV_MAT_DEPTH(stype) : ddepth, CV_MAT_CN(stype));
    Mat s = hdr(src, sstep, w, h, stype), d = hdr(dst, dstep, w, h, dtype);
    Mat mkx(1, kxlen, CV_32F, (void*)kx), mky(kylen, 1, CV_32F, (void*)ky);
    sepFilter2D(s, d, ddepth, mkx, mky, Point(ax, ay), delta, border);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_filter2d(const void* src, size_t sstep, void* dst, size_t dstep, int w, int h, int stype, int ddepth,
                     const float* kernel, int kw, int kh, int ax, int ay, double delta, int border)
{
    GUARD_BEGIN
    int dtype = CV_MAKETYPE(ddepth < 0 ? CV_MAT_DEPTH(stype) : ddepth, CV_MAT_CN(stype));
    Mat s = hdr(src, sstep, w, h, stype), d = hdr(dst, dstep, w, h, dtype);
    Mat k(kh, kw, CV_32F, (void*)kernel);
    filter2D(s, d, ddepth, k, Point(ax, ay), delta, border);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_sobel(const void* src, size_t sstep, void* dst, size_t dstep, int w, int h, int stype, int ddepth,
                  int dx, int dy, int ksize, double scale, double delta, int border)
{
    GUARD_BEGIN
    int dtype = CV_MAKETYPE(ddepth < 0 ? CV_MAT_DEPTH(stype) : ddepth, CV_MAT_CN(stype));
    Mat s = hdr(src, sstep, w, h, stype), d = hdr(dst, dstep, w, h, dtype);
    Sobel(s, d, ddepth, dx, dy, ksize, scale, delta, border);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_resize(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type, int interp)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, sw, sh, type), d = hdr(dst, dstep, dw, dh, type);
    resize(s, d, Size(dw, dh), 0, 0, interp);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

// cv::resize(src, dst, Size(), fx, fy): dst must be round(cols*fx) x round(rows*fy) (resize.cpp:4214-4228); the scale stays fx, fy
API int ref_resize_fxfy(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type, int interp, double fx, double fy)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, sw, sh, type), d = hdr(dst, dstep, dw, dh, type);
    resize(s, d, Size(), fx, fy, interp);
    CV_Assert(d.data == (uchar*)dst && d.cols == dw && d.rows == dh);
    GUARD_END
}

API int ref_warp_affine(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type,
                        const double* M, int flags, int border, const double* bv)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, sw, sh, type), d = hdr(dst, dstep, dw, dh, type);
    Mat m(2, 3, CV_64F, (void*)M);
    warpAffine(s, d, m, Size(dw, dh), flags, border, Scalar(bv[0], bv[1], bv[2], bv[3]));
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_warp_perspective(const void* src, size_t sstep, int sw, int sh, void* dst, size_t dstep, int dw, int dh, int type,
                             const double* M, int flags, int border, const double* bv)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, sw, sh, type), d = hdr(dst, dstep, dw, dh, type);
    Mat m(3, 3, CV_64F, (void*)M);
    warpPerspective(s, d, m, Size(dw, dh), flags, border, Scalar(bv[0], bv[1], bv[2], bv[3]));
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_remap(const void* src, size_t sstep, int sw, int sh, int type, void* dst, size_t dstep, int dw, int dh,
                  const void* m1, size_t m1step, int m1type, const void* m2, size_t m2step, int m2type, int interp, int border, const double* bv)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, sw, sh, type), d = hdr(dst, dstep, dw, dh, type);
    Mat a = hdr(m1, m1step, dw, dh, m1type), b;
    if (m2) b = hdr(m2, m2step, dw, dh, m2type);
    remap(s, d, a, b, interp, border, Scalar(bv[0], bv[1], bv[2], bv[3]));
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_convert_maps(const float* mx, const float* my, int w, int h, short* xy, unsigned short* frac, int nn)
{
    GUARD_BEGIN
    Mat a(h, w, CV_32FC1, (void*)mx), b(h, w, CV_32FC1, (void*)my), o1(h, w, CV_16SC2, xy), o2(h, w, CV_16UC1, frac);
    convertMaps(a, b, o1, o2, CV_16SC2, nn != 0);
    CV_Assert(o1.data == (uchar*)xy);
    GUARD_END
}

API int ref_pyr_down(const void* src, size_t sstep, int sw, int sh, int type, void* dst, size_t dstep, int border)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, sw, sh, type), d = hdr(dst, dstep, (sw + 1) / 2, (sh + 1) / 2, type);
    pyrDown(s, d, Size(), border);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_pyr_up(const void* src, size_t sstep, int sw, int sh, int type, void* dst, size_t dstep)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, sw, sh, type), d = hdr(dst, dstep, sw * 2, sh * 2, type);
    pyrUp(s, d);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_box_filter(const void* src, size_t sstep, int w, int h, int stype, void* dst, size_t dstep, int ddepth,
                       int kw, int kh, int ax, int ay, int normalize, int border)
{
    GUARD_BEGIN
    int dd = ddepth < 0 ? CV_MAT_DEPTH(stype) : ddepth;
    Mat s = hdr(src, sstep, w, h, stype), d = hdr(dst, dstep, w, h, CV_MAKETYPE(dd, CV_MAT_CN(stype)));
    boxFilter(s, d, dd, Size(kw, kh), Point(ax, ay), normalize != 0, border);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

// Filters on a ROI of a larger Mat (row a5: FilterEngine's wholeSize / ofs; the HAL sees margins / offsets): op 0 GaussianBlur(k, sigma),
// 1 blur(k), 2 sepFilter2D with getGaussianKernel(k, sigma) as CV_32F taps, 3 filter2D with a normalised k x k ramp, 4 Sobel(1, 0, k) (same depth).
// inplace != 0: the destination IS the ROI (then copied out), the case cv::filter2D / boxFilter allow.
API int ref_roi_filter(const void* parent, size_t pstep, int pw, int ph, int type, int rx, int ry, int rw, int rh, void* dst, size_t dstep,
                       int op, int k, double sigma, int border, int inplace)
{
    GUARD_BEGIN
    Mat par = hdr(parent, pstep, pw, ph, type).clone();
    Mat roi = par(Rect(rx, ry, rw, rh));
    Mat out = hdr(dst, dstep, rw, rh, type);
    Mat d = inplace ? roi : out;
    if (op == 0) GaussianBlur(roi, d, Size(k, k), sigma, sigma, border);
    else if (op == 1) blur(roi, d, Size(k, k), Point(-1, -1), border);
    else if (op == 2) { Mat kx = getGaussianKernel(k, sigma, CV_32F); sepFilter2D(roi, d, -1, kx, kx, Point(-1, -1), 0, border); }
    else if (op == 3) {
        Mat ker(k, k, CV_32F);
        float sum = 0;
        for (int i = 0; i < k * k; i++) { ker.at<float>(i / k, i % k) = (float)(1 + (i * 7) % 5); sum += ker.at<float>(i / k, i % k); }
        ker /= sum;
        filter2D(roi, d, -1, ker, Point(-1, -1), 0, border);
    } else if (op == 4) Sobel(roi, d, -1, 1, 0, k, 1, 0, border);
    else return -2;
    if (inplace) roi.copyTo(out);
    CV_Assert(out.data == (uchar*)dst);
    GUARD_END
}

API int ref_invert_affine(const double* M, double* iM)
{
    GUARD_BEGIN
    Mat m(2, 3, CV_64F, (void*)M), im(2, 3, CV_64F, iM);
    invertAffineTransform(m, im);
    GUARD_END
}

API int ref_invert3x3(const double* M, double* iM)
{
    GUARD_BEGIN
    Mat m(3, 3, CV_64F, (void*)M), im(3, 3, CV_64F, iM);
    invert(m, im);
    CV_Assert(im.data == (uchar*)iM);
    GUARD_END
}

API int ref_get_rotation_matrix2d(double cx, double cy, double angle, double scale, double* M)
{
    GUARD_BEGIN
    Mat m = getRotationMatrix2D(Point2f((float)cx, (float)cy), angle, scale);
    std::memcpy(M, m.data, 6 * sizeof(double));
    GUARD_END
}

API int ref_cvt_color(const void* src, size_t sstep, void* dst, size_t dstep, int w, int h, int stype, int dtype, int code)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, w, h, stype), d = hdr(dst, dstep, w, h, dtype);
    cvtColor(s, d, code, CV_MAT_CN(dtype));
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_cvt_color_yuv(const void* src, size_t sstep, int sw, int sh, int scn, void* dst, size_t dstep, int dw, int dh, int dcn, int code)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, sw, sh, CV_MAKETYPE(CV_8U, scn)), d = hdr(dst, dstep, dw, dh, CV_MAKETYPE(CV_8U, dcn));
    cvtColor(s, d, code, dcn);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_cvt_color_two_plane(const void* y, size_t ystep, const void* uv, size_t uvstep, int w, int h, void* dst, size_t dstep, int dcn, int code)
{
    GUARD_BEGIN
    Mat sy = hdr(y, ystep, w, h, CV_8UC1), suv = hdr(uv, uvstep, w / 2, h / 2, CV_8UC2), d = hdr(dst, dstep, w, h, CV_MAKETYPE(CV_8U, dcn));
    cvtColorTwoPlane(sy, suv, d, code);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_integral(const void* src, size_t sstep, int w, int h, int* sum, size_t sumstep, double* sqsum, size_t sqstep)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, w, h, CV_8UC1), o = hdr(sum, sumstep, w + 1, h + 1, CV_32SC1);
    if (sqsum) {
        Mat q = hdr(sqsum, sqstep, w + 1, h + 1, CV_64FC1);
        integral(s, o, q, CV_32S, CV_64F);
        CV_Assert(q.data == (uchar*)sqsum);
    } else integral(s, o, CV_32S);
    CV_Assert(o.data == (uchar*)sum);
    GUARD_END
}

API int ref_match_template(const void* img, size_t istep, int iw, int ih, const void* templ, size_t tstep, int tw, int th,
                           int type, float* result, size_t rstep, int method)
{
    GUARD_BEGIN
    Mat i = hdr(img, istep, iw, ih, type), t = hdr(templ, tstep, tw, th, type);
    Mat r = hdr(result, rstep, iw - tw + 1, ih - th + 1, CV_32F);
    matchTemplate(i, t, r, method);
    CV_Assert(r.data == (uchar*)result);
    GUARD_END
}

API int ref_match_template_masked(const void* img, size_t istep, int iw, int ih, const void* templ, size_t tstep, int tw, int th, int type,
                                  const void* mask, size_t mstep, int mask_type, float* result, size_t rstep, int method)
{
    GUARD_BEGIN
    Mat i = hdr(img, istep, iw, ih, type), t = hdr(templ, tstep, tw, th, type), m = hdr(mask, mstep, tw, th, mask_type);
    Mat r = hdr(result, rstep, iw - tw + 1, ih - th + 1, CV_32F);
    matchTemplate(i, t, r, method, m);
    CV_Assert(r.data == (uchar*)result);
    GUARD_END
}

API int ref_corner_harris(const void* src, size_t sstep, int w, int h, int type, float* dst, size_t dstep,
                          int blockSize, int ksize, double k, int border)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, w, h, type), d = hdr(dst, dstep, w, h, CV_32F);
    cornerHarris(s, d, blockSize, ksize, k, border);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

API int ref_corner_min_eigen_val(const void* src, size_t sstep, int w, int h, int type, float* dst, size_t dstep,
                                 int blockSize, int ksize, int border)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, w, h, type), d = hdr(dst, dstep, w, h, CV_32F);
    cornerMinEigenVal(s, d, blockSize, ksize, border);
    CV_Assert(d.data == (uchar*)dst);
    GUARD_END
}

// corners: out array of 2*maxOut floats (x,y); quality: optional out array of maxOut floats; returns count in *n
API int ref_good_features_to_track(const void* src, size_t sstep, int w, int h, int type, float* corners, float* quality,
                                   int maxOut, int* n, int maxCorners, double qualityLevel, double minDistance,
                                   int blockSize, int gradientSize, int useHarris, double k)
{
    GUARD_BEGIN
    Mat s = hdr(src, sstep, w, h, type);
    std::vector<Point2f> pts;
    std::vector<float> q;
    goodFeaturesToTrack(s, pts, maxCorners, qualityLevel, minDistance, noArray(), q, blockSize, gradientSize, useHarris != 0, k);
    int cnt = (int)std::min<size_t>(pts.size(), (size_t)maxOut);
    for (int i = 0; i < cnt; i++) {
        corners[2 * i] = pts[i].x; corners[2 * i + 1] = pts[i].y;
        if (quality) quality[i] = q[i];
    }
    *n = (int)pts.size();
    GUARD_END
}

// ---- the whole SIFT front end (detectAndCompute, sift.dispatch.cpp:501-580): keypoints + descriptors of the unmodified reference.
// kp: 6 floats per keypoint (x, y, size, angle, response, octave as int bits), desc: 128 floats per keypoint; at most max_kp are written,
// *n receives the number found.  The oracle for the SIFT front end (scale-space extrema, orientation, descriptors).
API int ref_sift_detect_and_compute(const void* gray, size_t step, int w, int h, int nfeatures, int nOctaveLayers, double contrastThreshold,
                                    double edgeThreshold, double sigma, int precise_upscale, const void* mask, size_t mask_step, int max_kp, float* kp,
                                    float* desc, int* n)
{
    GUARD_BEGIN
    Mat image = hdr(gray, step, w, h, CV_8UC1);
    Ptr<SIFT> sp = SIFT::create(nfeatures, nOctaveLayers, contrastThreshold, edgeThreshold, sigma, precise_upscale != 0);
    std::vector<KeyPoint> kps;
    Mat d;
    if (mask) sp->detectAndCompute(image, hdr(mask, mask_step, w, h, CV_8UC1), kps, d);
    else sp->detectAndCompute(image, noArray(), kps, d);
    *n = (int)kps.size();
    for (int i = 0; i < (int)kps.size() && i < max_kp; i++) {
        const KeyPoint& k = kps[i];
        float* o = kp + 6 * i;
        o[0] = k.pt.x; o[1] = k.pt.y; o[2] = k.size; o[3] = k.angle; o[4] = k.response;
        std::memcpy(o + 5, &k.octave, 4);
        if (desc) std::memcpy(desc + 128 * (size_t)i, d.ptr<float>(i), 128 * sizeof(float));
    }
    GUARD_END
}

// ---- SIFT Gaussian pyramid + DoG (sift.dispatch.cpp:176-310, :501-545 for the octave count) ----
// gray: 8UC1 w x h.  Outputs are packed tightly, image after image, octave-major:
//   gauss: nOctaves*(nOctaveLayers+3) images, dog: nOctaves*(nOctaveLayers+2) images, all CV_32F.
// dims (optional): per-octave (w,h) pairs, 2*nOctaves ints.  Pass gauss/dog = NULL to query sizes only:
//   *gauss_elems / *dog_elems receive the total float counts, *n_octaves the octave count.
API int ref_sift_pyramid(const void* gray, size_t step, int w, int h, int nOctaveLayers, double sigma, int firstOctave_upscale,
                         float* gauss, size_t* gauss_elems, float* dog, size_t* dog_elems, int* n_octaves, int* dims)
{
    GUARD_BEGIN
    Mat image = hdr(gray, step, w, h, CV_8UC1);
    int firstOctave = firstOctave_upscale ? -1 : 0;
    Ptr<SIFT> sp = SIFT::create(0, nOctaveLayers, 0.04, 10, sigma);
    SIFT_Impl* impl = dynamic_cast<SIFT_Impl*>(sp.get());
    CV_Assert(impl);
    Mat base = createInitialImage(image, firstOctave < 0, (float)sigma, firstOctave_upscale != 2);   // 2: SIFT::create's default (resize), 1: precise (warpAffine)
    int nOctaves = cvRound(std::log((double)std::min(base.cols, base.rows)) / std::log(2.) - 2) - firstOctave;
    // NB: the expression above mirrors sift.dispatch.cpp:538 (actualNOctaves == 0 branch)
    std::vector<Mat> gpyr, dogpyr;
    size_t ge = 0, de = 0;
    if (gauss || dog) {
        impl->buildGaussianPyramid(base, gpyr, nOctaves);
        impl->buildDoGPyramid(gpyr, dogpyr);
        for (size_t i = 0; i < gpyr.size(); i++) {
            const Mat& m = gpyr[i];
            if (gauss) for (int y = 0; y < m.rows; y++) std::memcpy(gauss + ge + (size_t)y * m.cols, m.ptr<float>(y), m.cols * sizeof(float));
            ge += (size_t)m.rows * m.cols;
            if (dims && i % (nOctaveLayers + 3) == 0) { dims[2 * (i / (nOctaveLayers + 3))] = m.cols; dims[2 * (i / (nOctaveLayers + 3)) + 1] = m.rows; }
        }
        for (size_t i = 0; i < dogpyr.size(); i++) {
            const Mat& m = dogpyr[i];
            if (dog) for (int y = 0; y < m.rows; y++) std::memcpy(dog + de + (size_t)y * m.cols, m.ptr<float>(y), m.cols * sizeof(float));
            de += (size_t)m.rows * m.cols;
        }
    } else {
        int cw = base.cols, ch = base.rows;
        for (int o = 0; o < nOctaves; o++) {
            ge += (size_t)cw * ch * (nOctaveLayers + 3);
            de += (size_t)cw * ch * (nOctaveLayers + 2);
            if (dims) { dims[2 * o] = cw; dims[2 * o + 1] = ch; }
            cw /= 2; ch /= 2;
        }
    }
    if (gauss_elems) *gauss_elems = ge;
    if (dog_elems) *dog_elems = de;
    if (n_octaves) *n_octaves = nOctaves;
    GUARD_END
}
