// extern "C" wrappers around the reference's cv::erode / cv::dilate / cv::morphologyEx and cv::getStructuringElement, built by
// tools/build_morph_ref.py into oracle/_ref/libmorphref.so against the reference library.  Test infrastructure only.
//
// ref_morphology: entry 0 calls cv::erode (op 0) or cv::dilate (op 1), entry 1 calls cv::morphologyEx(op).  kw or kh 0 is the empty
// element.  src and dst are h rows of w pixels of `type`; the return value is 0, or -1 where the reference refused the arguments.
#include <cstring>
#include <opencv2/imgproc.hpp>

extern "C" __attribute__((visibility("default"))) int ref_morphology(int type, const void* src, size_t sstep, void* dst, size_t dstep, int w,
                                                                    int h, int entry, int op, const unsigned char* k, int kw, int kh,
                                                                    int ax, int ay, int iterations, int border, const double* bv)
{
    try {
        cv::Mat s(h, w, type, const_cast<void*>(src), sstep), d;
        cv::Mat kern = kw > 0 && kh > 0 ? cv::Mat(kh, kw, CV_8UC1, const_cast<unsigned char*>(k)).clone() : cv::Mat();
        const cv::Scalar value(bv[0], bv[1], bv[2], bv[3]);
        if (entry == 0 && op == cv::MORPH_ERODE) cv::erode(s, d, kern, cv::Point(ax, ay), iterations, border, value);
        else if (entry == 0) cv::dilate(s, d, kern, cv::Point(ax, ay), iterations, border, value);
        else cv::morphologyEx(s, d, op, kern, cv::Point(ax, ay), iterations, border, value);
        const size_t row = (size_t)w * d.elemSize();
        for (int y = 0; y < h; y++) std::memcpy((char*)dst + (size_t)y * dstep, d.ptr(y), row);
        return 0;
    } catch (const cv::Exception&) {
        return -1;
    }
}

extern "C" __attribute__((visibility("default"))) int ref_structuring_element(int shape, int w, int h, int ax, int ay, unsigned char* out)
{
    try {
        cv::Mat e = cv::getStructuringElement(shape, cv::Size(w, h), cv::Point(ax, ay));
        for (int y = 0; y < h; y++) std::memcpy(out + (size_t)y * w, e.ptr(y), (size_t)w);
        return 0;
    } catch (const cv::Exception&) {
        return -1;
    }
}
