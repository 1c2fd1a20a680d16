// extern "C" wrapper around the reference's cv::Laplacian(src, dst, ddepth, ksize, scale, delta, borderType), built by
// tools/build_laplacian_ref.py into oracle/_ref/liblapref.so against the reference library.  Test infrastructure only.
//
// ref_laplacian has the signature of port_laplacian (oracle/port/port_laplacian.c): src is a whole continuous-row image of type stype,
// dst receives the result row by row, and the return value is 0, or -1 where the reference refused the arguments (a cv::Exception).
#include <cstring>
#include <opencv2/imgproc.hpp>

extern "C" __attribute__((visibility("default"))) int ref_laplacian(const void* src, size_t sstep, void* dst, size_t dstep, int w, int h,
                                                                   int stype, int ddepth, int ksize, double scale, double delta, int border)
{
    try {
        cv::Mat s(h, w, stype, const_cast<void*>(src), sstep), d;
        cv::Laplacian(s, d, ddepth, ksize, scale, delta, border);
        const size_t row = (size_t)w * d.elemSize();
        for (int y = 0; y < h; y++) std::memcpy((char*)dst + (size_t)y * dstep, d.ptr(y), row);
        return 0;
    } catch (const cv::Exception&) {
        return -1;
    }
}
