// canny_ref_shim.cpp -- extern "C" wrappers around the reference's two cv::Canny overloads (imgproc/src/canny.cpp:823-1003), for the
// Canny tests and tools/make_canny_golden.py.  tools/build_canny_ref.py compiles it against the reference's headers and links it twice:
// with the plain reference (libcannyref.so) and with the reference whose imgproc HAL is hal/b200cv_hal_replacement.hpp
// (libcannyref_hal.so), where cv::Canny reaches b200cv_hal_canny.
// Return: 0 = done, -1 = cv::Exception (a refused argument).
#include <opencv2/core.hpp>
#include <opencv2/imgproc.hpp>
#include <cstring>

#define SHIM extern "C" __attribute__((visibility("default")))

// dst is written in place; the reference keeps the buffer because it already has the right size and type (Mat::create is a no-op)
SHIM int ref_canny(const unsigned char* src, size_t src_step, int width, int height, int cn, unsigned char* dst, size_t dst_step,
                   double threshold1, double threshold2, int aperture_size, int l2gradient)
{
    try {
        cv::Mat s(height, width, CV_8UC(cn), const_cast<unsigned char*>(src), src_step);
        cv::Mat d(height, width, CV_8UC1, dst, dst_step);
        if ((const void*)src == (const void*)dst) cv::Canny(d, d, threshold1, threshold2, aperture_size, l2gradient != 0);
        else cv::Canny(s, d, threshold1, threshold2, aperture_size, l2gradient != 0);
        if (d.data != dst) return -2;
        return 0;
    } catch (const cv::Exception&) {
        return -1;
    }
}

SHIM int ref_canny_derivs(const short* dx, size_t dx_step, const short* dy, size_t dy_step, int width, int height, int cn, unsigned char* dst,
                          size_t dst_step, double threshold1, double threshold2, int l2gradient)
{
    try {
        cv::Mat x(height, width, CV_16SC(cn), const_cast<short*>(dx), dx_step);
        cv::Mat y(height, width, CV_16SC(cn), const_cast<short*>(dy), dy_step);
        cv::Mat d(height, width, CV_8UC1, dst, dst_step);
        cv::Canny(x, y, d, threshold1, threshold2, l2gradient != 0);
        if (d.data != dst) return -2;
        return 0;
    } catch (const cv::Exception&) {
        return -1;
    }
}
