// extern "C" wrapper around the reference's cv::distanceTransform(src, dst, distanceType, maskSize, dstType), built by
// tools/build_dist_ref.py into oracle/_ref/libdistref.so against the reference library.  Test infrastructure only.
//
// ref_distance_transform has the signature of port_distance_transform (oracle/port/port_distance.c): src is 8UC1, dst receives the
// result row by row (W floats or W bytes per row), and the return value is the depth the reference produced (0 = 8U, 5 = 32F), or
// -1 where it refused the arguments (a cv::Exception).
#include <cstring>
#include <opencv2/imgproc.hpp>

extern "C" __attribute__((visibility("default"))) int ref_distance_transform(const unsigned char* src, size_t sstep, void* dst, size_t dstep,
                                                                            int w, int h, int dist_type, int mask_size, int dst_type)
{
    try {
        cv::Mat s(h, w, CV_8UC1, const_cast<unsigned char*>(src), sstep), d;
        cv::distanceTransform(s, d, dist_type, mask_size, dst_type);
        const size_t row = (size_t)w * d.elemSize();
        for (int y = 0; y < h; y++) std::memcpy((char*)dst + (size_t)y * dstep, d.ptr(y), row);
        return d.depth();
    } catch (const cv::Exception&) {
        return -1;
    }
}
