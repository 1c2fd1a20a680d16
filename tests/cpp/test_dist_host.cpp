// b200cv::distanceTransform over GpuMat (opencv_b200/host/b200cv.hpp) on an image with one zero pixel.  Built with g++ and run on the GPU
// by tests/test_gpu_distance_transform.py.  Exit code 0 = the precise call gives the Euclidean distance to the zero pixel, the 3x3 L1
// chamfer the city-block one, the 8-bit L1 call (in place) the same saturated at 255, and a 7x7 mask is refused.
#include <cmath>
#include <cstdio>
#include <vector>
#include "../../opencv_b200/host/b200cv.hpp"
using namespace b200cv;
int main()
{
    try {
        check(b200cv_init(0), "init");
        const int W = 301, H = 67, X0 = 17, Y0 = 40;
        std::vector<unsigned char> img((size_t)W * H, 200), u8((size_t)W * H);
        img[(size_t)Y0 * W + X0] = 0;
        std::vector<float> e((size_t)W * H), l1((size_t)W * H);
        Stream stream;
        GpuMat d_img(H, W, makeType(CV_8U, 1)), d_e, d_l1;
        d_img.upload(img.data(), W, stream);
        distanceTransform(d_img, d_e, B200CV_DIST_L2, B200CV_DIST_MASK_PRECISE, CV_32F, stream);
        distanceTransform(d_img, d_l1, B200CV_DIST_L1, B200CV_DIST_MASK_3, CV_32F, stream);
        distanceTransform(d_img, d_img, B200CV_DIST_L1, B200CV_DIST_MASK_3, CV_8U, stream);
        d_e.download(e.data(), W * sizeof(float), stream);
        d_l1.download(l1.data(), W * sizeof(float), stream);
        d_img.download(u8.data(), W, stream);
        stream.waitForCompletion();
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) {
                const size_t i = (size_t)y * W + x;
                const int dx = x - X0, dy = y - Y0, city = std::abs(dx) + std::abs(dy);
                if (e[i] != std::sqrt((float)(dx * dx + dy * dy))) { printf("precise mismatch at %d,%d: %g\n", x, y, e[i]); return 2; }
                if (l1[i] != (float)city) { printf("L1 mismatch at %d,%d: %g\n", x, y, l1[i]); return 3; }
                if (u8[i] != (city < 255 ? city : 255)) { printf("8-bit L1 mismatch at %d,%d: %d\n", x, y, u8[i]); return 4; }
            }
        GpuMat d_bad;
        try { distanceTransform(d_img, d_bad, B200CV_DIST_L2, 7, CV_32F, stream); printf("mask 7 accepted\n"); return 5; } catch (const Error&) {}
        printf("b200cv::distanceTransform ok\n");
        return 0;
    } catch (const std::exception& ex) {
        printf("exception: %s\n", ex.what());
        return 1;
    }
}
