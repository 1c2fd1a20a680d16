// b200cv::Canny over GpuMat (opencv_b200/host/b200cv.hpp): both overloads on a vertical step edge.  Built with g++ and run on the GPU by
// tests/test_gpu_canny_exact.py.  Exit code 0 = the image overload marks exactly the column left of the step, and the derivative overload
// over the device's own 16S Sobel gives the same bytes.
#include <cstdio>
#include <cstring>
#include <vector>
#include "../../opencv_b200/host/b200cv.hpp"
using namespace b200cv;
int main()
{
    try {
        check(b200cv_init(0), "init");
        const int W = 97, H = 45;
        std::vector<unsigned char> img((size_t)W * H), e1((size_t)W * H), e2((size_t)W * H);
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) img[(size_t)y * W + x] = x < 40 ? 20 : 220;
        Stream stream;
        GpuMat d_img(H, W, makeType(CV_8U, 1)), d_e1, d_e2, d_dx, d_dy;
        d_img.upload(img.data(), W, stream);
        Canny(d_img, d_e1, 50, 150, 3, false, stream);
        Sobel(d_img, d_dx, CV_16S, 1, 0, 3, 1, 0, BORDER_REPLICATE, stream);
        Sobel(d_img, d_dy, CV_16S, 0, 1, 3, 1, 0, BORDER_REPLICATE, stream);
        Canny(d_dx, d_dy, d_e2, 50, 150, false, stream);
        d_e1.download(e1.data(), W, stream);
        d_e2.download(e2.data(), W, stream);
        stream.waitForCompletion();
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++)
                if (e1[(size_t)y * W + x] != (x == 39 ? 255 : 0)) { printf("edge mismatch at %d,%d: %d\n", x, y, e1[(size_t)y * W + x]); return 2; }
        if (memcmp(e1.data(), e2.data(), e1.size()) != 0) { printf("Canny(dx, dy) differs from Canny(image)\n"); return 3; }
        GpuMat d_bad;
        try { Canny(d_img, d_bad, 50, 150, 4, false, stream); printf("aperture 4 accepted\n"); return 4; } catch (const Error&) {}
        printf("b200cv::Canny ok\n");
        return 0;
    } catch (const std::exception& ex) {
        printf("exception: %s\n", ex.what());
        return 1;
    }
}
