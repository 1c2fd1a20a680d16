// b200cv::Laplacian over GpuMat (opencv_b200/host/b200cv.hpp) on an image with one bright pixel.  Built with g++ and run on the GPU
// by tests/test_gpu_laplacian.py.  Exit code 0 = ksize 1 gives the 4-neighbour stencil, ksize 5 the sum of the two separable second
// derivatives (kd = 1 0 -2 0 1, ks = 1 4 6 4 1) times the pixel, and ksize 4 is refused.
#include <cstdio>
#include <vector>
#include "../../opencv_b200/host/b200cv.hpp"
using namespace b200cv;
int main()
{
    try {
        check(b200cv_init(0), "init");
        const int W = 77, H = 41, X0 = 30, Y0 = 20, V = 100;
        std::vector<unsigned char> img((size_t)W * H, 0);
        img[(size_t)Y0 * W + X0] = V;
        std::vector<short> l1((size_t)W * H), l5((size_t)W * H);
        Stream stream;
        GpuMat d_img(H, W, makeType(CV_8U, 1)), d_l1, d_l5;
        d_img.upload(img.data(), W, stream);
        Laplacian(d_img, d_l1, CV_16S, 1, 1, 0, BORDER_DEFAULT, stream);
        Laplacian(d_img, d_l5, CV_16S, 5, 1, 0, BORDER_DEFAULT, stream);
        d_l1.download(l1.data(), W * sizeof(short), stream);
        d_l5.download(l5.data(), W * sizeof(short), stream);
        stream.waitForCompletion();
        const int kd[5] = {1, 0, -2, 0, 1}, ks[5] = {1, 4, 6, 4, 1};
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) {
                const size_t i = (size_t)y * W + x;
                const int dx = x - X0, dy = y - Y0;
                const int e1 = (dx == 0 && dy == 0) ? -4 * V : (dx * dx + dy * dy == 1) ? V : 0;
                int e5 = 0;
                if (dx >= -2 && dx <= 2 && dy >= -2 && dy <= 2) e5 = V * (kd[2 - dx] * ks[2 - dy] + ks[2 - dx] * kd[2 - dy]);
                if (l1[i] != e1) { printf("ksize 1 mismatch at %d,%d: %d (want %d)\n", x, y, l1[i], e1); return 2; }
                if (l5[i] != e5) { printf("ksize 5 mismatch at %d,%d: %d (want %d)\n", x, y, l5[i], e5); return 3; }
            }
        GpuMat d_bad;
        try { Laplacian(d_img, d_bad, CV_16S, 4, 1, 0, BORDER_DEFAULT, stream); printf("ksize 4 accepted\n"); return 4; } catch (const Error&) {}
        printf("b200cv::Laplacian ok\n");
        return 0;
    } catch (const std::exception& ex) {
        printf("exception: %s\n", ex.what());
        return 1;
    }
}
