// b200cv::erode / dilate / morphologyEx over GpuMat (opencv_b200/host/b200cv.hpp) on an 8-bit image with one bright pixel.  Built with
// g++ and run on the GPU by tests/test_gpu_morphology.py.  Exit code 0 = a 3x5 dilate paints the 3x5 box around the pixel, the erode of
// that box restores the pixel (CLOSE), GRADIENT of the pixel is the box, and an anchor outside the element is refused.
#include <cstdio>
#include <vector>
#include "../../opencv_b200/host/b200cv.hpp"
using namespace b200cv;
int main()
{
    try {
        check(b200cv_init(0), "init");
        const int W = 97, H = 41, X0 = 30, Y0 = 20;
        std::vector<unsigned char> img((size_t)W * H, 10), dil((size_t)W * H), clo((size_t)W * H), grad((size_t)W * H);
        img[(size_t)Y0 * W + X0] = 200;
        const unsigned char k[15] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1};
        Stream stream;
        GpuMat d_img(H, W, makeType(CV_8U, 1)), d_dil, d_clo, d_grad;
        d_img.upload(img.data(), W, stream);
        dilate(d_img, d_dil, k, Size(5, 3), Point(-1, -1), 1, BORDER_CONSTANT, morphologyDefaultBorderValue(), stream);
        erode(d_dil, d_clo, k, Size(5, 3), Point(-1, -1), 1, BORDER_REPLICATE, morphologyDefaultBorderValue(), stream);
        morphologyEx(d_img, d_grad, B200CV_MORPH_GRADIENT, k, Size(5, 3), Point(-1, -1), 1, BORDER_REPLICATE, morphologyDefaultBorderValue(), stream);
        d_dil.download(dil.data(), W, stream);
        d_clo.download(clo.data(), W, stream);
        d_grad.download(grad.data(), W, stream);
        stream.waitForCompletion();
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) {
                const size_t i = (size_t)y * W + x;
                const bool box = x >= X0 - 2 && x <= X0 + 2 && y >= Y0 - 1 && y <= Y0 + 1;
                if (dil[i] != (box ? 200 : 10)) { printf("dilate mismatch at %d,%d: %d\n", x, y, dil[i]); return 2; }
                if (clo[i] != img[i]) { printf("close mismatch at %d,%d: %d\n", x, y, clo[i]); return 3; }
                if (grad[i] != (box ? 190 : 0)) { printf("gradient mismatch at %d,%d: %d\n", x, y, grad[i]); return 4; }
            }
        GpuMat d_bad;
        try { erode(d_img, d_bad, k, Size(5, 3), Point(5, 0), 1, BORDER_CONSTANT, morphologyDefaultBorderValue(), stream); printf("anchor accepted\n"); return 5; }
        catch (const Error&) {}
        printf("b200cv::morphology ok\n");
        return 0;
    } catch (const std::exception& ex) {
        printf("exception: %s\n", ex.what());
        return 1;
    }
}
