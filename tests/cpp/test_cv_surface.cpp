// The cv::-typed face (opencv_b200/host/b200cv_opencv.hpp) compiled against the REAL OpenCV headers of the reference
// (-I/root/reference/modules/{core,imgproc}/include) and linked with the reference itself (oracle/_ref/libocvref.so = core + imgproc, no CUDA):
// cv::InputArray kinds MAT, CUDA_GPU_MAT, CUDA_HOST_MEM (mat.hpp:163-188) reach the sm_90a kernels, cv::cuda::Filter usage as in
// samples/cpp/tutorial_code/gpu/gpu-basics-similarity/gpu-basics-similarity.cpp:392-404, results checked against cv:: on the CPU.
// Built into oracle/_ref/ by oracle/build_cv_surface.py where the reference's sources are, run by tests/test_gpu_hal.py.  Exit code 0 = all checks passed.
#include <cstdio>
#include <opencv2/core.hpp>
#include <opencv2/imgproc.hpp>
#define B200CV_WITH_OPENCV
#include "../../opencv_b200/host/b200cv.hpp"

static int fails = 0;
#define EXPECT(cond, what) do { if (!(cond)) { fprintf(stderr, "FAIL %s (%s:%d)\n", what, __FILE__, __LINE__); fails++; } else printf("ok   %s\n", what); } while (0)

static double maxdiff(const cv::Mat& a, const cv::Mat& b)
{
    if (a.size() != b.size() || a.type() != b.type()) return 1e30;
    return cv::norm(a, b, cv::NORM_INF);
}

int main()
{
    namespace bc = b200cv::cuda;
    try {
        b200cv::check(b200cv_init(0), "init");
        cv::RNG rng(0x5eed);
        cv::Mat bgr(479, 641, CV_8UC3), gray8, f32;
        rng.fill(bgr, cv::RNG::UNIFORM, 0, 256);
        cv::cvtColor(bgr, gray8, cv::COLOR_BGR2GRAY);
        gray8.convertTo(f32, CV_32F);

        // ---- kind MAT: host cv::Mat in, cv::Mat out (allocated by OutputArray::create), against the reference on the CPU -----------------------
        cv::Mat got, want;
        bc::GaussianBlur(bgr, got, cv::Size(5, 5), 0);
        cv::GaussianBlur(bgr, want, cv::Size(5, 5), 0);
        EXPECT(maxdiff(got, want) == 0, "MAT GaussianBlur 5x5 8UC3 == cv::GaussianBlur");
        bc::cvtColor(bgr, got, cv::COLOR_BGR2YUV);
        cv::cvtColor(bgr, want, cv::COLOR_BGR2YUV);
        EXPECT(maxdiff(got, want) == 0, "MAT cvtColor BGR2YUV == cv::cvtColor");
        cv::Mat roi = bgr(cv::Rect(17, 9, 400, 300));                       // a ROI: step != cols * elemSize
        bc::resize(roi, got, cv::Size(), 0.5, 0.75, cv::INTER_LINEAR);
        cv::resize(roi, want, cv::Size(), 0.5, 0.75, cv::INTER_LINEAR);
        EXPECT(maxdiff(got, want) == 0, "MAT(ROI) resize fx,fy LINEAR == cv::resize");
        cv::Matx23d M(0.9, 0.1, 5, -0.1, 0.9, 7);                            // kind MATX for M
        bc::warpAffine(bgr, got, M, bgr.size(), cv::INTER_CUBIC, cv::BORDER_REPLICATE);
        cv::warpAffine(bgr, want, M, bgr.size(), cv::INTER_CUBIC, cv::BORDER_REPLICATE);
        EXPECT(maxdiff(got, want) == 0, "MAT warpAffine CUBIC (M as Matx23d) == cv::warpAffine");
        cv::Mat kx = cv::getGaussianKernel(7, 1.2, CV_64F), ky = cv::getGaussianKernel(5, 0.9, CV_64F);
        bc::sepFilter2D(f32, got, -1, kx, ky);
        cv::sepFilter2D(f32, want, -1, kx, ky);
        EXPECT(maxdiff(got, want) <= 1e-4, "MAT sepFilter2D f32 (CV_64F taps) ~ cv::sepFilter2D");

        // ---- kind CUDA_GPU_MAT: the gpu-basics-similarity pattern ---------------------------------------------------------------------------
        b200cv::Stream stream;
        b200cv::DeviceMat d_src, d_mu;                                       // IS-A cv::cuda::GpuMat
        d_src.upload(f32, stream);
        cv::Ptr<bc::Filter> gauss = bc::createGaussianFilter(d_src.type(), -1, cv::Size(11, 11), 1.5);
        gauss->apply(d_src, d_mu, stream);                                   // d_mu is empty: allocated like cv::cuda functions do
        cv::cuda::GpuMat plain;                                              // a plain reference GpuMat as destination
        gauss->apply(d_src, plain, stream);
        cv::Mat h_mu, h_plain(plain.rows, plain.cols, plain.type());
        d_mu.download(h_mu, stream);
        b200cv::check(b200cv_download(plain.data, plain.step, h_plain.data, h_plain.step, (size_t)plain.cols * plain.elemSize(), plain.rows, stream.cudaPtr()), "download");
        stream.waitForCompletion();
        cv::GaussianBlur(f32, want, cv::Size(11, 11), 1.5);
        EXPECT(d_mu.rows == f32.rows && d_mu.cols == f32.cols && d_mu.type() == CV_32FC1, "GPU_MAT destination created with the source's geometry");
        EXPECT(maxdiff(h_mu, want) <= 1e-4, "GPU_MAT createGaussianFilter(11x11, 1.5)->apply ~ cv::GaussianBlur");
        EXPECT(maxdiff(h_plain, h_mu) == 0, "GPU_MAT plain cv::cuda::GpuMat destination == DeviceMat destination");
        const uchar* before = plain.data;
        gauss->apply(d_src, plain, stream);                                  // right size already: reused, not reallocated
        EXPECT(plain.data == before, "GPU_MAT destination of the right size is reused");
        cv::cuda::GpuMat wrapped(d_src.rows, d_src.cols, d_src.type(), d_src.data, d_src.step);    // user memory through the reference's wrapping constructor
        b200cv::DeviceMat d_h;
        bc::cornerHarris(wrapped, d_h, 2, 3, 0.04, cv::BORDER_DEFAULT, stream);
        cv::Mat h_h;
        d_h.download(h_h, stream);
        stream.waitForCompletion();
        cv::cornerHarris(f32, want, 2, 3, 0.04);
        double mx; cv::minMaxLoc(cv::abs(want), nullptr, &mx);
        EXPECT(maxdiff(h_h, want) <= 5e-7 * mx, "GPU_MAT cornerHarris on a wrapped GpuMat ~ cv::cornerHarris");
        b200cv::DeviceMat d_u8, d_res, d_t;
        d_u8.upload(gray8); d_t.upload(gray8(cv::Rect(100, 60, 48, 32)));
        bc::matchTemplate(d_u8, d_t, d_res, cv::TM_CCORR_NORMED);
        cv::Mat h_res; d_res.download(h_res);
        cv::matchTemplate(gray8, gray8(cv::Rect(100, 60, 48, 32)), want, cv::TM_CCORR_NORMED);
        EXPECT(maxdiff(h_res, want) <= 1e-3, "GPU_MAT matchTemplate CCORR_NORMED ~ cv::matchTemplate");
        std::vector<cv::Point2f> corners, corners_ref;
        cv::Mat blurred; cv::GaussianBlur(gray8, blurred, cv::Size(9, 9), 2.0);
        bc::goodFeaturesToTrack(blurred, corners, 200, 0.01, 10, cv::noArray(), 3, true, 0.04);
        cv::goodFeaturesToTrack(blurred, corners_ref, 200, 0.01, 10, cv::noArray(), 3, true, 0.04);
        size_t same = 0;
        for (size_t i = 0; i < std::min(corners.size(), corners_ref.size()); i++) same += corners[i] == corners_ref[i];
        EXPECT(corners.size() == corners_ref.size() && same + 4 >= corners_ref.size(), "goodFeaturesToTrack -> std::vector<Point2f> ~ cv::goodFeaturesToTrack");
        // cv::GFTTDetector (features2d/src/gftt.cpp:131-151): keypoints = (corner, size = blockSize, angle -1, response = quality); BGR input -> BGR2GRAY
        cv::Ptr<bc::GFTTDetector> det = bc::GFTTDetector::create(200, 0.01, 10, 3, 3, true, 0.04);
        std::vector<cv::KeyPoint> kps;
        det->detect(blurred, kps);
        bool kp_ok = kps.size() == corners_ref.size();
        size_t kp_same = 0;
        for (size_t i = 0; kp_ok && i < kps.size(); i++) { kp_same += kps[i].pt == corners_ref[i]; kp_ok = kps[i].size == 3.f && kps[i].angle == -1.f && kps[i].response > 0; }
        EXPECT(kp_ok && kp_same + 4 >= corners_ref.size(), "GFTTDetector::detect(Mat) ~ cv::goodFeaturesToTrack corners, KeyPoint fields as gftt.cpp");
        cv::Mat bl3; cv::cvtColor(blurred, bl3, cv::COLOR_GRAY2BGR);
        b200cv::DeviceMat d_bl3; d_bl3.upload(bl3);
        std::vector<cv::KeyPoint> kps3;
        det->detect(d_bl3, kps3);
        bool same3 = kps3.size() == kps.size();
        for (size_t i = 0; same3 && i < kps.size(); i++) same3 = kps3[i].pt == kps[i].pt;
        EXPECT(same3, "GFTTDetector::detect(GpuMat 8UC3) == detect(gray)");
        det->setMaxFeatures(10);
        det->detect(blurred, kps);
        EXPECT(kps.size() == 10 && det->getMaxFeatures() == 10, "GFTTDetector::setMaxFeatures");
        bool threw = false;
        try { bc::GaussianBlur(d_src, got, cv::Size(3, 3), 0); } catch (const b200cv::Error&) { threw = true; }
        EXPECT(threw, "device source with a host destination is refused");

        // ---- kind CUDA_HOST_MEM: page-locked host memory --------------------------------------------------------------------------------------
        b200cv::PinnedMat p_src(bgr.rows, bgr.cols, CV_8UC3), p_dst(bgr.rows, bgr.cols, CV_8UC1);      // IS-A cv::cuda::HostMem
        bgr.copyTo(p_src.mat());
        bc::cvtColor(p_src, p_dst, cv::COLOR_BGR2GRAY);
        EXPECT(maxdiff(p_dst.mat(), gray8) == 0, "HOST_MEM cvtColor BGR2GRAY == cv::cvtColor");

        // ---- GpuMat::Allocator {allocate, free} (cuda.hpp:108-115) --------------------------------------------------------------------------------
        cv::cuda::GpuMat raw((cv::cuda::GpuMat::Allocator*)nullptr);
        EXPECT(b200cv::deviceAllocator().allocate(&raw, 100, 333, 4) && raw.data && raw.step >= 333 * 4 && raw.step % 256 == 0 && raw.refcount && *raw.refcount == 1,
               "DeviceAllocator::allocate fills data, step, refcount");
        b200cv::deviceAllocator().free(&raw);
        bc::releaseOutputs();
        printf("%s: %d failure(s)\n", fails ? "FAILED" : "cv surface ok", fails);
        return fails ? 10 : 0;
    } catch (const std::exception& e) {
        fprintf(stderr, "exception: %s\n", e.what());
        return 1;
    }
}
