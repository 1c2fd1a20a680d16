// sift_detect.cu -- the SIFT front end after the pyramid: scale-space extrema, sub-pixel refinement, orientation
// assignment and the 128-element descriptors, consuming the packed Gaussian / DoG pyramids that b200cv_sift_pyramid leaves in HBM.
//
// Reference: findScaleSpaceExtrema (sift.dispatch.cpp:368-402; sift.simd.hpp:400-681), adjustLocalExtrema (:291-397), calcOrientationHist
// (:160-288), calcSIFTDescriptor (:709-1035), removeDuplicatedSorted + first-octave rescaling (sift.dispatch.cpp:529-560).
//   extrema:     |v| > floor(0.5 * contrastThreshold / nOctaveLayers * 255) and v >= (<=) all 26 neighbours in the 3 adjacent DoG layers
//   refinement:  up to 5 Newton steps of the 3-D quadratic fit (3 x 3 solve by Cramer's rule in float, as Matx33f::solve does), contrast and
//                edge-response tests, KeyPoint{pt, size, response, packed octave}
//   orientation: 36-bin histogram of Gaussian-weighted gradient magnitudes over radius round(4.5 s), [1 4 6 4 1]/16 smoothing, every peak
//                >= 0.8 max becomes a keypoint with a parabola-interpolated angle
//   descriptor:  4 x 4 x 8 tri-linear histogram over radius round(3 s sqrt2 2.5), clipped at 0.2 |h|, renormalised to 512, saturated to bytes
// Parity is by tolerance, as for the port (oracle/port/port_features.c: the reference's objects are FMA-contracted and use OpenCV's own
// exp / atan2 approximations): keypoints agree to ~1e-4 px apart from borderline accept / reject decisions, descriptor bytes to +-1.
// fastAtan2's polynomial (mathfuncs_core.simd.hpp:52-72) is reproduced because its 0.3-degree error moves samples between bins.
// Two kernels, one thread per DoG pixel / candidate; candidates and keypoints are appended with atomics and the final order is fixed by
// the reference's own sort (KeyPoint12_LessThan) on the host, where the reference also does it.  The descriptors of the sorted keypoints
// are computed by sift_desc_warp.cu, a warp per keypoint.
#include <math.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "common.cuh"
#include "sift_detect.cuh"

namespace b200cv {

int sift_descriptors_warp(const SiftPyr& p, int first_octave, const SiftKp* kps, int nkp, float* desc, cudaStream_t st);   // sift_desc_warp.cu

namespace {

// ---- 1. extrema: one thread per interior pixel of DoG layer `layer` (1..nl) of octave o ------------------------------------------------
__global__ void __launch_bounds__(256) sift_extrema_kernel(SiftPyr p, int o, float threshold, SiftCand* cand, int* ncand, int cap)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x + SIFT_BORDER;
    const int r = blockIdx.y + SIFT_BORDER, layer = blockIdx.z + 1;
    const int cw = p.w[o], ch = p.h[o];
    if (c >= cw - SIFT_BORDER || r >= ch - SIFT_BORDER) return;
    const size_t n = (size_t)cw * ch;
    const float* img = p.dog + p.doff[o] + (size_t)layer * n;
    const float val = img[(size_t)r * cw + c];
    if (fabsf(val) <= threshold) return;
    bool ok = true;
    for (int dz = -1; dz <= 1 && ok; dz++) {
        const float* q = img + (ptrdiff_t)dz * (ptrdiff_t)n;
        for (int dy = -1; dy <= 1 && ok; dy++)
            for (int dx = -1; dx <= 1; dx++) {
                const float v = q[(size_t)(r + dy) * cw + c + dx];
                if (val > 0 ? val < v : val > v) { ok = false; break; }
            }
    }
    if (!ok) return;
    const int slot = atomicAdd(ncand, 1);
    if (slot < cap) { SiftCand s; s.o = o; s.layer = layer; s.r = r; s.c = c; cand[slot] = s; }
}

__device__ bool sift_adjust(const float* dogo, int cw, int ch, int nl, int octv, int& layer, int& r, int& c, float contrastThreshold, float edgeThreshold,
                            float sigma, SiftKp& kpt)
{
    const float img_scale = 1.f / 255, deriv_scale = img_scale * 0.5f, second_deriv_scale = img_scale, cross_deriv_scale = img_scale * 0.25f;
    const size_t n = (size_t)cw * ch;
    float xi = 0, xr = 0, xc = 0, contr = 0;
    int i = 0;
#define AT(P, R, C) (P)[(size_t)(R) * cw + (C)]
    for (; i < 5; i++) {
        const float* img = dogo + (size_t)layer * n; const float* prev = img - n; const float* next = img + n;
        const float d0 = (AT(img, r, c + 1) - AT(img, r, c - 1)) * deriv_scale, d1 = (AT(img, r + 1, c) - AT(img, r - 1, c)) * deriv_scale,
                    d2 = (AT(next, r, c) - AT(prev, r, c)) * deriv_scale;
        const float v2 = AT(img, r, c) * 2;
        const float dxx = (AT(img, r, c + 1) + AT(img, r, c - 1) - v2) * second_deriv_scale;
        const float dyy = (AT(img, r + 1, c) + AT(img, r - 1, c) - v2) * second_deriv_scale;
        const float dss = (AT(next, r, c) + AT(prev, r, c) - v2) * second_deriv_scale;
        const float dxy = (AT(img, r + 1, c + 1) - AT(img, r + 1, c - 1) - AT(img, r - 1, c + 1) + AT(img, r - 1, c - 1)) * cross_deriv_scale;
        const float dxs = (AT(next, r, c + 1) - AT(next, r, c - 1) - AT(prev, r, c + 1) + AT(prev, r, c - 1)) * cross_deriv_scale;
        const float dys = (AT(next, r + 1, c) - AT(next, r - 1, c) - AT(prev, r + 1, c) + AT(prev, r - 1, c)) * cross_deriv_scale;
        const float a00 = dxx, a01 = dxy, a02 = dxs, a10 = dxy, a11 = dyy, a12 = dys, a20 = dxs, a21 = dys, a22 = dss;
        float d = a00 * (a11 * a22 - a21 * a12) - a01 * (a10 * a22 - a20 * a12) + a02 * (a10 * a21 - a20 * a11);
        float X0 = 0, X1 = 0, X2 = 0;
        if (d != 0) {
            d = 1 / d;
            X0 = d * (d0 * (a11 * a22 - a12 * a21) - a01 * (d1 * a22 - a12 * d2) + a02 * (d1 * a21 - a11 * d2));
            X1 = d * (a00 * (d1 * a22 - a12 * d2) - d0 * (a10 * a22 - a12 * a20) + a02 * (a10 * d2 - d1 * a20));
            X2 = d * (a00 * (a11 * d2 - d1 * a21) - a01 * (a10 * d2 - d1 * a20) + d0 * (a10 * a21 - a11 * a20));
        }
        xi = -X2; xr = -X1; xc = -X0;
        if (fabsf(xi) < 0.5f && fabsf(xr) < 0.5f && fabsf(xc) < 0.5f) break;
        if (fabsf(xi) > (float)(2147483647 / 3) || fabsf(xr) > (float)(2147483647 / 3) || fabsf(xc) > (float)(2147483647 / 3)) return false;
        c += __float2int_rn(xc); r += __float2int_rn(xr); layer += __float2int_rn(xi);
        if (layer < 1 || layer > nl || c < SIFT_BORDER || c >= cw - SIFT_BORDER || r < SIFT_BORDER || r >= ch - SIFT_BORDER) return false;
    }
    if (i >= 5) return false;
    {
        const float* img = dogo + (size_t)layer * n; const float* prev = img - n; const float* next = img + n;
        const float d0 = (AT(img, r, c + 1) - AT(img, r, c - 1)) * deriv_scale, d1 = (AT(img, r + 1, c) - AT(img, r - 1, c)) * deriv_scale,
                    d2 = (AT(next, r, c) - AT(prev, r, c)) * deriv_scale;
        const float t = d0 * xc + d1 * xr + d2 * xi;
        contr = AT(img, r, c) * img_scale + t * 0.5f;
        if (fabsf(contr) * nl < contrastThreshold) return false;
        const float v2 = AT(img, r, c) * 2.f;
        const float dxx = (AT(img, r, c + 1) + AT(img, r, c - 1) - v2) * second_deriv_scale;
        const float dyy = (AT(img, r + 1, c) + AT(img, r - 1, c) - v2) * second_deriv_scale;
        const float dxy = (AT(img, r + 1, c + 1) - AT(img, r + 1, c - 1) - AT(img, r - 1, c + 1) + AT(img, r - 1, c - 1)) * cross_deriv_scale;
        const float tr = dxx + dyy, det = dxx * dyy - dxy * dxy;
        if (det <= 0 || tr * tr * edgeThreshold >= (edgeThreshold + 1) * (edgeThreshold + 1) * det) return false;
    }
#undef AT
    kpt.x = (c + xc) * (1 << octv);
    kpt.y = (r + xr) * (1 << octv);
    kpt.octave = octv + (layer << 8) + (__double2int_rn(((double)xi + 0.5) * 255) << 16);
    kpt.size = sigma * powf(2.f, (layer + xi) / nl) * (1 << octv) * 2;
    kpt.response = fabsf(contr);
    return true;
}

// ---- 2. refinement + orientation: one thread per candidate ----------------------------------------------------------------------------
__global__ void __launch_bounds__(128) sift_refine_kernel(SiftPyr p, const SiftCand* cand, const int* ncand, int cand_cap, float contrastThreshold,
                                                         float edgeThreshold, float sigma, SiftKp* kps, int* nkp, int kp_cap)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(*ncand, cand_cap)) return;
    const SiftCand cd = cand[i];
    const int o = cd.o, cw = p.w[o], ch = p.h[o];
    const size_t n = (size_t)cw * ch;
    int layer = cd.layer, r = cd.r, c = cd.c;
    SiftKp kpt;
    if (!sift_adjust(p.dog + p.doff[o], cw, ch, p.nl, o, layer, r, c, contrastThreshold, edgeThreshold, sigma, kpt)) return;
    const float scl_octv = kpt.size * 0.5f / (1 << o);
    const int radius = __float2int_rn(4.5f * scl_octv);
    const float osigma = 1.5f * scl_octv, expf_scale = -1.f / (2.f * osigma * osigma);
    const float* img = p.gauss + p.goff[o] + (size_t)layer * n;
    float temp[SIFT_ORI_BINS + 4], hist[SIFT_ORI_BINS];
    float* th = temp + 2;
    for (int k = 0; k < SIFT_ORI_BINS; k++) th[k] = 0.f;
    for (int dy = -radius; dy <= radius; dy++) {
        const int y = r + dy;
        if (y <= 0 || y >= ch - 1) continue;
        for (int dx = -radius; dx <= radius; dx++) {
            const int x = c + dx;
            if (x <= 0 || x >= cw - 1) continue;
            const float gx = img[(size_t)y * cw + x + 1] - img[(size_t)y * cw + x - 1];
            const float gy = img[(size_t)(y - 1) * cw + x] - img[(size_t)(y + 1) * cw + x];
            const float w = expf((dy * dy + dx * dx) * expf_scale), ori = fast_atan2_deg(gy, gx), mag = sqrtf(gx * gx + gy * gy);
            int bin = __float2int_rn((SIFT_ORI_BINS / 360.f) * ori);
            if (bin >= SIFT_ORI_BINS) bin -= SIFT_ORI_BINS;
            if (bin < 0) bin += SIFT_ORI_BINS;
            th[bin] += w * mag;
        }
    }
    th[-1] = th[SIFT_ORI_BINS - 1]; th[-2] = th[SIFT_ORI_BINS - 2]; th[SIFT_ORI_BINS] = th[0]; th[SIFT_ORI_BINS + 1] = th[1];
    float omax = 0.f;
    for (int k = 0; k < SIFT_ORI_BINS; k++) {
        hist[k] = (th[k - 2] + th[k + 2]) * (1.f / 16.f) + (th[k - 1] + th[k + 1]) * (4.f / 16.f) + th[k] * (6.f / 16.f);
        omax = k == 0 ? hist[0] : fmaxf(omax, hist[k]);
    }
    const float mag_thr = omax * 0.8f;
    for (int j = 0; j < SIFT_ORI_BINS; j++) {
        const int l = j > 0 ? j - 1 : SIFT_ORI_BINS - 1, r2 = j < SIFT_ORI_BINS - 1 ? j + 1 : 0;
        if (hist[j] > hist[l] && hist[j] > hist[r2] && hist[j] >= mag_thr) {
            float bin = j + 0.5f * (hist[l] - hist[r2]) / (hist[l] - 2 * hist[j] + hist[r2]);
            bin = bin < 0 ? SIFT_ORI_BINS + bin : bin >= SIFT_ORI_BINS ? bin - SIFT_ORI_BINS : bin;
            kpt.angle = 360.f - (360.f / SIFT_ORI_BINS) * bin;
            if (fabsf(kpt.angle - 360.f) < 1.1920929e-07f) kpt.angle = 0.f;
            const int slot = atomicAdd(nkp, 1);
            if (slot < kp_cap) kps[slot] = kpt;
        }
    }
}

struct KpLess {      // KeyPoint12_LessThan, features2d/src/keypoint.cpp:253-271 (class_id is always -1)
    bool operator()(const SiftKp& a, const SiftKp& b) const
    {
        if (a.x != b.x) return a.x < b.x;
        if (a.y != b.y) return a.y < b.y;
        if (a.size != b.size) return a.size > b.size;
        if (a.angle != b.angle) return a.angle < b.angle;
        if (a.response != b.response) return a.response > b.response;
        return a.octave > b.octave;
    }
};

}  // namespace

// gauss / dog: device pointers to ONE frame's packed pyramids (layout of b200cv_sift_pyramid_layout); kp_host: 6 floats per keypoint
// (x, y, size, angle, response, octave bits), desc_host: 128 floats per keypoint or null; both host memory.  Synchronises the stream.
int sift_detect_impl(const float* gauss, const float* dog, const int* dims, int n_oct, int nl, double contrastThreshold, double edgeThreshold, double sigma,
                     int first_octave, int nfeatures, const unsigned char* mask_host, size_t mask_step, int mask_w, int mask_h, int max_kp, float* kp_host,
                     float* desc_host, int* n_out, cudaStream_t st)
{
    B200_REQUIRE(gauss && dog && dims && kp_host && n_out && n_oct > 0 && n_oct <= SIFT_MAX_OCT && nl > 0 && nl <= 8 && max_kp > 0, "sift_detect: bad arguments");
    SiftPyr p;
    memset(&p, 0, sizeof(p));
    p.gauss = gauss; p.dog = dog; p.n_oct = n_oct; p.nl = nl;
    unsigned long long go = 0, dofs = 0;
    size_t px_total = 0;
    for (int o = 0; o < n_oct; o++) {
        p.w[o] = dims[2 * o]; p.h[o] = dims[2 * o + 1];
        B200_REQUIRE(p.w[o] > 0 && p.h[o] > 0 && p.h[o] < 65536 + 2 * SIFT_BORDER, "sift_detect: bad octave size");
        p.goff[o] = go; p.doff[o] = dofs;
        const unsigned long long n = (unsigned long long)p.w[o] * p.h[o];
        go += n * (nl + 3); dofs += n * (nl + 2);
        px_total += (size_t)n;
    }
    // candidates are a few per thousand pixels; cap generously, report truncation through the counters
    const int cand_cap = (int)std::min<size_t>(std::max<size_t>(px_total / 8, 4096), (size_t)1 << 24);
    const int kp_cap = std::max(max_kp, 1024) * 2;       // before duplicate removal
    char* scratch = nullptr;
    const size_t cand_bytes = sizeof(SiftCand) * (size_t)cand_cap, kp_bytes = sizeof(SiftKp) * (size_t)kp_cap;
    B200_CUDA(cudaMallocAsync((void**)&scratch, cand_bytes + kp_bytes + 16, st));
    SiftCand* cand = (SiftCand*)scratch;
    SiftKp* kps = (SiftKp*)(scratch + cand_bytes);
    int* counters = (int*)(scratch + cand_bytes + kp_bytes);      // [0] candidates, [1] keypoints
    cudaError_t ce = cudaMemsetAsync(counters, 0, 16, st);
    const float threshold = (float)(int)floor(0.5 * contrastThreshold / nl * 255);
    int launches = 0;
    for (int o = 0; o < n_oct && ce == cudaSuccess; o++) {
        const int iw = p.w[o] - 2 * SIFT_BORDER, ih = p.h[o] - 2 * SIFT_BORDER;
        if (iw <= 0 || ih <= 0) continue;
        const dim3 block(256);
        const dim3 grid(div_up((unsigned)iw, 256), (unsigned)ih, (unsigned)nl);
        sift_extrema_kernel<<<grid, block, 0, st>>>(p, o, threshold, cand, counters, cand_cap);
        launches++;
    }
    {
        const dim3 block(128);
        const dim3 grid(div_up((unsigned)cand_cap, 128));
        sift_refine_kernel<<<grid, block, 0, st>>>(p, cand, counters, cand_cap, (float)contrastThreshold, (float)edgeThreshold, (float)sigma, kps, counters + 1, kp_cap);
        launches++;
    }
    int host_cnt[2] = {0, 0};
    if (ce == cudaSuccess) ce = cudaGetLastError();
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(host_cnt, counters, 8, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    count_launch(launches);
    if (ce != cudaSuccess) { cudaFreeAsync(scratch, st); return cuda_fail(ce, "sift_detect", __FILE__, __LINE__); }
    if (host_cnt[0] > cand_cap || host_cnt[1] > kp_cap) {
        cudaFreeAsync(scratch, st);
        set_error("sift_detect: %d candidates / %d keypoints exceed the buffers (%d / %d): raise max_kp", host_cnt[0], host_cnt[1], cand_cap, kp_cap);
        return B200CV_ERR_BAD_ARG;
    }
    std::vector<SiftKp> hk((size_t)host_cnt[1]);
    if (!hk.empty()) {
        ce = cudaMemcpyAsync(hk.data(), kps, sizeof(SiftKp) * hk.size(), cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        if (ce != cudaSuccess) { cudaFreeAsync(scratch, st); return cuda_fail(ce, "sift_detect (keypoints)", __FILE__, __LINE__); }
        // KeyPointsFilter::removeDuplicatedSorted (keypoint.cpp:273-291), then the first-octave rescaling (sift.dispatch.cpp:548-555)
        std::sort(hk.begin(), hk.end(), KpLess());
        size_t m = 0;
        for (size_t j = 1; j < hk.size(); j++)
            if (hk[m].x != hk[j].x || hk[m].y != hk[j].y || hk[m].size != hk[j].size || hk[m].angle != hk[j].angle) hk[++m] = hk[j];
        hk.resize(m + 1);
        // KeyPointsFilter::retainBest (keypoint.cpp:69-90): everything at least as strong as the nfeatures-th response; the same std:: calls on the
        // same sequence, so the same order comes out
        if (nfeatures > 0 && hk.size() > (size_t)nfeatures) {
            std::nth_element(hk.begin(), hk.begin() + nfeatures - 1, hk.end(), [](const SiftKp& a, const SiftKp& b) { return a.response > b.response; });
            const float ambiguous = hk[nfeatures - 1].response;
            auto new_end = std::partition(hk.begin() + nfeatures, hk.end(), [ambiguous](const SiftKp& k) { return k.response >= ambiguous; });
            hk.resize(new_end - hk.begin());
        }
        if (first_octave < 0) {
            const float scale = 1.f / (float)(1 << -first_octave);
            for (SiftKp& k : hk) { k.octave = (k.octave & ~255) | ((k.octave + first_octave) & 255); k.x *= scale; k.y *= scale; k.size *= scale; }
        }
        // KeyPointsFilter::runByPixelsMask (keypoint.cpp:144-169): drop keypoints whose rounded position has a zero mask byte
        if (mask_host) {
            size_t w = 0;
            for (size_t j = 0; j < hk.size(); j++) {
                const int my = (int)(hk[j].y + 0.5f), mx = (int)(hk[j].x + 0.5f);
                if (my >= 0 && my < mask_h && mx >= 0 && mx < mask_w && mask_host[(size_t)my * mask_step + mx] != 0) hk[w++] = hk[j];
            }
            hk.resize(w);
        }
    }
    *n_out = (int)hk.size();
    const size_t nret = std::min(hk.size(), (size_t)max_kp);
    for (size_t j = 0; j < nret; j++) {
        float* o6 = kp_host + 6 * j;
        o6[0] = hk[j].x; o6[1] = hk[j].y; o6[2] = hk[j].size; o6[3] = hk[j].angle; o6[4] = hk[j].response; memcpy(o6 + 5, &hk[j].octave, 4);
    }
    int rc = B200CV_OK;
#ifndef B200CV_HOST_EMULATION
    if (desc_host && nret) {
        // the sorted keypoints go back up (they fit in the keypoint buffer), descriptors come down
        float* ddesc = nullptr;
        ce = cudaMallocAsync((void**)&ddesc, sizeof(float) * 128 * nret, st);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(kps, hk.data(), sizeof(SiftKp) * nret, cudaMemcpyHostToDevice, st);
        if (ce == cudaSuccess && sift_descriptors_warp(p, first_octave, kps, (int)nret, ddesc, st) != B200CV_OK) ce = cudaErrorUnknown;
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(desc_host, ddesc, sizeof(float) * 128 * nret, cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        if (ddesc) cudaFreeAsync(ddesc, st);
        if (ce != cudaSuccess) rc = cuda_fail(ce, "sift descriptors", __FILE__, __LINE__);
    }
#endif
    cudaFreeAsync(scratch, st);
    return rc;
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_sift_detect_and_compute(const float* gauss, const float* dog, const int* dims, int n_octaves, int n_octave_layers, double contrast_threshold,
                                              double edge_threshold, double sigma, int first_octave, int n_features, const unsigned char* mask,
                                              size_t mask_step, int mask_width, int mask_height, int max_keypoints, float* keypoints, float* descriptors,
                                              int* n_keypoints, void* stream)
{
    return sift_detect_impl(gauss, dog, dims, n_octaves, n_octave_layers, contrast_threshold, edge_threshold, sigma, first_octave, n_features, mask, mask_step,
                            mask_width, mask_height, max_keypoints, keypoints, descriptors, n_keypoints, as_stream(stream));
}
