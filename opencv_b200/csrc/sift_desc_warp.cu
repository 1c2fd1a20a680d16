// sift_desc_warp.cu -- SIFT descriptors of the keypoints sift_detect.cu found.  A WARP owns a keypoint: the (2 r + 1)^2 samples of the patch
// are dealt out to the lanes (a thread per keypoint would be a few thousand threads, each running ~10^5 dependent instructions), and the
// 6 x 6 x 10 tri-linear histogram lives in shared memory.  Float atomics would make the sum depend on the order the lanes happen to arrive
// in (run-to-run differences of +-1 in a descriptor byte); instead every contribution is added as a 64-bit fixed-point integer
// (2^-24 units: integer addition is associative, so the histogram
// is the same whatever the order, and the quantisation -- 6e-8 per contribution against bin totals of 10..1000 -- is below the float
// rounding of the reference's own sequential accumulation).  Same arithmetic otherwise: calcSIFTDescriptor, sift.simd.hpp:709-1035
// (fastAtan2's polynomial, exp, the tri-linear split, clipping at 0.2 |h|, scaling to 512, saturation to bytes).
#include "sift_detect.cuh"

namespace b200cv {

namespace {

constexpr int SD_D = 4, SD_N = 8;
constexpr int SD_HIST = (SD_D + 2) * (SD_D + 2) * (SD_N + 2);      // 360
constexpr float SD_FIX = 16777216.f;                                // 2^24

__global__ void __launch_bounds__(128) sift_descriptor_warp_kernel(SiftPyr p, int first_octave, const SiftKp* kps, int nkp, float* desc)
{
    __shared__ long long s_hist[4][SD_HIST];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q = blockIdx.x * 4 + warp;
    if (q >= nkp) return;                                            // warp-uniform
    enum { d = SD_D, n = SD_N };
    const SiftKp k = kps[q];
    int octave = k.octave & 255;
    const int layer = (k.octave >> 8) & 255;
    octave = octave < 128 ? octave : (-128 | octave);
    const float scale = octave >= 0 ? 1.f / (1 << octave) : (float)(1 << -octave);
    const int oi = octave - first_octave;
    float* out = desc + (size_t)q * 128;
    if (oi < 0 || oi >= p.n_oct || layer > p.nl + 2) { for (int e = lane; e < 128; e += 32) out[e] = 0.f; return; }
    const int cols = p.w[oi], rows = p.h[oi];
    const float* img = p.gauss + p.goff[oi] + (size_t)layer * cols * rows;
    const float size = k.size * scale, ptx = k.x * scale, pty = k.y * scale;
    float ori = 360.f - k.angle;
    if (fabsf(ori - 360.f) < 1.1920929e-07f) ori = 0.f;
    const float scl = size * 0.5f;
    const int px = __float2int_rn(ptx), py = __float2int_rn(pty);
    float cos_t = cosf(ori * (float)(3.1415926535897932384626433832795 / 180)), sin_t = sinf(ori * (float)(3.1415926535897932384626433832795 / 180));
    const float bins_per_rad = n / 360.f, exp_scale = -1.f / (d * d * 0.5f), hist_width = 3.f * scl;
    int radius = __float2int_rn(hist_width * 1.4142135623730951f * (d + 1) * 0.5f);
    radius = min(radius, (int)sqrt((double)cols * cols + (double)rows * rows));
    cos_t /= hist_width; sin_t /= hist_width;
    long long* hist = s_hist[warp];
    for (int i = lane; i < SD_HIST; i += 32) hist[i] = 0;
    __syncwarp();
    const int side = 2 * radius + 1, total = side * side;
    for (int t = lane; t < total; t += 32) {
        const int i = t / side - radius, j = t - (t / side) * side - radius;
        const float c_rot = j * cos_t - i * sin_t, r_rot = j * sin_t + i * cos_t;
        float rbin = r_rot + d / 2 - 0.5f, cbin = c_rot + d / 2 - 0.5f;
        const int r = py + i, c = px + j;
        if (!(rbin > -1 && rbin < d && cbin > -1 && cbin < d && r > 0 && r < rows - 1 && c > 0 && c < cols - 1)) continue;
        const float dx = img[(size_t)r * cols + c + 1] - img[(size_t)r * cols + c - 1];
        const float dy = img[(size_t)(r - 1) * cols + c] - img[(size_t)(r + 1) * cols + c];
        const float w = expf((c_rot * c_rot + r_rot * r_rot) * exp_scale);
        float obin = (fast_atan2_deg(dy, dx) - ori) * bins_per_rad;
        const float mag = sqrtf(dx * dx + dy * dy) * w;
        const int r0 = (int)floorf(rbin), c0 = (int)floorf(cbin);
        int o0 = (int)floorf(obin);
        rbin -= r0; cbin -= c0; obin -= o0;
        if (o0 < 0) o0 += n;
        if (o0 >= n) o0 -= n;
        // tri-linear split: the upper share of each axis is weight * fraction, the lower share the remainder (sift.simd.hpp:864-882)
        const int idx = ((r0 + 1) * (d + 2) + c0 + 1) * (n + 2) + o0;
        const float up_r = mag * rbin;
#pragma unroll
        for (int ri = 0; ri < 2; ri++) {
            const float w_r = ri ? up_r : mag - up_r;
            const float up_c = w_r * cbin;
#pragma unroll
            for (int ci = 0; ci < 2; ci++) {
                const float w_c = ci ? up_c : w_r - up_c;
                const float up_o = w_c * obin;
                unsigned long long* cell = (unsigned long long*)(hist + idx + ri * (d + 2) * (n + 2) + ci * (n + 2));
                atomicAdd(cell, (unsigned long long)__float2ll_rn((w_c - up_o) * SD_FIX));
                atomicAdd(cell + 1, (unsigned long long)__float2ll_rn(up_o * SD_FIX));
            }
        }
    }
    __syncwarp();
    // the 128 entries: lane l holds entries l, l + 32, l + 64, l + 96 (orientation bins 0 and 1 take the circular wrap from bins 8 and 9)
    float v[4];
    float nrm2 = 0;
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int e = lane + 32 * u, cell = e >> 3, ob = e & 7, ci = cell >> 2, cj = cell & 3;
        const int idx = ((ci + 1) * (d + 2) + (cj + 1)) * (n + 2) + ob;
        long long h = hist[idx];
        if (ob < 2) h += hist[idx + n];
        v[u] = (float)h * (1.f / SD_FIX);
        nrm2 += v[u] * v[u];
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) nrm2 += __shfl_xor_sync(0xffffffffu, nrm2, o);
    const float thr = sqrtf(nrm2) * 0.2f;
    nrm2 = 0;
#pragma unroll
    for (int u = 0; u < 4; u++) { v[u] = fminf(v[u], thr); nrm2 += v[u] * v[u]; }
#pragma unroll
    for (int o = 16; o; o >>= 1) nrm2 += __shfl_xor_sync(0xffffffffu, nrm2, o);
    nrm2 = 512.f / fmaxf(sqrtf(nrm2), 1.1920929e-07f);

#pragma unroll
    for (int u = 0; u < 4; u++) out[lane + 32 * u] = (float)sat_u8(__float2int_rn(v[u] * nrm2));
}

}  // namespace

int sift_descriptors_warp(const SiftPyr& p, int first_octave, const SiftKp* kps, int nkp, float* desc, cudaStream_t st)
{
    if (nkp <= 0) return B200CV_OK;
    sift_descriptor_warp_kernel<<<div_up((unsigned)nkp, 4), 128, 0, st>>>(p, first_octave, kps, nkp, desc);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}

}  // namespace b200cv
