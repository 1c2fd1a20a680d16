// sift.cu -- SIFT scale space: initial image, Gaussian pyramid and difference-of-Gaussians pyramid.
//
// Reference (modules/features2d/src/sift.dispatch.cpp): createInitialImage :176-221 (u8 -> f32, optional 2x upsample through
// warpAffine(INTER_LINEAR | WARP_INVERSE_MAP, BORDER_REFLECT), GaussianBlur(sig_diff)), buildGaussianPyramid :224-263
// (octave base = INTER_NEAREST half-size of layer nOctaveLayers of the previous octave; layer i = GaussianBlur(layer i-1,
// Size(), sig[i])), buildDoGPyramid :266-310 (DoG[i] = G[i+1] - G[i]).  On the CPU the 66 blurs of a 4K frame run on the
// single-threaded FilterEngine.
//
// Here the pyramid of a whole batch of frames is a fixed launch sequence on one stream: every step is one of this
// library's kernels over all frames at once (grid z = frame), and each DoG level is produced by the blur kernel that
// writes its minuend (the subtrahend is the blur's own input, already in shared memory) -- no separate subtract pass and
// no re-read of either Gaussian level.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "common.cuh"
#include "host_tables.h"

namespace b200cv {

int gaussian_blur_impl(const b200cvMat* src, const b200cvMat* dst, int kw, int kh, double sigma1, double sigma2, int border, void* stream,
                       const b200cvMat* dog);

__global__ void __launch_bounds__(256) u8_to_f32_kernel(Img src, Img dst)
{
    const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    if (x < src.cols) dst.row<float>(f, y)[x] = (float)src.row<uchar>(f, y)[x];
}

// createInitialImage's precise 2x upscale, fused with the u8 -> f32 conversion: warpAffine(H = diag(0.5, 0.5), INTER_LINEAR | WARP_INVERSE_MAP,
// BORDER_REFLECT) of the float image (sift.dispatch.cpp:196-202).  In the reference's fixed-point coordinates X = (16 + 512 x) >> 5 = 16 x
// (hal::warpAffine, imgwarp.cpp:2673-2700): source column x >> 1, 5-bit fraction 16 (x & 1), the same in y -- the four bilinear table entries
// (1,0,0,0), (.5,.5,0,0), (.5,0,.5,0), (.25,.25,.25,.25) -- and remapBilinear's float sum ((v0 w0 + v1 w1) + v2 w2) + v3 w3 (imgwarp.cpp:675-904),
// written out term by term so that the result is the general warp kernel's bit for bit (tests/test_gpu_features.py).  One thread = two source
// columns of one source row = a 4 x 2 block of the doubled image: 16-byte stores, every source byte fetched through L1.
__device__ __forceinline__ float sift_bilin(float v0, float v1, float v2, float v3, float w0, float w1, float w2, float w3)
{
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(v0, w0), __fmul_rn(v1, w1)), __fmul_rn(v2, w2)), __fmul_rn(v3, w3));
}
__global__ void __launch_bounds__(256) sift_upsample2x_kernel(Img src, Img dst)
{
    const int i0 = (blockIdx.x * 256 + threadIdx.x) * 2, j = blockIdx.y, f = blockIdx.z;
    const int W = src.cols, H = src.rows;
    if (i0 >= W) return;
    const uchar* r0 = src.row<uchar>(f, j);
    const uchar* r1 = src.row<uchar>(f, j + 1 < H ? j + 1 : H - 1);           // BORDER_REFLECT: row H -> H - 1
    const int i1 = i0 + 1 < W ? i0 + 1 : W - 1, i2 = i0 + 2 < W ? i0 + 2 : W - 1;   // column W -> W - 1
    const float a0 = (float)r0[i0], a1 = (float)r0[i1], a2 = (float)r0[i2];
    const float b0 = (float)r1[i0], b1 = (float)r1[i1], b2 = (float)r1[i2];
    float e[4], o[4];      // doubled rows 2j and 2j + 1, columns 2 i0 .. 2 i0 + 3
    e[0] = sift_bilin(a0, a1, b0, b1, 1.f, 0.f, 0.f, 0.f);       e[1] = sift_bilin(a0, a1, b0, b1, .5f, .5f, 0.f, 0.f);
    e[2] = sift_bilin(a1, a2, b1, b2, 1.f, 0.f, 0.f, 0.f);       e[3] = sift_bilin(a1, a2, b1, b2, .5f, .5f, 0.f, 0.f);
    o[0] = sift_bilin(a0, a1, b0, b1, .5f, 0.f, .5f, 0.f);       o[1] = sift_bilin(a0, a1, b0, b1, .25f, .25f, .25f, .25f);
    o[2] = sift_bilin(a1, a2, b1, b2, .5f, 0.f, .5f, 0.f);       o[3] = sift_bilin(a1, a2, b1, b2, .25f, .25f, .25f, .25f);
    float* d0 = dst.row<float>(f, 2 * j) + 2 * i0;
    float* d1 = dst.row<float>(f, 2 * j + 1) + 2 * i0;
    if (i0 + 1 < W && (((uintptr_t)d0 | (uintptr_t)d1) & 15) == 0) {
        *(float4*)d0 = make_float4(e[0], e[1], e[2], e[3]);
        *(float4*)d1 = make_float4(o[0], o[1], o[2], o[3]);
    } else {
        const int n = i0 + 1 < W ? 4 : 2;
        for (int c = 0; c < n; c++) { d0[c] = e[c]; d1[c] = o[c]; }
    }
}

// ---- the small octaves in ONE launch -------------------------------------------------------------------------------------------------------
// From the first octave whose levels fit shared memory (w * h <= SS_CAP floats; 60 x 33 and below for a doubled 4K frame) the rest of the
// pyramid is one kernel, one CTA per frame: base = INTER_NEAREST half-size of the previous octave's layer nOctaveLayers (resize.cpp:1131-1135
// index arithmetic: min(floor(x * (1 / (dw / sw))), sw - 1) in double), then layer after layer the separable Gaussian in the operation order
// of the library's float filter kernels (rows: fma in tap order from 0; columns: fma(ky[c], S[c], 0) then fma(ky[c+k], S[c+k] + S[c-k], .),
// BORDER_REFLECT_101 by index), each DoG level with the blur that writes its minuend.  As separate launches these ~6 x 4 tiny dependent
// kernels are a chain of launches, each far below one wave.
constexpr int SS_CAP = 3072;          // floats per level buffer
constexpr int SS_MAXO = 8, SS_MAXL = 10, SS_MAXK = 33;
struct SiftSmallParams {
    int no, n_layers;
    int w[SS_MAXO], h[SS_MAXO];
    unsigned long long goff[SS_MAXO], doff[SS_MAXO];      // element offsets of the octave's first Gaussian / DoG level inside a frame's pyramid
    double ifx[SS_MAXO], ify[SS_MAXO];                    // NEAREST index scale from the previous octave
    int pw, ph; unsigned long long poff;                  // the octave before the first small one: size and offset of its layer n_layers
    int ks[SS_MAXL];
    float taps[SS_MAXL][SS_MAXK];
};

__global__ void __launch_bounds__(256) sift_small_octaves_kernel(float* gauss, size_t gframe, float* dog, size_t dframe, const __grid_constant__ SiftSmallParams p)
{
    __shared__ float s_a[SS_CAP], s_b[SS_CAP], s_mid[SS_CAP], s_next[SS_CAP / 4 + 64];
    const int f = blockIdx.x, tid = threadIdx.x;
    float* G = gauss + (size_t)f * gframe;
    float* D = dog ? dog + (size_t)f * dframe : nullptr;
    float* A = s_a; float* B = s_b;
    for (int o = 0; o < p.no; o++) {
        const int w = p.w[o], h = p.h[o], n = w * h;
        // ---- octave base ----
        if (o == 0) {
            const float* prev = G + p.poff;
            for (int idx = tid; idx < n; idx += 256) {
                const int y = idx / w, x = idx - y * w;
                const int sy = min((int)floor(__dmul_rn((double)y, p.ify[0])), p.ph - 1), sx = min((int)floor(__dmul_rn((double)x, p.ifx[0])), p.pw - 1);
                A[idx] = prev[(size_t)sy * p.pw + sx];
            }
        } else {
            for (int idx = tid; idx < n; idx += 256) A[idx] = s_next[idx];
        }
        __syncthreads();
        for (int idx = tid; idx < n; idx += 256) G[p.goff[o] + idx] = A[idx];
        // ---- layers 1 .. n_layers + 2 ----
        for (int i = 1; i < p.n_layers + 3; i++) {
            const int K = p.ks[i], RB = K / 2;
            const float* t = p.taps[i];
            for (int idx = tid; idx < n; idx += 256) {
                const int y = idx / w, x = idx - y * w;
                const float* row = A + y * w;
                float acc = 0.f;
                if (x >= RB && x + RB < w) {
                    for (int k = 0; k < K; k++) acc = fmaf(row[x - RB + k], t[k], acc);
                } else {
                    for (int k = 0; k < K; k++) acc = fmaf(row[border_interpolate(x - RB + k, w, B200CV_BORDER_REFLECT_101)], t[k], acc);
                }
                s_mid[idx] = acc;
            }
            __syncthreads();
            float* Gl = G + p.goff[o] + (size_t)i * n;
            float* Dl = D ? D + p.doff[o] + (size_t)(i - 1) * n : nullptr;
            for (int idx = tid; idx < n; idx += 256) {
                const int y = idx / w, x = idx - y * w;
                float acc = fmaf(t[RB], s_mid[idx], 0.f);
                if (y >= RB && y + RB < h) {
                    for (int k = 1; k <= RB; k++) acc = fmaf(t[RB + k], __fadd_rn(s_mid[idx + k * w], s_mid[idx - k * w]), acc);
                } else {
                    for (int k = 1; k <= RB; k++)
                        acc = fmaf(t[RB + k], __fadd_rn(s_mid[border_interpolate(y + k, h, B200CV_BORDER_REFLECT_101) * w + x],
                                                         s_mid[border_interpolate(y - k, h, B200CV_BORDER_REFLECT_101) * w + x]), acc);
                }
                B[idx] = acc;
                Gl[idx] = acc;
                if (Dl) Dl[idx] = __fsub_rn(acc, A[idx]);
            }
            __syncthreads();
            if (i == p.n_layers && o + 1 < p.no) {
                // the next octave's base: NEAREST half-size of this layer
                const int nw = p.w[o + 1], nh = p.h[o + 1];
                for (int idx = tid; idx < nw * nh; idx += 256) {
                    const int y = idx / nw, x = idx - y * nw;
                    const int sy = min((int)floor(__dmul_rn((double)y, p.ify[o + 1])), h - 1), sx = min((int)floor(__dmul_rn((double)x, p.ifx[o + 1])), w - 1);
                    s_next[idx] = B[sy * w + sx];
                }
            }
            float* tmpp = A; A = B; B = tmpp;
        }
        __syncthreads();
    }
}

static int octave_count(int base_w, int base_h, int first_octave)
{
    // sift.dispatch.cpp:538
    return (int)lrint(std::log((double)(base_w < base_h ? base_w : base_h)) / std::log(2.) - 2) - first_octave;
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_sift_pyramid_layout(int width, int height, int n_layers, int upscale, int* n_octaves, size_t* gauss_elems,
                                          size_t* dog_elems, int* dims)
{
    B200_REQUIRE(width > 0 && height > 0 && n_layers > 0, "bad arguments");
    int bw = upscale ? width * 2 : width, bh = upscale ? height * 2 : height;
    int no = octave_count(bw, bh, upscale ? -1 : 0);
    B200_REQUIRE(no > 0, "image too small for a SIFT pyramid");
    size_t ge = 0, de = 0;
    int cw = bw, ch = bh;
    for (int o = 0; o < no; o++) {
        if (dims) { dims[2 * o] = cw; dims[2 * o + 1] = ch; }
        ge += (size_t)cw * ch * (n_layers + 3);
        de += (size_t)cw * ch * (n_layers + 2);
        cw /= 2; ch /= 2;
    }
    if (n_octaves) *n_octaves = no;
    if (gauss_elems) *gauss_elems = ge;
    if (dog_elems) *dog_elems = de;
    return B200CV_OK;
}

extern "C" int b200cv_sift_pyramid(const b200cvMat* src, int n_layers, double sigma, int upscale, float* gauss, size_t gauss_frame_elems,
                                   float* dog, size_t dog_frame_elems, void* stream)
{
    int rc;
    if ((rc = check_mat(src, "src"))) return rc;
    B200_REQUIRE(src->type == B200CV_MAKETYPE(B200CV_8U, 1), "SIFT pyramid input must be CV_8UC1");
    B200_REQUIRE(gauss && n_layers > 0 && n_layers <= 8, "bad arguments");
    const int W = src->cols, H = src->rows, frames = src->frames > 1 ? src->frames : 1;
    int no; size_t ge, de;
    std::vector<int> dims(64);
    if ((rc = b200cv_sift_pyramid_layout(W, H, n_layers, upscale, &no, &ge, &de, dims.data()))) return rc;
    B200_REQUIRE(gauss_frame_elems >= ge && (!dog || dog_frame_elems >= de), "output buffers too small");
    cudaStream_t st = as_stream(stream);
    const int F32 = B200CV_MAKETYPE(B200CV_32F, 1);
    auto level = [&](float* base, size_t frame_elems, size_t off, int w, int h) {
        b200cvMat m = {base + off, (size_t)w * 4, w, h, F32, frames, frame_elems * 4};
        return m;
    };

    // ---- createInitialImage ----
    float* tmp = nullptr;   // gray_fpt (W x H) followed by dbl (2W x 2H), per frame
    const size_t gray_elems = (size_t)W * H, dbl_elems = upscale ? gray_elems * 4 : 0;
    const size_t tmp_frame = (gray_elems + dbl_elems + 3) & ~(size_t)3;
    B200_CUDA(cudaMallocAsync(&tmp, tmp_frame * frames * sizeof(float), st));
    b200cvMat gray = level(tmp, tmp_frame, 0, W, H);
    const bool fused_upscale = upscale == 1 && !getenv("B200CV_SIFT_UPSCALE_WARP");       // the switch: the general warpAffine kernel (parity test)
    if (!fused_upscale) {
        Img s = make_img(src), d = make_img(&gray);
        u8_to_f32_kernel<<<dim3(div_up((unsigned)W, 256), H, frames), 256, 0, st>>>(s, d);
        count_launch();
    }
    const float fsigma = (float)sigma;
    b200cvMat g00 = level(gauss, gauss_frame_elems, 0, dims[0], dims[1]);
    if (upscale) {
        float sig_diff = sqrtf(fmaxf(fsigma * fsigma - 0.5f * 0.5f * 4, 0.01f));
        b200cvMat dbl = level(tmp, tmp_frame, gray_elems, 2 * W, 2 * H);
        const double Mh[6] = {0.5, 0, 0, 0, 0.5, 0};
        // upscale == 2: SIFT::create's default, enable_precise_upscale = false -> cv::resize(INTER_LINEAR) (sift.dispatch.cpp:203-208)
        if (upscale == 2) rc = b200cv_resize(&gray, &dbl, B200CV_INTER_LINEAR, stream);
        else if (fused_upscale) {
            sift_upsample2x_kernel<<<dim3(div_up((unsigned)(W + 1) / 2, 256), H, frames), 256, 0, st>>>(make_img(src), make_img(&dbl));
            count_launch();
            if (cudaGetLastError() != cudaSuccess) rc = B200CV_ERR_CUDA;
        }
        else rc = b200cv_warp_affine(&gray, &dbl, Mh, B200CV_INTER_LINEAR | B200CV_WARP_INVERSE_MAP, B200CV_BORDER_REFLECT, nullptr, stream);
        if (!rc) rc = gaussian_blur_impl(&dbl, &g00, 0, 0, sig_diff, sig_diff, B200CV_BORDER_REFLECT_101, stream, nullptr);
    } else {
        float sig_diff = sqrtf(fmaxf(fsigma * fsigma - 0.5f * 0.5f, 0.01f));
        rc = gaussian_blur_impl(&gray, &g00, 0, 0, sig_diff, sig_diff, B200CV_BORDER_REFLECT_101, stream, nullptr);
    }
    if (rc) { cudaFreeAsync(tmp, st); return rc; }

    // ---- buildGaussianPyramid + buildDoGPyramid ----
    std::vector<double> sig(n_layers + 3);
    sig[0] = sigma;
    const double k = std::pow(2., 1. / n_layers);
    for (int i = 1; i < n_layers + 3; i++) {
        double sig_prev = std::pow(k, (double)(i - 1)) * sigma;
        double sig_total = sig_prev * k;
        sig[i] = std::sqrt(sig_total * sig_total - sig_prev * sig_prev);
    }
    // the first octave (>= 1) from which every level fits the small-octave kernel's shared memory
    int o_small = no;
    if (!getenv("B200CV_SIFT_NO_SMALL_OCTAVES") && n_layers + 3 <= SS_MAXL) {
        for (int o = no - 1; o >= 1 && (size_t)dims[2 * o] * dims[2 * o + 1] <= (size_t)SS_CAP; o--) o_small = o;
        if (no - o_small > SS_MAXO) o_small = no - SS_MAXO;
        // the next octave's base lives in a quarter-size buffer
        for (int o = o_small; o + 1 < no; o++) if ((size_t)dims[2 * (o + 1)] * dims[2 * (o + 1) + 1] > (size_t)SS_CAP / 4 + 64) { o_small = no; break; }
    }
    size_t goff = 0, doff = 0;
    for (int o = 0; o < no && !rc; o++) {
        const int w = dims[2 * o], h = dims[2 * o + 1];
        const size_t n = (size_t)w * h;
        if (o == o_small) {
            static thread_local SiftSmallParams sp;
            memset(&sp, 0, sizeof(sp));
            sp.no = no - o_small; sp.n_layers = n_layers;
            sp.pw = dims[2 * (o - 1)]; sp.ph = dims[2 * (o - 1) + 1];
            sp.poff = goff - (size_t)sp.pw * sp.ph * (n_layers + 3) + (size_t)sp.pw * sp.ph * n_layers;
            bool ok = true;
            for (int i = 1; i < n_layers + 3 && ok; i++) {
                const int ks = gaussian_auto_ksize(sig[i], false);
                if (ks > SS_MAXK || !(ks & 1)) { ok = false; break; }
                std::vector<double> dk;
                gaussian_kernel_bitexact(ks, sig[i], dk);
                sp.ks[i] = ks;
                for (int t = 0; t < ks; t++) sp.taps[i][t] = (float)dk[t];
            }
            size_t go = goff, dO = doff;
            for (int q = 0; q < sp.no; q++) {
                const int ow = dims[2 * (o + q)], oh = dims[2 * (o + q) + 1], qw = dims[2 * (o + q - 1)], qh = dims[2 * (o + q - 1) + 1];
                sp.w[q] = ow; sp.h[q] = oh; sp.goff[q] = go; sp.doff[q] = dO;
                sp.ifx[q] = 1. / ((double)ow / qw); sp.ify[q] = 1. / ((double)oh / qh);
                go += (size_t)ow * oh * (n_layers + 3); dO += (size_t)ow * oh * (n_layers + 2);
            }
            if (ok) {
                sift_small_octaves_kernel<<<frames, 256, 0, st>>>(gauss, gauss_frame_elems, dog, dog_frame_elems, sp);
                count_launch();
                if (cudaGetLastError() != cudaSuccess) rc = B200CV_ERR_CUDA;
                break;
            }
        }
        if (o > 0) {
            const int pw = dims[2 * (o - 1)], ph = dims[2 * (o - 1) + 1];
            b200cvMat prev = level(gauss, gauss_frame_elems, goff - (size_t)pw * ph * (n_layers + 3) + (size_t)pw * ph * n_layers, pw, ph);
            b200cvMat base = level(gauss, gauss_frame_elems, goff, w, h);
            rc = b200cv_resize(&prev, &base, B200CV_INTER_NEAREST, stream);
        }
        for (int i = 1; i < n_layers + 3 && !rc; i++) {
            b200cvMat a = level(gauss, gauss_frame_elems, goff + (size_t)(i - 1) * n, w, h);
            b200cvMat b = level(gauss, gauss_frame_elems, goff + (size_t)i * n, w, h);
            b200cvMat dg;
            if (dog) dg = level(dog, dog_frame_elems, doff + (size_t)(i - 1) * n, w, h);
            rc = gaussian_blur_impl(&a, &b, 0, 0, sig[i], sig[i], B200CV_BORDER_REFLECT_101, stream, dog ? &dg : nullptr);
        }
        goff += n * (n_layers + 3);
        doff += n * (n_layers + 2);
    }
    cudaFreeAsync(tmp, st);
    return rc;
}
