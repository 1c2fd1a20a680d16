// matchtemplate_mask.cu -- cv::matchTemplate with a mask, one channel, 8-bit or float images / templates, 8-bit (binarised)
// or float (weight) masks, all six methods.
//
// Reference (matchTemplateMask, templmatch.cpp:762-905): everything becomes float, then up to four cross-correlations through the block DFT:
//   S1 = CC(I, W1), S2 = CC(I^2, M^2), S3 = CC(I, M), S4 = CC(I, M^2);  W1 = T M^2 (SQDIFF / CCORR) or M^2 (T - mu), mu = sum(M T) / sum(M) (CCOEFF)
//   SQDIFF  -2 S1 + S2 + c              c = sum((T M)^2)            NORMED: / sqrt(c S2)
//   CCORR   S1                                                        NORMED: / sqrt(c S2)
//   CCOEFF  S1 - S3 sum(W1) / sum(M)                                  NORMED: / (sqrt(S2 + S3 / sum(M) (S3 sum(M^2) / sum(M) - 2 S4)) |M (T - mu)|)
// Here the four sums are direct, in double, one thread per result element (the weights W1, M, M^2 and the scalars come from a one-thread
// preparation kernel): more accurate than the reference's float DFT, parity by the tolerance its own test uses (1e-3 of the result range).
// A first version: w*h taps per result element through L1, no tiling, no tensor cores -- the unmasked 8-bit numerator has those
// (matchtemplate_tc.cu); masked matching with float weights does not map onto the exact integer MMA.
#include "common.cuh"

namespace b200cv {

namespace {

struct MaskPrep {             // written by the preparation kernel
    double sumM, sumM2, c, sumW1, norm_templx;
};

template <typename TT, typename TM>
__global__ void mt_mask_prep_kernel(Img templ, Img mask, int tw, int th, int coeff, float* w1, float* m, float* m2, MaskPrep* out)
{
    if (blockIdx.x != 0 || threadIdx.x != 0) return;          // a few thousand elements, summed in one fixed order
    double sumM = 0, sumMT = 0, sumM2 = 0, c = 0;
    for (int y = 0; y < th; y++)
        for (int x = 0; x < tw; x++) {
            const float T = (float)templ.row<TT>(0, y)[x];
            float M;
            if constexpr (sizeof(TM) == 1) M = mask.row<TM>(0, y)[x] ? 1.f : 0.f;        // threshold(mask, 0, 1, THRESH_BINARY)
            else M = (float)mask.row<TM>(0, y)[x];
            const int i = y * tw + x;
            m[i] = M; m2[i] = __fmul_rn(M, M);
            sumM += M; sumMT += (double)__fmul_rn(M, T); sumM2 += m2[i];
            const float tm = __fmul_rn(T, M);
            c += (double)tm * tm;
        }
    const float mu = (float)(sumMT / sumM);
    double sumW1 = 0, nt2 = 0;
    for (int y = 0; y < th; y++)
        for (int x = 0; x < tw; x++) {
            const float T = (float)templ.row<TT>(0, y)[x];
            const int i = y * tw + x;
            const float q = __fmul_rn(m[i], T - mu);
            w1[i] = coeff ? __fmul_rn(m[i], q) : __fmul_rn(T, m2[i]);
            sumW1 += w1[i];
            nt2 += (double)q * q;
        }
    out->sumM = sumM; out->sumM2 = sumM2; out->c = c; out->sumW1 = sumW1; out->norm_templx = sqrt(nt2);
}

template <typename TI>
__global__ void __launch_bounds__(256) mt_mask_kernel(Img img, Img res, int ow, int tw, int th, int method, const float* __restrict__ w1,
                                                      const float* __restrict__ m, const float* __restrict__ m2, const MaskPrep* __restrict__ pp)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y, f = blockIdx.z;
    if (x >= ow) return;
    double S1 = 0, S2 = 0, S3 = 0, S4 = 0;
    for (int v = 0; v < th; v++) {
        const TI* row = img.row<TI>(f, y + v) + x;
        for (int u = 0; u < tw; u++) {
            const double I = (double)row[u];
            const int i = v * tw + u;
            S1 += I * w1[i]; S2 += I * I * m2[i]; S3 += I * m[i]; S4 += I * m2[i];
        }
    }
    const MaskPrep p = *pp;
    double r;
    if (method <= 1) { r = -2 * S1 + S2 + p.c; if (method == 1) r /= sqrt(p.c * S2); }
    else if (method <= 3) { r = S1; if (method == 3) r /= sqrt(p.c * S2); }
    else {
        r = S1 - S3 * (p.sumW1 / p.sumM);
        if (method == 5) { const double nimg = S2 + (S3 / p.sumM) * (S3 * (p.sumM2 / p.sumM) - 2 * S4); r /= sqrt(nimg) * p.norm_templx; }
    }
    res.row<float>(f, y)[x] = (float)r;
}

}  // namespace

// image: 8UC1 / 32FC1 (batch allowed); templ: same type, one frame; mask: 8UC1 / 32FC1 of the template's size; result: 32FC1 (W-w+1) x (H-h+1)
int match_template_masked(const b200cvMat* image, const b200cvMat* templ, const b200cvMat* mask, const b200cvMat* result, int method, cudaStream_t st)
{
    B200_REQUIRE(method >= 0 && method <= 5, "bad method");
    B200_REQUIRE(image->type == templ->type, "image/template type mismatch");
    const int u8i = image->type == B200CV_MAKETYPE(B200CV_8U, 1), f32i = image->type == B200CV_MAKETYPE(B200CV_32F, 1);
    const int u8m = mask->type == B200CV_MAKETYPE(B200CV_8U, 1), f32m = mask->type == B200CV_MAKETYPE(B200CV_32F, 1);
    if ((!u8i && !f32i) || (!u8m && !f32m)) return B200CV_NOT_IMPLEMENTED;
    B200_REQUIRE(result->type == B200CV_MAKETYPE(B200CV_32F, 1), "result must be CV_32FC1");
    const int W = image->cols, H = image->rows, w = templ->cols, h = templ->rows;
    B200_REQUIRE(mask->cols == w && mask->rows == h, "the mask must have the template's size");
    if (w > W || h > H || (long long)w * h > (1 << 22)) return B200CV_NOT_IMPLEMENTED;
    const int ow = W - w + 1, oh = H - h + 1;
    B200_REQUIRE(result->cols == ow && result->rows == oh, "result must be (W-w+1) x (H-h+1)");
    Img im = make_img(image), tp = make_img(templ), mk = make_img(mask), rs = make_img(result);
    B200_REQUIRE(im.frames == rs.frames, "image/result batch mismatch");
    if (oh >= 65536 || im.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    const size_t n = (size_t)w * h;
    float* scratch = nullptr;
    B200_CUDA(cudaMallocAsync((void**)&scratch, sizeof(float) * 3 * n + sizeof(MaskPrep) + 16, st));
    float *w1 = scratch, *m = scratch + n, *m2 = scratch + 2 * n;
    MaskPrep* pp = (MaskPrep*)(((uintptr_t)(scratch + 3 * n) + 15) & ~(uintptr_t)15);
    const int coeff = method >= 4;
    {
        const dim3 grid(1), block(1);
        if (u8i && u8m) mt_mask_prep_kernel<uchar, uchar><<<grid, block, 0, st>>>(tp, mk, w, h, coeff, w1, m, m2, pp);
        else if (u8i) mt_mask_prep_kernel<uchar, float><<<grid, block, 0, st>>>(tp, mk, w, h, coeff, w1, m, m2, pp);
        else if (u8m) mt_mask_prep_kernel<float, uchar><<<grid, block, 0, st>>>(tp, mk, w, h, coeff, w1, m, m2, pp);
        else mt_mask_prep_kernel<float, float><<<grid, block, 0, st>>>(tp, mk, w, h, coeff, w1, m, m2, pp);
    }
    {
        const dim3 block(256);
        const dim3 grid(div_up((unsigned)ow, 256), (unsigned)oh, (unsigned)im.frames);
        if (u8i) mt_mask_kernel<uchar><<<grid, block, 0, st>>>(im, rs, ow, w, h, method, w1, m, m2, pp);
        else mt_mask_kernel<float><<<grid, block, 0, st>>>(im, rs, ow, w, h, method, w1, m, m2, pp);
    }
    const cudaError_t e = cudaGetLastError();
    count_launch(2);
    cudaFreeAsync(scratch, st);
    if (e != cudaSuccess) return cuda_fail(e, "kernel launch", __FILE__, __LINE__);
    return B200CV_OK;
}

}  // namespace b200cv

using namespace b200cv;

extern "C" int b200cv_match_template_masked(const b200cvMat* image, const b200cvMat* templ, const b200cvMat* mask, const b200cvMat* result, int method,
                                            void* stream)
{
    int rc;
    if ((rc = check_mat(image, "image")) || (rc = check_mat(templ, "templ")) || (rc = check_mat(mask, "mask")) || (rc = check_mat(result, "result"))) return rc;
    return match_template_masked(image, templ, mask, result, method, as_stream(stream));
}
