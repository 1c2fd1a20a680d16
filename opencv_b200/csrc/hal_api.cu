// hal_api.cu -- host-pointer entry points: the cv_hal_* replacement functions and the batched host pipeline.
// No arithmetic here: upload, call the device API of b200cv.h, download.
#include <functional>
#include <vector>
#include "common.cuh"
#include "../../include/b200cv_hal.h"

namespace b200cv {

constexpr int NPIPE = 3;                            // host pipeline streams
constexpr size_t CHUNK_BYTES = (size_t)32 << 20;    // upload + download bytes per chunk of frames (at least one frame per chunk)

struct HostCtx {                      // one per host thread: OpenCV calls HAL functions concurrently from many threads
    cudaStream_t st[NPIPE] = {};
    void* dbuf[NPIPE][2] = {};
    size_t cap[NPIPE][2] = {};
    void* daux = nullptr; size_t caux = 0;
    ~HostCtx()
    {
        for (int i = 0; i < NPIPE; i++) {
            for (int j = 0; j < 2; j++) if (dbuf[i][j]) cudaFree(dbuf[i][j]);
            if (st[i]) cudaStreamDestroy(st[i]);
        }
        if (daux) cudaFree(daux);
    }
};
static thread_local HostCtx g_ctx;

static int ensure(void** p, size_t* cap, size_t bytes)
{
    if (*cap >= bytes) return B200CV_OK;
    if (*p) { B200_CUDA(cudaFree(*p)); *p = nullptr; *cap = 0; }
    size_t want = bytes + bytes / 4;
    B200_CUDA(cudaMalloc(p, want));
    *cap = want;
    return B200CV_OK;
}

static inline size_t pitch_of(const b200cvMat* m) { return ((size_t)m->cols * elem_size(m->type) + 255) & ~(size_t)255; }

void configure_mem_pool();     // runtime.cu

typedef std::function<int(const b200cvMat*, const b200cvMat*, void*)> DevOp;

// Generic pipeline: src/dst are HOST descriptors (batches allowed); frames flow in chunks through NPIPE streams.
static int host_pipeline(const b200cvMat* hsrc, const b200cvMat* hdst, const DevOp& op)
{
    int rc;
    configure_mem_pool();
    if ((rc = check_mat(hsrc, "src")) || (rc = check_mat(hdst, "dst"))) return rc;
    const int frames = hsrc->frames > 1 ? hsrc->frames : 1;
    B200_REQUIRE((hdst->frames > 1 ? hdst->frames : 1) == frames, "src/dst batch mismatch");
    const size_t sp = pitch_of(hsrc), dp = pitch_of(hdst);
    const size_t sfb = sp * hsrc->rows, dfb = dp * hdst->rows;
    // chunk so that a chunk is ~>= 32 MB of traffic but at least 1 frame; single frames use one stream
    int chunk = (int)std::max<size_t>(1, CHUNK_BYTES / std::max<size_t>(1, sfb + dfb));
    if (chunk > frames) chunk = frames;
    HostCtx& c = g_ctx;
    const int nchunks = (frames + chunk - 1) / chunk;
    const int npipe = nchunks < NPIPE ? nchunks : NPIPE;
    for (int i = 0; i < npipe; i++) {
        if (!c.st[i]) B200_CUDA(cudaStreamCreateWithFlags(&c.st[i], cudaStreamNonBlocking));
        if ((rc = ensure(&c.dbuf[i][0], &c.cap[i][0], sfb * chunk)) || (rc = ensure(&c.dbuf[i][1], &c.cap[i][1], dfb * chunk))) return rc;
    }
    const size_t swb = (size_t)hsrc->cols * elem_size(hsrc->type), dwb = (size_t)hdst->cols * elem_size(hdst->type);
    for (int ci = 0; ci < nchunks; ci++) {
        const int i = ci % npipe, f0 = ci * chunk, n = std::min(chunk, frames - f0);
        cudaStream_t st = c.st[i];
        const char* hs = (const char*)hsrc->data + (size_t)f0 * hsrc->frame_step;
        char* hd = (char*)hdst->data + (size_t)f0 * hdst->frame_step;
        const bool packed_s = hsrc->frame_step == hsrc->step * (size_t)hsrc->rows || n == 1;
        const bool packed_d = hdst->frame_step == hdst->step * (size_t)hdst->rows || n == 1;
        // identical pitches on both sides (e.g. 3840-byte rows): one linear DMA instead of a row-by-row 2-D copy
        if (packed_s && hsrc->step == sp) B200_CUDA(cudaMemcpyAsync(c.dbuf[i][0], hs, sfb * n, cudaMemcpyHostToDevice, st));
        else if (packed_s) B200_CUDA(cudaMemcpy2DAsync(c.dbuf[i][0], sp, hs, hsrc->step, swb, (size_t)hsrc->rows * n, cudaMemcpyHostToDevice, st));
        else for (int f = 0; f < n; f++)
            B200_CUDA(cudaMemcpy2DAsync((char*)c.dbuf[i][0] + f * sfb, sp, hs + (size_t)f * hsrc->frame_step, hsrc->step, swb, hsrc->rows, cudaMemcpyHostToDevice, st));
        b200cvMat ds = {c.dbuf[i][0], sp, hsrc->cols, hsrc->rows, hsrc->type, n, sfb};
        b200cvMat dd = {c.dbuf[i][1], dp, hdst->cols, hdst->rows, hdst->type, n, dfb};
        if ((rc = op(&ds, &dd, (void*)st))) { for (int k = 0; k < npipe; k++) cudaStreamSynchronize(c.st[k]); return rc; }
        if (packed_d && hdst->step == dp) B200_CUDA(cudaMemcpyAsync(hd, c.dbuf[i][1], dfb * n, cudaMemcpyDeviceToHost, st));
        else if (packed_d) B200_CUDA(cudaMemcpy2DAsync(hd, hdst->step, c.dbuf[i][1], dp, dwb, (size_t)hdst->rows * n, cudaMemcpyDeviceToHost, st));
        else for (int f = 0; f < n; f++)
            B200_CUDA(cudaMemcpy2DAsync(hd + (size_t)f * hdst->frame_step, hdst->step, (char*)c.dbuf[i][1] + f * dfb, dp, dwb, hdst->rows, cudaMemcpyDeviceToHost, st));
    }
    for (int i = 0; i < npipe; i++) B200_CUDA(cudaStreamSynchronize(c.st[i]));
    return B200CV_OK;
}

// ROI of a larger cv::Mat (row a5 of the scope table: FilterEngine's wholeSize / ofs, filterengine.hpp:68-246; HAL arguments
// full_width / full_height / offset_x / offset_y, hal_replacement.hpp:125, and margin_*, :1146): the pixels around the ROI are REAL and the
// border rule only applies at the edges of the parent image.  A filter with reach (l, t, r, b) needs at most that many parent pixels on each
// side: upload the ROI extended by min(reach, available margin), run the same device op on the extended image and download the ROI part.
// Where the extension was clipped by the parent's edge the extended image's edge IS the parent's edge (the border rule lands where the
// reference applies it); where it was not, no output pixel of the ROI reaches the artificial edge.  One frame (what the HAL passes).
static int host_roi_call(const b200cvMat* hsrc, const b200cvMat* hdst, int l, int t, int r, int b, const DevOp& op)
{
    int rc;
    configure_mem_pool();
    if ((rc = check_mat(hsrc, "src")) || (rc = check_mat(hdst, "dst"))) return rc;
    B200_REQUIRE(hsrc->frames <= 1 && hdst->frames <= 1, "ROI context is a single-frame path");
    B200_REQUIRE(hsrc->cols == hdst->cols && hsrc->rows == hdst->rows, "ROI context: src/dst size mismatch");
    const size_t es_s = elem_size(hsrc->type), es_d = elem_size(hdst->type);
    b200cvMat es = *hsrc, ed = *hdst;
    es.cols += l + r; es.rows += t + b; ed.cols = es.cols; ed.rows = es.rows;
    const char* hs = (const char*)hsrc->data - (size_t)t * hsrc->step - (size_t)l * es_s;
    const size_t sp = pitch_of(&es), dp = pitch_of(&ed);
    HostCtx& c = g_ctx;
    if (!c.st[0]) B200_CUDA(cudaStreamCreateWithFlags(&c.st[0], cudaStreamNonBlocking));
    if ((rc = ensure(&c.dbuf[0][0], &c.cap[0][0], sp * es.rows)) || (rc = ensure(&c.dbuf[0][1], &c.cap[0][1], dp * ed.rows))) return rc;
    cudaStream_t st = c.st[0];
    B200_CUDA(cudaMemcpy2DAsync(c.dbuf[0][0], sp, hs, hsrc->step, (size_t)es.cols * es_s, es.rows, cudaMemcpyHostToDevice, st));
    b200cvMat ds = {c.dbuf[0][0], sp, es.cols, es.rows, hsrc->type, 1, 0};
    b200cvMat dd = {c.dbuf[0][1], dp, ed.cols, ed.rows, hdst->type, 1, 0};
    if ((rc = op(&ds, &dd, (void*)st))) { cudaStreamSynchronize(st); return rc; }
    B200_CUDA(cudaMemcpy2DAsync(hdst->data, hdst->step, (const char*)c.dbuf[0][1] + (size_t)t * dp + (size_t)l * es_d, dp, (size_t)hdst->cols * es_d, hdst->rows,
                                cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200CV_OK;
}

// how much of the filter's reach the parent image can supply on each side; all zero -> the plain pipeline.  BORDER_ISOLATED: the ROI is the image.
struct RoiExt { int l, t, r, b; bool any() const { return (l | t | r | b) != 0; } };
static inline RoiExt roi_ext(size_t ml, size_t mt, size_t mr, size_t mb, int rl, int rt, int rr, int rb, int border)
{
    RoiExt e = {0, 0, 0, 0};
    if (border & B200CV_BORDER_ISOLATED) return e;
    e.l = (int)std::min<size_t>(ml, (size_t)std::max(rl, 0)); e.t = (int)std::min<size_t>(mt, (size_t)std::max(rt, 0));
    e.r = (int)std::min<size_t>(mr, (size_t)std::max(rr, 0)); e.b = (int)std::min<size_t>(mb, (size_t)std::max(rb, 0));
    return e;
}

static inline b200cvMat hmat(const void* p, size_t step, int w, int h, int type)
{
    b200cvMat m = {const_cast<void*>(p), step, w, h, type, 1, 0};
    return m;
}

struct FilterCtxImpl {
    int separable;
    std::vector<float> kx, ky, k2d;
    int kw, kh, ax, ay, src_type, dst_type, border;
    double delta;
};

static bool taps_to_float(const uchar* data, size_t step, int type, int w, int h, std::vector<float>& out)
{
    out.resize((size_t)w * h);
    const int depth = B200CV_DEPTH(type);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uchar* p = data + (size_t)y * step;
            if (depth == B200CV_32F) out[(size_t)y * w + x] = ((const float*)p)[x];
            else if (depth == 6) out[(size_t)y * w + x] = (float)((const double*)p)[x];
            else if (depth == 4) out[(size_t)y * w + x] = (float)((const int*)p)[x];
            else return false;
        }
    return true;
}

// matchTemplate over host frames with the template ALREADY on the device (batch.cu: the template arrives by ncclBroadcast)
int host_match_template_dev(const b200cvMat* image, const b200cvMat* dtempl, const b200cvMat* result, int method)
{
    return host_pipeline(image, result, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_match_template(a, dtempl, b, method, st); });
}

}  // namespace b200cv

using namespace b200cv;

// ---- batched host API -----------------------------------------------------------------------------------------------------
extern "C" int b200cv_host_gaussian_blur(const b200cvMat* s, const b200cvMat* d, int kw, int kh, double sx, double sy, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_gaussian_blur(a, b, kw, kh, sx, sy, border, st); }); }
extern "C" int b200cv_host_sep_filter2d(const b200cvMat* s, const b200cvMat* d, const float* kx, int nx, const float* ky, int ny, int ax, int ay, double delta, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_sep_filter2d(a, b, kx, nx, ky, ny, ax, ay, delta, border, st); }); }
extern "C" int b200cv_host_filter2d(const b200cvMat* s, const b200cvMat* d, const float* k, int kw, int kh, int ax, int ay, double delta, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_filter2d(a, b, k, kw, kh, ax, ay, delta, border, st); }); }
extern "C" int b200cv_host_sobel(const b200cvMat* s, const b200cvMat* d, int dx, int dy, int ksize, double scale, double delta, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_sobel(a, b, dx, dy, ksize, scale, delta, border, st); }); }
extern "C" int b200cv_host_laplacian(const b200cvMat* s, const b200cvMat* d, int ksize, double scale, double delta, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_laplacian(a, b, ksize, scale, delta, border, st); }); }
extern "C" int b200cv_host_box_filter(const b200cvMat* s, const b200cvMat* d, int kw, int kh, int ax, int ay, int normalize, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_box_filter(a, b, kw, kh, ax, ay, normalize, border, st); }); }
extern "C" int b200cv_host_resize(const b200cvMat* s, const b200cvMat* d, int interp)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_resize(a, b, interp, st); }); }
extern "C" int b200cv_host_resize_scaled(const b200cvMat* s, const b200cvMat* d, int interp, double fx, double fy)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_resize_scaled(a, b, interp, fx, fy, st); }); }
// BORDER_TRANSPARENT keeps destination pixels: the host path would have to upload the destination too -- declined (the caller's CPU path runs)
extern "C" int b200cv_host_warp_affine(const b200cvMat* s, const b200cvMat* d, const double* M, int flags, int border, const double* bv)
{ if ((border & ~B200CV_BORDER_ISOLATED) == B200CV_BORDER_TRANSPARENT) return B200CV_NOT_IMPLEMENTED;
  return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_warp_affine(a, b, M, flags, border, bv, st); }); }
extern "C" int b200cv_host_warp_perspective(const b200cvMat* s, const b200cvMat* d, const double* M, int flags, int border, const double* bv)
{ if ((border & ~B200CV_BORDER_ISOLATED) == B200CV_BORDER_TRANSPARENT) return B200CV_NOT_IMPLEMENTED;
  return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_warp_perspective(a, b, M, flags, border, bv, st); }); }
extern "C" int b200cv_host_cvt_color(const b200cvMat* s, const b200cvMat* d, int code)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_cvt_color(a, b, code, st); }); }
extern "C" int b200cv_host_corner_harris(const b200cvMat* s, const b200cvMat* d, int bs, int ks, double k, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_corner_harris(a, b, bs, ks, k, border, st); }); }
extern "C" int b200cv_host_corner_min_eigen_val(const b200cvMat* s, const b200cvMat* d, int bs, int ks, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_corner_min_eigen_val(a, b, bs, ks, border, st); }); }
extern "C" int b200cv_host_canny(const b200cvMat* s, const b200cvMat* d, double t1, double t2, int aperture, int l2)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_canny(a, b, t1, t2, aperture, l2, st); }); }
extern "C" int b200cv_host_morphology(const b200cvMat* s, const b200cvMat* d, int op, const unsigned char* kernel_data, size_t kernel_step, int kw,
                                      int kh, int anchor_x, int anchor_y, int iterations, int border, const double border_value[4])
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) {
      return b200cv_morphology(a, b, op, kernel_data, kernel_step, kw, kh, anchor_x, anchor_y, iterations, border, border_value, st); }); }
extern "C" int b200cv_host_distance_transform(const b200cvMat* s, const b200cvMat* d, int distance_type, int mask_size)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_distance_transform(a, b, distance_type, mask_size, st); }); }

extern "C" int b200cv_host_match_template(const b200cvMat* image, const b200cvMat* templ, const b200cvMat* result, int method)
{
    int rc;
    if ((rc = check_mat(templ, "templ"))) return rc;
    HostCtx& c = g_ctx;
    const size_t tp = pitch_of(templ);
    if ((rc = ensure(&c.daux, &c.caux, tp * templ->rows))) return rc;
    B200_CUDA(cudaMemcpy2D(c.daux, tp, templ->data, templ->step, (size_t)templ->cols * elem_size(templ->type), templ->rows, cudaMemcpyHostToDevice));
    B200_CUDA(cudaStreamSynchronize(cudaStreamLegacy));          // pageable source: the call may return once the data is STAGED; the pipeline streams are non-blocking
    b200cvMat dt = {c.daux, tp, templ->cols, templ->rows, templ->type, 1, 0};
    return host_pipeline(image, result, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_match_template(a, &dt, b, method, st); });
}

// ---- cv_hal_* replacements ----------------------------------------------------------------------------------------------
extern "C" int b200cv_hal_gaussianBlur(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int cn,
                                       size_t ml, size_t mt, size_t mr, size_t mb, size_t kw, size_t kh, double sx, double sy, int border)
{
    // in place (src == dst) is fine on this path: the source is on the device before the result comes back
    b200cvMat s = hmat(src, sstep, w, h, B200CV_MAKETYPE(depth, cn)), d = hmat(dst, dstep, w, h, B200CV_MAKETYPE(depth, cn));
    if ((ml | mt | mr | mb) != 0 && !(border & B200CV_BORDER_ISOLATED)) {
        if (kw < 1 || kh < 1) return B200CV_NOT_IMPLEMENTED;      // size left to be derived from sigma: the reach is not known here
        const RoiExt e = roi_ext(ml, mt, mr, mb, (int)kw / 2, (int)kh / 2, (int)kw / 2, (int)kh / 2, border);
        if (e.any())
            return host_roi_call(&s, &d, e.l, e.t, e.r, e.b, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_gaussian_blur(a, b, (int)kw, (int)kh, sx, sy, border, st); });
    }
    return b200cv_host_gaussian_blur(&s, &d, (int)kw, (int)kh, sx, sy, border);
}

extern "C" int b200cv_hal_gaussianBlurBinomial(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int cn,
                                               size_t ml, size_t mt, size_t mr, size_t mb, size_t ksize, int border)
{
    b200cvMat s = hmat(src, sstep, w, h, B200CV_MAKETYPE(depth, cn)), d = hmat(dst, dstep, w, h, B200CV_MAKETYPE(depth, cn));
    const RoiExt e = roi_ext(ml, mt, mr, mb, (int)ksize / 2, (int)ksize / 2, (int)ksize / 2, (int)ksize / 2, border);
    if (e.any())
        return host_roi_call(&s, &d, e.l, e.t, e.r, e.b, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_gaussian_blur(a, b, (int)ksize, (int)ksize, 0, 0, border, st); });
    return b200cv_host_gaussian_blur(&s, &d, (int)ksize, (int)ksize, 0, 0, border);
}

extern "C" int b200cv_hal_sepFilterInit(b200cvFilterCtx** context, int src_type, int dst_type, int kernel_type, uchar* kx, int nx, uchar* ky, int ny,
                                        int ax, int ay, double delta, int border)
{
    if (!context) return B200CV_ERR_BAD_ARG;
    FilterCtxImpl* c = new FilterCtxImpl();
    c->separable = 1;
    if (!taps_to_float(kx, 0, kernel_type, nx, 1, c->kx) || !taps_to_float(ky, 0, kernel_type, ny, 1, c->ky)) { delete c; return B200CV_NOT_IMPLEMENTED; }
    c->ax = ax; c->ay = ay; c->delta = delta; c->border = border; c->src_type = src_type; c->dst_type = dst_type;
    *context = (b200cvFilterCtx*)c;
    return B200CV_OK;
}

extern "C" int b200cv_hal_sepFilter(b200cvFilterCtx* context, uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int fw, int fh, int ox, int oy)
{
    FilterCtxImpl* c = (FilterCtxImpl*)context;
    if (!c) return B200CV_ERR_BAD_ARG;
    b200cvMat s = hmat(src, sstep, w, h, c->src_type), d = hmat(dst, dstep, w, h, c->dst_type);
    const int nx = (int)c->kx.size(), ny = (int)c->ky.size(), ax = c->ax < 0 ? nx / 2 : c->ax, ay = c->ay < 0 ? ny / 2 : c->ay;
    if (ox < 0 || oy < 0 || fw < ox + w || fh < oy + h) return B200CV_NOT_IMPLEMENTED;
    const RoiExt e = roi_ext((size_t)ox, (size_t)oy, (size_t)(fw - w - ox), (size_t)(fh - h - oy), ax, ay, nx - 1 - ax, ny - 1 - ay, c->border);
    const float *kx = c->kx.data(), *ky = c->ky.data();
    const int cax = c->ax, cay = c->ay, cb = c->border; const double cd = c->delta;
    if (e.any())
        return host_roi_call(&s, &d, e.l, e.t, e.r, e.b, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_sep_filter2d(a, b, kx, nx, ky, ny, cax, cay, cd, cb, st); });
    return b200cv_host_sep_filter2d(&s, &d, kx, nx, ky, ny, cax, cay, cd, cb);
}

extern "C" int b200cv_hal_sepFilterFree(b200cvFilterCtx* context) { delete (FilterCtxImpl*)context; return B200CV_OK; }

extern "C" int b200cv_hal_filterInit(b200cvFilterCtx** context, uchar* kdata, size_t kstep, int ktype, int kw, int kh, int, int, int src_type, int dst_type,
                                     int border, double delta, int ax, int ay, bool, bool)
{
    if (!context) return B200CV_ERR_BAD_ARG;
    FilterCtxImpl* c = new FilterCtxImpl();
    c->separable = 0;
    if (B200CV_CN(ktype) != 1 || !taps_to_float(kdata, kstep, ktype, kw, kh, c->k2d)) { delete c; return B200CV_NOT_IMPLEMENTED; }
    c->kw = kw; c->kh = kh; c->ax = ax; c->ay = ay; c->delta = delta; c->border = border; c->src_type = src_type; c->dst_type = dst_type;
    *context = (b200cvFilterCtx*)c;
    return B200CV_OK;
}

extern "C" int b200cv_hal_filter(b200cvFilterCtx* context, uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int fw, int fh, int ox, int oy)
{
    FilterCtxImpl* c = (FilterCtxImpl*)context;
    if (!c) return B200CV_ERR_BAD_ARG;
    b200cvMat s = hmat(src, sstep, w, h, c->src_type), d = hmat(dst, dstep, w, h, c->dst_type);
    const int ax = c->ax < 0 ? c->kw / 2 : c->ax, ay = c->ay < 0 ? c->kh / 2 : c->ay;
    if (ox < 0 || oy < 0 || fw < ox + w || fh < oy + h) return B200CV_NOT_IMPLEMENTED;
    const RoiExt e = roi_ext((size_t)ox, (size_t)oy, (size_t)(fw - w - ox), (size_t)(fh - h - oy), ax, ay, c->kw - 1 - ax, c->kh - 1 - ay, c->border);
    const float* k2 = c->k2d.data();
    const int kw = c->kw, kh = c->kh, cax = c->ax, cay = c->ay, cb = c->border; const double cd = c->delta;
    if (e.any())
        return host_roi_call(&s, &d, e.l, e.t, e.r, e.b, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_filter2d(a, b, k2, kw, kh, cax, cay, cd, cb, st); });
    return b200cv_host_filter2d(&s, &d, k2, kw, kh, cax, cay, cd, cb);
}

extern "C" int b200cv_hal_filterFree(b200cvFilterCtx* context) { delete (FilterCtxImpl*)context; return B200CV_OK; }

extern "C" int b200cv_hal_sobel(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int sdepth, int ddepth, int cn,
                                int ml, int mt, int mr, int mb, int dx, int dy, int ksize, double scale, double delta, int border)
{
    if (src == dst && sdepth != ddepth) return B200CV_NOT_IMPLEMENTED;
    b200cvMat s = hmat(src, sstep, w, h, B200CV_MAKETYPE(sdepth, cn)), d = hmat(dst, dstep, w, h, B200CV_MAKETYPE(ddepth, cn));
    const int rr = ksize <= 0 ? 1 : ksize / 2;                 // Scharr (ksize -1) and 1 x 3 / 3 x 1 kernels reach one pixel
    const RoiExt e = roi_ext((size_t)std::max(ml, 0), (size_t)std::max(mt, 0), (size_t)std::max(mr, 0), (size_t)std::max(mb, 0), rr, rr, rr, rr, border);
    if (e.any())
        return host_roi_call(&s, &d, e.l, e.t, e.r, e.b, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_sobel(a, b, dx, dy, ksize, scale, delta, border, st); });
    return b200cv_host_sobel(&s, &d, dx, dy, ksize, scale, delta, border);
}

extern "C" int b200cv_hal_scharr(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int sdepth, int ddepth, int cn,
                                 int ml, int mt, int mr, int mb, int dx, int dy, double scale, double delta, int border)
{
    return b200cv_hal_sobel(src, sstep, dst, dstep, w, h, sdepth, ddepth, cn, ml, mt, mr, mb, dx, dy, -1, scale, delta, border);
}

extern "C" int b200cv_hal_boxFilter(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int sdepth, int ddepth, int cn,
                                    int ml, int mt, int mr, int mb, size_t kw, size_t kh, int ax, int ay, bool normalize, int border)
{
    if ((src == dst && sdepth != ddepth) || kw > 128 || kh > 128) return B200CV_NOT_IMPLEMENTED;
    b200cvMat s = hmat(src, sstep, w, h, B200CV_MAKETYPE(sdepth, cn)), d = hmat(dst, dstep, w, h, B200CV_MAKETYPE(ddepth, cn));
    const int bax = ax < 0 ? (int)kw / 2 : ax, bay = ay < 0 ? (int)kh / 2 : ay;
    const RoiExt e = roi_ext((size_t)std::max(ml, 0), (size_t)std::max(mt, 0), (size_t)std::max(mr, 0), (size_t)std::max(mb, 0), bax, bay, (int)kw - 1 - bax, (int)kh - 1 - bay, border);
    const int ikw = (int)kw, ikh = (int)kh, nrm = normalize ? 1 : 0;
    if (e.any())
        return host_roi_call(&s, &d, e.l, e.t, e.r, e.b, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_box_filter(a, b, ikw, ikh, ax, ay, nrm, border, st); });
    return b200cv_host_box_filter(&s, &d, ikw, ikh, ax, ay, nrm, border);
}

// cv::integral has two outputs: sum through the pipeline; sqsum (rare) as a second pass over the same source
extern "C" int b200cv_host_integral(const b200cvMat* s, const b200cvMat* sum, const b200cvMat* sqsum)
{
    int rc = host_pipeline(s, sum, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_integral(a, b, nullptr, st); });
    if (rc || !sqsum || !sqsum->data) return rc;
    if (sqsum->type != B200CV_MAKETYPE(B200CV_64F, 1)) return B200CV_NOT_IMPLEMENTED;
    // the device entry wants both outputs: give it a scratch sum next to the squares (stream-ordered, freed right after)
    return host_pipeline(s, sqsum, [=](const b200cvMat* a, const b200cvMat* b, void* st) {
        b200cvMat tmp = *b;
        tmp.type = B200CV_MAKETYPE(B200CV_32S, 1);
        tmp.step = (size_t)b->cols * 4; tmp.frame_step = tmp.step * b->rows;
        void* p = nullptr;
        const int frames = b->frames > 1 ? b->frames : 1;
        if (cudaMallocAsync(&p, tmp.frame_step * frames, (cudaStream_t)st) != cudaSuccess) { cudaGetLastError(); return (int)B200CV_ERR_CUDA; }
        tmp.data = p;
        const int r = b200cv_integral(a, &tmp, b, st);
        cudaFreeAsync(p, (cudaStream_t)st);
        return r;
    });
}

extern "C" int b200cv_hal_integral(int depth, int sdepth, int sqdepth, const uchar* src, size_t sstep, uchar* sum, size_t sumstep, uchar* sqsum, size_t sqstep,
                                   uchar* tilted, size_t, int w, int h, int cn)
{
    if (depth != B200CV_8U || sdepth != B200CV_32S || cn != 1 || tilted || !sum || (sqsum && sqdepth != B200CV_64F)) return B200CV_NOT_IMPLEMENTED;
    b200cvMat s = hmat(src, sstep, w, h, B200CV_MAKETYPE(B200CV_8U, 1)), d = hmat(sum, sumstep, w + 1, h + 1, B200CV_MAKETYPE(B200CV_32S, 1));
    b200cvMat q = hmat(sqsum, sqstep, w + 1, h + 1, B200CV_MAKETYPE(B200CV_64F, 1));
    return b200cv_host_integral(&s, &d, sqsum ? &q : nullptr);
}

extern "C" int b200cv_hal_resize(int type, const uchar* src, size_t sstep, int sw, int sh, uchar* dst, size_t dstep, int dw, int dh,
                                 double inv_x, double inv_y, int interp)
{
    // inv_x, inv_y = cv::resize's fx, fy when it was called with an empty dsize, else dsize / ssize (resize.cpp:4214-4228): passed through
    b200cvMat s = hmat(src, sstep, sw, sh, type), d = hmat(dst, dstep, dw, dh, type);
    return b200cv_host_resize_scaled(&s, &d, interp, inv_x, inv_y);
}

extern "C" int b200cv_hal_warpAffine(int type, const uchar* src, size_t sstep, int sw, int sh, uchar* dst, size_t dstep, int dw, int dh,
                                     const double M[6], int interp, int border, const double bv[4])
{
    b200cvMat s = hmat(src, sstep, sw, sh, type), d = hmat(dst, dstep, dw, dh, type);
    return b200cv_host_warp_affine(&s, &d, M, interp | B200CV_WARP_INVERSE_MAP, border, bv);
}

extern "C" int b200cv_hal_warpPerspective(int type, const uchar* src, size_t sstep, int sw, int sh, uchar* dst, size_t dstep, int dw, int dh,
                                          const double M[9], int interp, int border, const double bv[4])
{
    b200cvMat s = hmat(src, sstep, sw, sh, type), d = hmat(dst, dstep, dw, dh, type);
    return b200cv_host_warp_perspective(&s, &d, M, interp | B200CV_WARP_INVERSE_MAP, border, bv);
}

extern "C" int b200cv_host_pyr_down(const b200cvMat* s, const b200cvMat* d, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_pyr_down(a, b, border, st); }); }
extern "C" int b200cv_host_pyr_up(const b200cvMat* s, const b200cvMat* d, int border)
{ return host_pipeline(s, d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_pyr_up(a, b, border, st); }); }

extern "C" int b200cv_hal_pyrdown(const uchar* src, size_t sstep, int sw, int sh, uchar* dst, size_t dstep, int dw, int dh, int depth, int cn, int border)
{
    if (src == dst) return B200CV_NOT_IMPLEMENTED;
    b200cvMat s = hmat(src, sstep, sw, sh, B200CV_MAKETYPE(depth, cn)), d = hmat(dst, dstep, dw, dh, B200CV_MAKETYPE(depth, cn));
    return b200cv_host_pyr_down(&s, &d, border);
}

extern "C" int b200cv_host_remap(const b200cvMat* src, const b200cvMat* dst, const b200cvMat* map1, const b200cvMat* map2, int interp, int border, const double* bv)
{
    int rc;
    if ((border & ~B200CV_BORDER_ISOLATED) == B200CV_BORDER_TRANSPARENT) return B200CV_NOT_IMPLEMENTED;
    if ((rc = check_mat(map1, "map1"))) return rc;
    const bool has2 = map2 && map2->data;
    if (has2 && (rc = check_mat(map2, "map2"))) return rc;
    // the maps are uploaded once (aux buffer), the frames flow through the pipeline
    HostCtx& c = g_ctx;
    const size_t p1 = pitch_of(map1), p2 = has2 ? pitch_of(map2) : 0;
    const size_t b1 = p1 * map1->rows, b2 = has2 ? p2 * map2->rows : 0;
    if ((rc = ensure(&c.daux, &c.caux, b1 + b2))) return rc;
    B200_CUDA(cudaMemcpy2D(c.daux, p1, map1->data, map1->step, (size_t)map1->cols * elem_size(map1->type), map1->rows, cudaMemcpyHostToDevice));
    if (has2) B200_CUDA(cudaMemcpy2D((char*)c.daux + b1, p2, map2->data, map2->step, (size_t)map2->cols * elem_size(map2->type), map2->rows, cudaMemcpyHostToDevice));
    B200_CUDA(cudaStreamSynchronize(cudaStreamLegacy));          // pageable sources: see b200cv_host_match_template
    b200cvMat d1 = {c.daux, p1, map1->cols, map1->rows, map1->type, 1, 0};
    b200cvMat d2 = {has2 ? (void*)((char*)c.daux + b1) : nullptr, p2, has2 ? map2->cols : 0, has2 ? map2->rows : 0, has2 ? map2->type : 0, 1, 0};
    return host_pipeline(src, dst, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return b200cv_remap(a, b, &d1, has2 ? &d2 : nullptr, interp, border, bv, st); });
}

extern "C" int b200cv_hal_remap32f(int type, const uchar* src, size_t sstep, int sw, int sh, uchar* dst, size_t dstep, int dw, int dh,
                                   float* mapx, size_t mapx_step, float* mapy, size_t mapy_step, int interp, int border, const double bv[4])
{
    if (src == dst) return B200CV_NOT_IMPLEMENTED;
    b200cvMat s = hmat(src, sstep, sw, sh, type), d = hmat(dst, dstep, dw, dh, type);
    b200cvMat mx = hmat(mapx, mapx_step, dw, dh, B200CV_MAKETYPE(B200CV_32F, 1)), my = hmat(mapy, mapy_step, dw, dh, B200CV_MAKETYPE(B200CV_32F, 1));
    return b200cv_host_remap(&s, &d, &mx, &my, interp, border, bv);
}

static int cvt(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int scn, int dcn, int code)
{
    // 16-bit and float images: the channel reorders, GRAY, XYZ and YCrCb / YUV families (cvtcolor_depth.cu); everything else is 8-bit only
    const bool depth_family = code <= 11 || (code >= 32 && code <= 39) || (code >= 82 && code <= 85);
    const bool hsv = code == 40 || code == 41 || code == 54 || code == 55 || code == 66 || code == 67 || code == 70 || code == 71;      // float only
    if (depth != B200CV_8U && !((depth == B200CV_16U || depth == B200CV_32F) && depth_family) && !(depth == B200CV_32F && hsv)) return B200CV_NOT_IMPLEMENTED;
    b200cvMat s = hmat(src, sstep, w, h, B200CV_MAKETYPE(depth, scn)), d = hmat(dst, dstep, w, h, B200CV_MAKETYPE(depth, dcn));
    return b200cv_host_cvt_color(&s, &d, code);
}

extern "C" int b200cv_hal_cvtBGRtoXYZ(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int scn, bool swapBlue)
{ return cvt(src, sstep, dst, dstep, w, h, depth, scn, 3, swapBlue ? 33 : 32); }
extern "C" int b200cv_hal_cvtXYZtoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int dcn, bool swapBlue)
{ return cvt(src, sstep, dst, dstep, w, h, depth, 3, dcn, swapBlue ? 35 : 34); }
extern "C" int b200cv_hal_cvtBGRtoLab(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int scn, bool swapBlue, bool isLab, bool srgb)
{
    if (!isLab || depth != B200CV_8U) return B200CV_NOT_IMPLEMENTED;      // Luv, float Lab: not on the device path
    return cvt(src, sstep, dst, dstep, w, h, depth, scn, 3, srgb ? (swapBlue ? 45 : 44) : (swapBlue ? 75 : 74));
}
extern "C" int b200cv_hal_cvtLabtoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int dcn, bool swapBlue, bool isLab, bool srgb)
{
    if (!isLab || depth != B200CV_8U) return B200CV_NOT_IMPLEMENTED;
    return cvt(src, sstep, dst, dstep, w, h, depth, 3, dcn, srgb ? (swapBlue ? 57 : 56) : (swapBlue ? 79 : 78));
}

// subsampled YUV wire formats (cvtcolor_yuv.cu); source and destination differ in size
static int cvt_yuv(const uchar* src, size_t sstep, int sw, int sh, int scn, uchar* dst, size_t dstep, int dw, int dh, int dcn, int code)
{
    if ((dw & 1) || (sw & 1) || src == dst) return B200CV_NOT_IMPLEMENTED;
    b200cvMat s = hmat(src, sstep, sw, sh, B200CV_MAKETYPE(B200CV_8U, scn)), d = hmat(dst, dstep, dw, dh, B200CV_MAKETYPE(B200CV_8U, dcn));
    return b200cv_host_cvt_color(&s, &d, code);
}
extern "C" int b200cv_hal_cvtTwoPlaneYUVtoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int dw, int dh, int dcn, bool swapBlue, int uIdx)
{
    if ((dcn != 3 && dcn != 4) || (uIdx != 0 && uIdx != 1) || (dh & 1)) return B200CV_NOT_IMPLEMENTED;
    return cvt_yuv(src, sstep, dw, dh * 3 / 2, 1, dst, dstep, dw, dh, dcn, 90 + (swapBlue ? 0 : 1) + 2 * uIdx + (dcn == 4 ? 4 : 0));
}
extern "C" int b200cv_hal_cvtThreePlaneYUVtoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int dw, int dh, int dcn, bool swapBlue, int uIdx)
{
    if ((dcn != 3 && dcn != 4) || (uIdx != 0 && uIdx != 1) || (dh & 1)) return B200CV_NOT_IMPLEMENTED;
    return cvt_yuv(src, sstep, dw, dh * 3 / 2, 1, dst, dstep, dw, dh, dcn, 98 + (swapBlue ? 0 : 1) + (uIdx == 1 ? 0 : 2) + (dcn == 4 ? 4 : 0));
}
extern "C" int b200cv_hal_cvtBGRtoThreePlaneYUV(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int scn, bool swapBlue, int uIdx)
{
    if ((scn != 3 && scn != 4) || (uIdx != 1 && uIdx != 2) || (h & 1)) return B200CV_NOT_IMPLEMENTED;
    return cvt_yuv(src, sstep, w, h, scn, dst, dstep, w, h * 3 / 2, 1, (uIdx == 2 ? 131 : 127) + (swapBlue ? 0 : 1) + (scn == 4 ? 2 : 0));
}
extern "C" int b200cv_hal_cvtOnePlaneYUVtoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int dcn, bool swapBlue, int uIdx, int ycn)
{
    if ((dcn != 3 && dcn != 4) || (uIdx != 0 && uIdx != 1) || (ycn != 0 && ycn != 1) || (ycn == 1 && uIdx == 1)) return B200CV_NOT_IMPLEMENTED;
    // UYVY: 107 RGB 108 BGR 111 RGBA 112 BGRA; YUY2: 115 116 119 120; YVYU: 117 118 121 122
    const int base = ycn == 1 ? (dcn == 3 ? 107 : 111) : (dcn == 3 ? 115 : 119) + (uIdx == 1 ? 2 : 0);
    return cvt_yuv(src, sstep, w, h, 2, dst, dstep, w, h, dcn, base + (swapBlue ? 0 : 1));
}

extern "C" int b200cv_hal_cvtOnePlaneBGRtoYUV(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int scn, bool swapBlue, int uIdx, int ycn)
{
    if ((scn != 3 && scn != 4) || (uIdx != 0 && uIdx != 1) || (ycn != 0 && ycn != 1) || (ycn == 1 && uIdx == 1)) return B200CV_NOT_IMPLEMENTED;
    // UYVY: 143 RGB 144 BGR 145 RGBA 146 BGRA; YUY2: 147 148 151 152; YVYU: 149 150 153 154
    const int base = ycn == 1 ? (scn == 3 ? 143 : 145) : (scn == 3 ? 147 : 151) + (uIdx == 1 ? 2 : 0);
    return cvt_yuv(src, sstep, w, h, scn, dst, dstep, w, h, 2, base + (swapBlue ? 0 : 1));
}

extern "C" int b200cv_hal_cvtBGRtoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int scn, int dcn, bool swapBlue)
{
    int code = scn == 3 ? (dcn == 4 ? (swapBlue ? 2 : 0) : (swapBlue ? 4 : -1)) : (dcn == 3 ? (swapBlue ? 3 : 1) : (swapBlue ? 5 : -1));
    if (code < 0) return B200CV_NOT_IMPLEMENTED;
    return cvt(src, sstep, dst, dstep, w, h, depth, scn, dcn, code);
}
extern "C" int b200cv_hal_cvtBGRtoGray(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int scn, bool swapBlue)
{ return cvt(src, sstep, dst, dstep, w, h, depth, scn, 1, scn == 3 ? (swapBlue ? 7 : 6) : (swapBlue ? 11 : 10)); }
extern "C" int b200cv_hal_cvtGraytoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int dcn)
{ return cvt(src, sstep, dst, dstep, w, h, depth, 1, dcn, dcn == 3 ? 8 : 9); }
extern "C" int b200cv_hal_cvtBGRtoYUV(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int scn, bool swapBlue, bool isCbCr)
{ return cvt(src, sstep, dst, dstep, w, h, depth, scn, 3, isCbCr ? (swapBlue ? 37 : 36) : (swapBlue ? 83 : 82)); }
extern "C" int b200cv_hal_cvtYUVtoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int dcn, bool swapBlue, bool isCbCr)
{ return cvt(src, sstep, dst, dstep, w, h, depth, 3, dcn, isCbCr ? (swapBlue ? 39 : 38) : (swapBlue ? 85 : 84)); }
extern "C" int b200cv_hal_cvtBGRtoHSV(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int scn, bool swapBlue, bool full, bool isHSV)
{
    if (!isHSV) return B200CV_NOT_IMPLEMENTED;   // HLS: not on the device path
    return cvt(src, sstep, dst, dstep, w, h, depth, scn, 3, full ? (swapBlue ? 67 : 66) : (swapBlue ? 41 : 40));
}
extern "C" int b200cv_hal_cvtHSVtoBGR(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int depth, int dcn, bool swapBlue, bool full, bool isHSV)
{
    if (!isHSV) return B200CV_NOT_IMPLEMENTED;
    return cvt(src, sstep, dst, dstep, w, h, depth, 3, dcn, full ? (swapBlue ? 71 : 70) : (swapBlue ? 55 : 54));
}

// cv::Canny has already turned the user's arguments into these (canny.cpp:838-856) and dropped the ROI context (:861-862): the thresholds
// go to the computation as they are
extern "C" int b200cv_hal_canny(const uchar* src, size_t sstep, uchar* dst, size_t dstep, int w, int h, int cn, double low, double high, int ksize,
                                bool L2gradient)
{
    b200cvMat s = hmat(src, sstep, w, h, B200CV_MAKETYPE(B200CV_8U, cn)), d = hmat(dst, dstep, w, h, B200CV_MAKETYPE(B200CV_8U, 1));
    const int l2 = L2gradient ? 1 : 0;
    return host_pipeline(&s, &d, [=](const b200cvMat* a, const b200cvMat* b, void* st) { return canny_prepared(a, nullptr, b, low, high, ksize, l2, st); });
}
