// runtime.cu -- device/stream/event/allocator runtime behind the C ABI.
// Own implementation of the surface cv::cuda::{Stream,Event,HostMem,GpuMat::Allocator} expose
// (reference decls: modules/core/include/opencv2/core/cuda.hpp:105-115,791-870,909-1016); the reference's
// own implementation (modules/core/src/cuda_stream.cpp, cuda/gpu_mat.cu) cannot be built without contrib's cudev.
#include <atomic>
#include <cstdarg>
#include <cstring>
#include "common.cuh"

namespace b200cv {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};
static int g_num_sms[64] = {};

void set_error(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line)
{
    set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    return e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver ? B200CV_ERR_NO_DEVICE : B200CV_ERR_CUDA;
}

void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

int num_sms()
{
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    int& slot = g_num_sms[dev & 63];
    if (slot == 0) slot = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
    return slot;
}

int check_mat(const b200cvMat* m, const char* name)
{
    if (!m) { set_error("%s: null descriptor", name); return B200CV_ERR_BAD_ARG; }
    if (!m->data || m->cols <= 0 || m->rows <= 0) { set_error("%s: empty image", name); return B200CV_ERR_BAD_ARG; }
    if (m->step < (size_t)m->cols * elem_size(m->type)) { set_error("%s: step %zu < row bytes", name, m->step); return B200CV_ERR_BAD_ARG; }
    if (m->frames > 1 && m->frame_step < m->step * (size_t)m->rows) { set_error("%s: frame_step too small", name); return B200CV_ERR_BAD_ARG; }
    return B200CV_OK;
}

// Scratch buffers (padded images, coefficient tables, candidate lists) are stream-ordered allocations.  By default the pool hands
// unused memory back to the OS at every synchronisation, so the next call pays a fresh allocation (the host path
// synchronises after every op).  Keep the memory in the pool.
void configure_mem_pool()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return; }
    static bool done[64] = {};
    if (dev < 0 || dev >= 64 || done[dev]) return;
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        unsigned long long keep = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    cudaGetLastError();
    done[dev] = true;
}

}  // namespace b200cv

using namespace b200cv;

extern "C" {

const char* b200cv_last_error(void) { return g_err; }
const char* b200cv_version(void) { return "b200cv 0.1 (sm_90a)"; }
unsigned long long b200cv_launch_count(void) { return g_launches.load(); }

int b200cv_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}


int b200cv_init(int device)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        set_error("no CUDA device visible: the b200cv hot path has no CPU fallback");
        return B200CV_ERR_NO_DEVICE;
    }
    B200_REQUIRE(device >= 0 && device < n, "bad device index");
    B200_CUDA(cudaSetDevice(device));
    cudaDeviceProp p;
    B200_CUDA(cudaGetDeviceProperties(&p, device));
    if (p.major != 9 || p.minor != 0) {
        set_error("device %d is sm_%d%d; this library contains sm_90a code only", device, p.major, p.minor);
        return B200CV_ERR_NO_DEVICE;
    }
    g_num_sms[device & 63] = p.multiProcessorCount;
    B200_CUDA(cudaFree(0));
    configure_mem_pool();
    return B200CV_OK;
}

int b200cv_malloc_pitch(void** dptr, size_t* step, size_t width_bytes, size_t rows)
{
    B200_REQUIRE(dptr && step && width_bytes > 0 && rows > 0, "bad malloc_pitch args");
    size_t pitch = (width_bytes + 255) & ~(size_t)255;
    B200_CUDA(cudaMalloc(dptr, pitch * rows));
    *step = pitch;
    return B200CV_OK;
}

int b200cv_free(void* dptr)
{
    B200_CUDA(cudaFree(dptr));
    return B200CV_OK;
}

int b200cv_host_alloc(void** hptr, size_t bytes)
{
    B200_REQUIRE(hptr && bytes > 0, "bad host_alloc args");
    B200_CUDA(cudaHostAlloc(hptr, bytes, cudaHostAllocDefault));
    return B200CV_OK;
}

int b200cv_host_free(void* hptr)
{
    B200_CUDA(cudaFreeHost(hptr));
    return B200CV_OK;
}

int b200cv_upload(const void* hsrc, size_t hstep, void* ddst, size_t dstep, size_t width_bytes, size_t rows, void* stream)
{
    B200_CUDA(cudaMemcpy2DAsync(ddst, dstep, hsrc, hstep, width_bytes, rows, cudaMemcpyHostToDevice, as_stream(stream)));
    return B200CV_OK;
}

int b200cv_download(const void* dsrc, size_t dstep, void* hdst, size_t hstep, size_t width_bytes, size_t rows, void* stream)
{
    B200_CUDA(cudaMemcpy2DAsync(hdst, hstep, dsrc, dstep, width_bytes, rows, cudaMemcpyDeviceToHost, as_stream(stream)));
    return B200CV_OK;
}

int b200cv_stream_create(void** stream)
{
    B200_REQUIRE(stream, "null out pointer");
    cudaStream_t s;
    B200_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    *stream = (void*)s;
    return B200CV_OK;
}

int b200cv_stream_destroy(void* stream)
{
    B200_CUDA(cudaStreamDestroy(as_stream(stream)));
    return B200CV_OK;
}

int b200cv_stream_query(void* stream)
{
    cudaError_t e = cudaStreamQuery(as_stream(stream));
    if (e == cudaSuccess) return 0;
    if (e == cudaErrorNotReady) { cudaGetLastError(); return 1; }
    return cuda_fail(e, "cudaStreamQuery", __FILE__, __LINE__);
}

int b200cv_stream_synchronize(void* stream)
{
    B200_CUDA(cudaStreamSynchronize(as_stream(stream)));
    return B200CV_OK;
}

int b200cv_stream_wait_event(void* stream, void* event)
{
    B200_CUDA(cudaStreamWaitEvent(as_stream(stream), (cudaEvent_t)event, 0));
    return B200CV_OK;
}

struct HostCb { void (*fn)(int, void*); void* user; };
static void CUDART_CB host_cb_trampoline(void* p)
{
    HostCb* cb = (HostCb*)p;
    cb->fn(0, cb->user);
    delete cb;
}

int b200cv_stream_add_callback(void* stream, void (*fn)(int, void*), void* user)
{
    B200_REQUIRE(fn, "null callback");
    HostCb* cb = new HostCb{fn, user};
    cudaError_t e = cudaLaunchHostFunc(as_stream(stream), host_cb_trampoline, cb);
    if (e != cudaSuccess) { delete cb; return cuda_fail(e, "cudaLaunchHostFunc", __FILE__, __LINE__); }
    return B200CV_OK;
}

int b200cv_event_create(void** event)
{
    B200_REQUIRE(event, "null out pointer");
    cudaEvent_t e;
    B200_CUDA(cudaEventCreate(&e));
    *event = (void*)e;
    return B200CV_OK;
}

int b200cv_event_destroy(void* event)
{
    B200_CUDA(cudaEventDestroy((cudaEvent_t)event));
    return B200CV_OK;
}

int b200cv_event_record(void* event, void* stream)
{
    B200_CUDA(cudaEventRecord((cudaEvent_t)event, as_stream(stream)));
    return B200CV_OK;
}

int b200cv_event_synchronize(void* event)
{
    B200_CUDA(cudaEventSynchronize((cudaEvent_t)event));
    return B200CV_OK;
}

int b200cv_event_elapsed_ms(void* start, void* end, float* ms)
{
    B200_CUDA(cudaEventElapsedTime(ms, (cudaEvent_t)start, (cudaEvent_t)end));
    return B200CV_OK;
}

}  // extern "C"

// ---- TMA tensor maps ---------------------------------------------------------------------------------------------------
#include "tma.cuh"
namespace b200cv {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

int make_tensor_map_3d(CUtensorMap* map, const void* base, int elem_bytes, int cols, int rows, int frames, size_t step, size_t fstep,
                       int box_w, int box_h)
{
    EncodeTiledFn fn = encode_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return B200CV_ERR_CUDA; }
    CUtensorMapDataType dt = elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)(frames > 0 ? frames : 1)};
    cuuint64_t strides[2] = {(cuuint64_t)step, (cuuint64_t)(frames > 1 ? fstep : step * (size_t)rows)};
    cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(map, dt, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return B200CV_ERR_CUDA; }
    return B200CV_OK;
}

int upload_tensor_map(const CUtensorMap& tm, CUtensorMap** dptr, cudaStream_t st)
{
    void* p = nullptr;
    B200_CUDA(cudaMallocAsync(&p, sizeof(CUtensorMap), st));
    cudaError_t e = cudaMemcpyAsync(p, &tm, sizeof(CUtensorMap), cudaMemcpyHostToDevice, st);   // pageable source: staged before return
    if (e != cudaSuccess) { cudaFreeAsync(p, st); return cuda_fail(e, "tensor map upload", __FILE__, __LINE__); }
    *dptr = (CUtensorMap*)p;
    return B200CV_OK;
}
}  // namespace b200cv
