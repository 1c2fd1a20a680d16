/*
 * b200cv_batch.h -- the multi-GPU batch driver of the hot path.
 *
 * A batch of independent frames in HOST memory (cv::Mat layout, b200cvMat with frames > 1) is sharded over the GPUs of one box:
 * frame block [lo, hi) of device i = b200cv_batch_shard (contiguous blocks that differ by at most one frame), one persistent host
 * thread per device (pinned to the CPUs next to that GPU, so the page-locked staging rings it allocates are NUMA-local), each thread
 * drives its own upload / kernel / download streams -- the arrangement of the reference's multi-GPU sample
 * (samples/gpu/multi.cpp:27-68: one worker per device, cv::cuda::setDevice, no shared state), with the sharding, pinning and
 * stream pipeline inside the library instead of in every application.
 *
 * The path has no cross-frame state; the ONLY exchange is the broadcast of the small shared operand (matchTemplate's template) from the
 * first device to the others: ncclBroadcast over NVLink (libnccl.so.2 is loaded at run time; a driver over ONE device needs no NCCL --
 * that is the torchrun arrangement, one process per GPU, where the process group owns the broadcast).  Filter taps, warp matrices and
 * resize scales are kernel parameters read from the caller's host memory, the same address space for every worker: nothing to send.
 *
 * Error convention: b200cv.h's (0 ok, 1 not implemented, < 0 error; b200cv_last_error() on the calling thread carries the first
 * failing worker's message).  Calls are synchronous: results are in the destination host buffers on return.
 */
#ifndef B200CV_BATCH_H
#define B200CV_BATCH_H
#include "b200cv.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200cvBatch b200cvBatch;

/* devices == NULL or n_devices <= 0: every visible device.  Starts one worker thread per device (cudaSetDevice, b200cv_init, CPU affinity
 * from /sys/bus/pci/devices/<gpu>/local_cpulist).  With more than one device an NCCL communicator is created (ncclCommInitAll). */
B200CV_API int b200cv_batch_create(b200cvBatch** batch, const int* devices, int n_devices);
B200CV_API int b200cv_batch_destroy(b200cvBatch* batch);
B200CV_API int b200cv_batch_device_count(const b200cvBatch* batch);
B200CV_API int b200cv_batch_device(const b200cvBatch* batch, int index);           /* CUDA ordinal of worker `index` */
B200CV_API int b200cv_batch_uses_nccl(const b200cvBatch* batch);                    /* 1 when the shared-operand broadcast runs through NCCL */
/* frame block of worker `index` out of `n_workers` for a batch of `frames`: pure host arithmetic (callable without a GPU) */
B200CV_API int b200cv_batch_shard(int frames, int index, int n_workers, int* first, int* count);
/* page-locked host memory allocated AND first touched by worker `index` (lands on the NUMA node next to its GPU); frames
 * [first, first + count) of a batch buffer should come from the worker that b200cv_batch_shard assigns them to */
B200CV_API int b200cv_batch_host_alloc(b200cvBatch* batch, int index, void** hptr, size_t bytes);
B200CV_API int b200cv_batch_host_free(b200cvBatch* batch, int index, void* hptr);
/* one CONTIGUOUS page-locked batch buffer (frames x frame_bytes) whose frame blocks are first touched by the workers that own them
 * (b200cv_batch_shard), then page-locked in place: every device streams from / to its own NUMA node */
B200CV_API int b200cv_batch_host_alloc_frames(b200cvBatch* batch, void** hptr, size_t frame_bytes, int frames);
B200CV_API int b200cv_batch_host_free_frames(b200cvBatch* batch, void* hptr);
/* frames processed by worker `index` during the last call (reporting) */
B200CV_API int b200cv_batch_last_count(const b200cvBatch* batch, int index);

/* ---- ops over sharded host batches: the argument lists of b200cv_host_* (b200cv_hal.h) behind the batch handle ---- */
B200CV_API int b200cv_batch_gaussian_blur(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* dst, int ksize_w, int ksize_h, double sigma_x, double sigma_y, int border);
B200CV_API int b200cv_batch_sep_filter2d(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* dst, const float* kx, int kx_len, const float* ky, int ky_len,
                                         int anchor_x, int anchor_y, double delta, int border);
B200CV_API int b200cv_batch_filter2d(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* dst, const float* kernel, int kw, int kh, int anchor_x, int anchor_y,
                                     double delta, int border);
B200CV_API int b200cv_batch_resize(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* dst, int interpolation, double fx, double fy);
B200CV_API int b200cv_batch_warp_affine(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* dst, const double* M, int flags, int border, const double* border_value);
B200CV_API int b200cv_batch_warp_perspective(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* dst, const double* M, int flags, int border, const double* border_value);
B200CV_API int b200cv_batch_cvt_color(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* dst, int code);
B200CV_API int b200cv_batch_corner_harris(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* dst, int block_size, int ksize, double k, int border);
/* templ: HOST, one frame.  Uploaded to the first device and broadcast to the others (ncclBroadcast), then every worker matches its frames */
B200CV_API int b200cv_batch_match_template(b200cvBatch* batch, const b200cvMat* image, const b200cvMat* templ, const b200cvMat* result, int method);

/* the bench.py c5 workload: SIFT Gaussian pyramid + DoG (b200cv_sift_pyramid) and cornerHarris over a sharded batch of 8UC1 host frames, in WAVES
 * of `wave` frames per device (a 4K frame's pyramids are 1.06 + 0.88 GB: a device holds one wave's pyramids in a reusable arena).
 * harris: HOST CV_32FC1 batch receiving the responses, or NULL (they stay on the device like the pyramids).
 * consumer: NULL, or called on the worker's thread after each wave with DEVICE pointers to that wave's pyramids (layout of b200cv_sift_pyramid,
 * per-frame strides gauss_frame_elems / dog_frame_elems) and Harris responses -- the hook for what comes next (b200cv_sift_detect_and_compute);
 * the stream is synchronised before the call, the arena is reused when it returns.  Upload of wave w+1 overlaps the kernels of wave w. */
typedef int (*b200cvWaveConsumer)(void* user, int device_index, int first_frame, int n_frames, const float* gauss, size_t gauss_frame_elems,
                                  const float* dog, size_t dog_frame_elems, const float* harris, size_t harris_step, size_t harris_frame_step);
B200CV_API int b200cv_batch_sift_harris(b200cvBatch* batch, const b200cvMat* src, const b200cvMat* harris, int n_octave_layers, double sigma, int upscale,
                                        int harris_block_size, int harris_ksize, double harris_k, int wave, b200cvWaveConsumer consumer, void* user);

#ifdef __cplusplus
}
#endif
#endif /* B200CV_BATCH_H */
