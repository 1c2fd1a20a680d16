"""opencv_b200.batch -- sharding a batch of independent frames over the GPUs of one box (one process per GPU).

The hot path has no cross-frame state: rank r owns a contiguous block of frames, runs the whole per-frame
pipeline on its own stream(s) and keeps its results.  The ONLY exchange is a broadcast of the small shared operand
(template / filter taps / warp matrix) from rank 0 -- NCCL over NVLink on GPUs, gloo in the CPU tests.
"""
import numpy as np


def shard_range(n_frames, rank, world):
    """contiguous block [lo, hi) of frames owned by `rank`; blocks differ in size by at most one frame"""
    base, rem = divmod(int(n_frames), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def broadcast_operand(arr, src=0, device=None):
    """broadcast a small numpy operand (taps, template, matrix) from rank `src`; returns the numpy array on every rank.
    Works with any initialised torch.distributed backend; a no-op without one."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return np.asarray(arr)
    a = np.ascontiguousarray(arr)
    t = torch.from_numpy(a.copy())
    if device is not None:
        t = t.to(device)
    dist.broadcast(t, src)
    return t.cpu().numpy()


def gather_counts(local_count, device=None):
    """per-rank frame counts (for reporting whole-job throughput)"""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [int(local_count)]
    t = torch.tensor([int(local_count)], dtype=torch.int64, device=device)
    out = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t)
    return [int(x.item()) for x in out]


# ---------------------------------------------------------------------------------------------------------------------------
# ctypes mirror of include/b200cv_batch.h: one driver over several GPUs of the box (worker thread + streams per device inside the
# library), or over ONE device when a process group (torchrun, one process per GPU) owns the sharding.
# ---------------------------------------------------------------------------------------------------------------------------
class BatchDriver:
    """host batches (numpy, cv::Mat layout, shape (N,H,W,C)) sharded over `devices` (None = every visible GPU)"""

    def __init__(self, devices=None):
        import ctypes
        from . import _check, lib
        self._ct, self._check, self._L = ctypes, _check, lib()
        self._h = ctypes.c_void_p()
        if devices is None:
            rc = self._L.b200cv_batch_create(ctypes.byref(self._h), None, 0)
        else:
            arr = (ctypes.c_int * len(devices))(*[int(d) for d in devices])
            rc = self._L.b200cv_batch_create(ctypes.byref(self._h), arr, len(devices))
        _check(rc, "batch_create")
        self._regions = []

    # -- bookkeeping ---------------------------------------------------------------------------------------------------------
    @property
    def n_devices(self):
        return int(self._L.b200cv_batch_device_count(self._h))

    @property
    def devices(self):
        return [int(self._L.b200cv_batch_device(self._h, i)) for i in range(self.n_devices)]

    @property
    def uses_nccl(self):
        return bool(self._L.b200cv_batch_uses_nccl(self._h))

    def last_counts(self):
        return [int(self._L.b200cv_batch_last_count(self._h, i)) for i in range(self.n_devices)]

    def shard(self, frames, index):
        ct = self._ct
        f, c = ct.c_int(), ct.c_int()
        self._check(self._L.b200cv_batch_shard(int(frames), int(index), self.n_devices, ct.byref(f), ct.byref(c)), "batch_shard")
        return f.value, f.value + c.value

    def pinned_frames(self, shape, dtype):
        """contiguous page-locked (N,H,W,C) batch whose frame blocks sit on the NUMA node of the device that owns them"""
        ct = self._ct
        shape = tuple(int(x) for x in shape)
        fb = int(np.prod(shape[1:])) * np.dtype(dtype).itemsize
        p = ct.c_void_p()
        self._check(self._L.b200cv_batch_host_alloc_frames(self._h, ct.byref(p), ct.c_size_t(fb), shape[0]), "batch_host_alloc_frames")
        buf = (ct.c_ubyte * (fb * shape[0])).from_address(p.value)
        self._regions.append((p, buf))
        return np.frombuffer(buf, dtype=dtype).reshape(shape)

    def close(self):
        if self._h:
            self._regions.clear()
            self._L.b200cv_batch_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # noqa: BLE001 -- interpreter shutdown
            pass

    # -- ops (names and argument meaning of opencv_b200.hal) -------------------------------------------------------------------
    def _io(self, src, dst, **new):
        from . import hal
        dst = dst if dst is not None else hal._new(src, **new)
        return dst, hal.describe(src), hal.describe(dst)

    def GaussianBlur(self, src, ksize, sigmaX, sigmaY=0, borderType=4, dst=None):
        ct = self._ct
        dst, ms, md = self._io(src, dst)
        self._check(self._L.b200cv_batch_gaussian_blur(self._h, ct.byref(ms), ct.byref(md), int(ksize[0]), int(ksize[1]), ct.c_double(sigmaX), ct.c_double(sigmaY),
                                                       int(borderType)), "batch GaussianBlur")
        return dst

    def sepFilter2D(self, src, ddepth, kernelX, kernelY, anchor=(-1, -1), delta=0.0, borderType=4, dst=None):
        ct = self._ct
        from . import hal
        dst, ms, md = self._io(src, dst, dtype=hal._ddt(src, ddepth))
        kx = np.ascontiguousarray(kernelX, np.float32).reshape(-1); ky = np.ascontiguousarray(kernelY, np.float32).reshape(-1)
        self._check(self._L.b200cv_batch_sep_filter2d(self._h, ct.byref(ms), ct.byref(md), kx.ctypes.data_as(ct.c_void_p), len(kx), ky.ctypes.data_as(ct.c_void_p), len(ky),
                                                      int(anchor[0]), int(anchor[1]), ct.c_double(delta), int(borderType)), "batch sepFilter2D")
        return dst

    def filter2D(self, src, ddepth, kernel, anchor=(-1, -1), delta=0.0, borderType=4, dst=None):
        ct = self._ct
        from . import hal
        dst, ms, md = self._io(src, dst, dtype=hal._ddt(src, ddepth))
        k = np.ascontiguousarray(kernel, np.float32)
        self._check(self._L.b200cv_batch_filter2d(self._h, ct.byref(ms), ct.byref(md), k.ctypes.data_as(ct.c_void_p), k.shape[1], k.shape[0], int(anchor[0]), int(anchor[1]),
                                                  ct.c_double(delta), int(borderType)), "batch filter2D")
        return dst

    def resize(self, src, dsize, fx=0, fy=0, interpolation=1, dst=None):
        ct = self._ct
        from . import hal
        m = hal.describe(src)
        if not dsize or dsize[0] <= 0:
            dsize = (int(round(m.cols * fx)), int(round(m.rows * fy)))
        else:
            fx = fy = 0.0          # scale = dsize / ssize
        dst, ms, md = self._io(src, dst, size=(int(dsize[0]), int(dsize[1])))
        self._check(self._L.b200cv_batch_resize(self._h, ct.byref(ms), ct.byref(md), int(interpolation), ct.c_double(fx), ct.c_double(fy)), "batch resize")
        return dst

    def _warp(self, fn, name, src, M, dsize, flags, borderMode, borderValue, dst):
        ct = self._ct
        dst, ms, md = self._io(src, dst, size=(int(dsize[0]), int(dsize[1])))
        m = np.ascontiguousarray(M, np.float64).reshape(-1)
        bv = np.zeros(4, np.float64); b = np.atleast_1d(np.asarray(borderValue, np.float64)); bv[:len(b)] = b
        self._check(fn(self._h, ct.byref(ms), ct.byref(md), m.ctypes.data_as(ct.c_void_p), int(flags), int(borderMode), bv.ctypes.data_as(ct.c_void_p)), name)
        return dst

    def warpAffine(self, src, M, dsize, flags=1, borderMode=0, borderValue=0, dst=None):
        return self._warp(self._L.b200cv_batch_warp_affine, "batch warpAffine", src, M, dsize, flags, borderMode, borderValue, dst)

    def warpPerspective(self, src, M, dsize, flags=1, borderMode=0, borderValue=0, dst=None):
        return self._warp(self._L.b200cv_batch_warp_perspective, "batch warpPerspective", src, M, dsize, flags, borderMode, borderValue, dst)

    def cvtColor(self, src, code, dstCn=0, dst=None):
        ct = self._ct
        from . import _cvt_dst_geometry, hal
        m = hal.describe(src)
        w, h, dcn = _cvt_dst_geometry(int(code), m.cols, m.rows, dstCn)
        dst, ms, md = self._io(src, dst, channels=dcn, size=(w, h))
        self._check(self._L.b200cv_batch_cvt_color(self._h, ct.byref(ms), ct.byref(md), int(code)), "batch cvtColor")
        return dst

    def cornerHarris(self, src, blockSize, ksize, k, borderType=4, dst=None):
        ct = self._ct
        dst, ms, md = self._io(src, dst, dtype=np.float32)
        self._check(self._L.b200cv_batch_corner_harris(self._h, ct.byref(ms), ct.byref(md), int(blockSize), int(ksize), ct.c_double(k), int(borderType)), "batch cornerHarris")
        return dst

    def matchTemplate(self, image, templ, method, result=None):
        ct = self._ct
        from . import hal
        mi, mt = hal.describe(image), hal.describe(templ)
        if result is None:
            result = np.empty((max(mi.frames, 1), mi.rows - mt.rows + 1, mi.cols - mt.cols + 1, 1), np.float32)
        mr = hal.describe(result)
        self._check(self._L.b200cv_batch_match_template(self._h, ct.byref(mi), ct.byref(mt), ct.byref(mr), int(method)), "batch matchTemplate")
        return result

    def sift_harris(self, src, harris=None, nOctaveLayers=3, sigma=1.6, upscale=1, blockSize=2, ksize=3, k=0.04, wave=4, consumer=None):
        """bench.py workload c5: SIFT pyramid + DoG and cornerHarris over a sharded (N,H,W,1) uint8 batch, `wave` frames per device at a time.
        harris: (N,H,W,1) float32 host batch or None.  consumer(device_index, first_frame, n_frames, gauss_ptr, gauss_stride, dog_ptr, dog_stride,
        harris_ptr, harris_step, harris_frame_step) -> 0, called on the worker threads with DEVICE pointers after every wave."""
        ct = self._ct
        from . import hal
        ms = hal.describe(src)
        mh = hal.describe(harris) if harris is not None else None
        CB = ct.CFUNCTYPE(ct.c_int, ct.c_void_p, ct.c_int, ct.c_int, ct.c_int, ct.c_void_p, ct.c_size_t, ct.c_void_p, ct.c_size_t, ct.c_void_p, ct.c_size_t, ct.c_size_t)
        cb = CB(lambda user, *a: int(consumer(*a) or 0)) if consumer is not None else ct.cast(None, CB)
        self._check(self._L.b200cv_batch_sift_harris(self._h, ct.byref(ms), ct.byref(mh) if mh is not None else None, int(nOctaveLayers), ct.c_double(sigma), int(upscale),
                                                     int(blockSize), int(ksize), ct.c_double(k), int(wave), cb, None), "batch sift_harris")
        return harris
