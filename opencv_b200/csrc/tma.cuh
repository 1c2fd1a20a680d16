// tma.cuh -- Tensor Memory Accelerator plumbing (sm_90a): tensor-map creation on the host (through the driver entry point,
// no link-time dependency on libcuda) and the mbarrier / cp.async.bulk.tensor PTX wrappers used by the tile kernels.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "common.cuh"

namespace b200cv {

// 3-D tiled tensor map over a batch of row-major images: dims (x = cols [elements], y = rows, z = frames).
// Requirements (cuTensorMapEncodeTiled): base 16-byte aligned, step and frame step multiples of 16, box_w*elem multiple of 16,
// box dims <= 256.  Out-of-bounds box elements are filled with ZEROS.
int make_tensor_map_3d(CUtensorMap* map, const void* base, int elem_bytes, int cols, int rows, int frames, size_t step, size_t fstep,
                       int box_w, int box_h);
// Kernels take the descriptor as a `const __grid_constant__ CUtensorMap` parameter (no allocation, and above all no small H2D copy
// per launch: on the host path such a copy queues behind the bulk frame uploads on the copy engine and stalls the kernel that
// needs it -- measured as a 2-4x loss of end-to-end throughput).  upload_tensor_map (descriptor in global memory) is kept for
// tools/tma_test.cu.
int upload_tensor_map(const CUtensorMap& tm, CUtensorMap** dptr, cudaStream_t st);
static inline bool tma_compatible(const Img& m) { return (((uintptr_t)m.data | m.step | m.fstep) & 15) == 0; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    while (!mbar_try_wait(bar, parity)) {}
}
// one 3-D box: global (x, y, z) -> shared, completion signalled on `bar` with the byte count
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, int x, int y, int z, uint64_t* bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_u32(smem_dst)), "l"(map), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) { asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory"); }

}  // namespace b200cv
