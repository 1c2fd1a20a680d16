// wgmma.cuh -- Hopper warpgroup MMA (wgmma.mma_async) plumbing for the Toeplitz tensor-core kernels (matchtemplate_tc.cu,
// filter2d_tc.cu, filter2d_tc_f32.cu).
//
// A warpgroup (four consecutive warps, 128 threads) issues one wgmma for a 64-row slab of D; the accumulators live in the registers
// of its threads.  Thread t = 32 w + l of the warpgroup holds, for every 8-column block j of D, the elements
//   d[4 j + 2 i + c] = D[16 w + l / 4 + 8 i][8 j + 2 (l % 4) + c]          (i, c in {0, 1})
// Operands are read from shared memory through 64-bit matrix descriptors in the K-major, no-swizzle core-matrix layout: a core
// matrix is 8 rows of 16 contiguous bytes (128 B); LBO = byte distance between core matrices adjacent in K, SBO = between core
// matrices adjacent in M (A) or N (B).
#pragma once
#include <stdint.h>

namespace b200cv {

// K-major, no swizzle: start >> 4 at [0,14) | LBO >> 4 at [16,30) | SBO >> 4 at [32,46); base offset 0, layout type 0 (bits 62-63)
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// orders this thread's register accesses before the wgmma instructions that follow (required before the first one)
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins accumulator registers at this point of the program: reads after wg_wait cannot be hoisted above it
template <int R>
__device__ __forceinline__ void wg_fence_operand(uint32_t (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+r"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void wg_fence_operand(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// arrive on `bar` from the threads where `pred` holds.  Predicated rather than branched: a branch between wgmma groups in flight makes
// ptxas serialise the MMAs.
__device__ __forceinline__ void wg_mbar_arrive_if(uint64_t* bar, bool pred)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}"
                 ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"((uint32_t)pred) : "memory");
}
// named barriers (ids 1..15; 0 is __syncthreads) between warpgroups.  `n` counts every thread taking part, arriving and waiting.
// wg_bar_arrive does not wait.  Between wgmma groups in flight use it unconditionally: even a predicated bar.arrive there makes ptxas
// serialise the MMAs (C7520).  wg_bar_sync_if takes a `pred` uniform over each warp.
__device__ __forceinline__ void wg_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void wg_bar_sync_if(int id, int n, bool pred)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p bar.sync %0, %1;\n\t}" ::"r"(id), "r"(n), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ void wg_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// one bulk copy global -> shared, completion signalled on `bar` with the byte count
__device__ __forceinline__ void wg_bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(bar)) : "memory");
}

// D[64 x 64] += A[64 x 32] * B[32 x 64], u8 x u8 -> s32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_u8u8_n64(uint32_t (&d)[32], uint64_t adesc, uint64_t bdesc)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.u8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
                   "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
                   "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(adesc), "l"(bdesc) : "memory");
}

// D[64 x 48] += A[64 x 32] * B[32 x 48], u8 x s8 -> s32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_u8s8_n48(uint32_t (&d)[24], uint64_t adesc, uint64_t bdesc)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n48k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
                   "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23])
                 : "l"(adesc), "l"(bdesc) : "memory");
}

// D[64 x 96] += A[64 x 32] * B[32 x 96], u8 x s8 -> s32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_u8s8_n96(uint32_t (&d)[48], uint64_t adesc, uint64_t bdesc)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n96k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
                   "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
                   "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]),
                   "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47])
                 : "l"(adesc), "l"(bdesc) : "memory");
}

// D[64 x 64] += A[64 x 16] * B[16 x 64], bf16 x bf16 -> f32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(adesc), "l"(bdesc) : "memory");
}

// D[64 x 32] += A[64 x 16] * B[16 x 32], bf16 x bf16 -> f32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(adesc), "l"(bdesc) : "memory");
}


}  // namespace b200cv
