// tc05.cuh -- thin inline-PTX layer over the Hopper (sm_90a) tensor path used by ozaki.cu:
// mbarrier, bulk async copies executed by the TMA unit (cp.async.bulk), warpgroup MMA (wgmma.mma_async, s8 x s8 with
// int32 accumulation in registers).
// Bit layout of the shared-memory matrix descriptor follows the PTX ISA ("Matrix Descriptor Format" of the
// asynchronous warpgroup-level matrix instructions).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {
namespace sm90 {

__device__ __forceinline__ uint32_t smem_addr(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
// make barrier initialisation visible to the async proxy (TMA unit)
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_addr(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_addr(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Wait for the phase with the given parity.  A kernel must never hang the device: after `limit` polls
// (~seconds) the wait gives up, raises *abort_flag and returns false; callers unwind.
__device__ __forceinline__ bool mbar_wait(uint64_t *bar, uint32_t parity, volatile int *abort_flag,
                                          uint32_t limit = 1u << 26) {
    for (uint32_t it = 0; it < limit; ++it) {
        if (mbar_try_wait(bar, parity)) return true;
        if ((it & 1023u) == 1023u && *abort_flag) return false;
    }
    *abort_flag = 1;
    return false;
}

// ---- bulk async copy global -> shared (TMA unit), completion on an mbarrier ---------------------------
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
            smem_addr(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_addr(bar))
        : "memory");
}

// ---- shared-memory matrix descriptor ----------------------------------------------------------------
//   bits [0,14)  start address >> 4     bits [16,30) leading byte offset >> 4 (K direction between core matrices)
//   bits [32,46) stride byte offset >> 4 (M/N direction between 8-row core matrices)
//   bits [62,64) layout: 0 = no swizzle (interleaved core matrices of 8 rows x 16 bytes), 1 = 128B, 2 = 64B, 3 = 32B
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}

// ---- warpgroup MMA -----------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }

// D (64 x 64, int32, registers of the warpgroup) (+)= A (64 x 32 bytes of K, smem) . B (64 x 32 bytes of K, smem)^T,
// both operands signed 8-bit and K-major.  Fragment of D held by thread (warp w, lane l) of the warpgroup:
//   d[4j + 0] = D[16w + l/4][8j + 2(l%4)]      d[4j + 1] = D[16w + l/4][8j + 2(l%4) + 1]
//   d[4j + 2] = D[16w + l/4 + 8][8j + 2(l%4)]  d[4j + 3] = D[16w + l/4 + 8][8j + 2(l%4) + 1]      (j = 0..7)
__device__ __forceinline__ void wgmma_s8_m64n64k32(uint32_t (&d)[32], uint64_t a_desc, uint64_t b_desc,
                                                   uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n\t}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
          "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]),
          "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
          "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

}  // namespace sm90
}  // namespace b200
