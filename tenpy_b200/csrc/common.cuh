// common.cuh -- shared helpers of libb200npc (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>

#include "../../include/b200npc.h"

namespace b200 {

// ---- error handling ---------------------------------------------------------------------------
extern thread_local std::string g_last_error;
int set_error(int code, const char *fmt, ...);

#define B200_CUDA_CHECK(expr)                                                                        \
    do {                                                                                             \
        cudaError_t _e = (expr);                                                                     \
        if (_e != cudaSuccess)                                                                       \
            return b200::set_error(B200_ERR_CUDA, "%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, \
                                   cudaGetErrorString(_e));                                          \
    } while (0)

#define B200_CHECK_LAUNCH()                                                                          \
    do {                                                                                             \
        b200::g_kernel_launches.fetch_add(1, std::memory_order_relaxed);                             \
        cudaError_t _e = cudaGetLastError();                                                         \
        if (_e != cudaSuccess)                                                                       \
            return b200::set_error(B200_ERR_CUDA, "kernel launch failed at %s:%d: %s", __FILE__,       \
                                   __LINE__, cudaGetErrorString(_e));                                \
    } while (0)

int sm_count();  // SM count of the current device (cached)
extern std::atomic<long long> g_kernel_launches;  // every kernel launch of this library is counted

// ---- FP64 tensor-core MMA (DMMA) -----------------------------------------------------------------
// D(16x8) += A(16x8) * B(8x8), all f64.  Fragment ownership (lane = 4*g + t, g = 0..7, t = 0..3):
//   a0 = A[g][t]      a1 = A[g+8][t]      a2 = A[g][t+4]      a3 = A[g+8][t+4]
//   b0 = B[t][g]      b1 = B[t+4][g]
//   c0 = C[g][2t]     c1 = C[g][2t+1]     c2 = C[g+8][2t]     c3 = C[g+8][2t+1]
// Two implementations with identical semantics: one m16n8k8 instruction, or four m8n8k4 instructions.
#ifndef B200_DMMA_K4
#define B200_DMMA_K4 0
#endif

__device__ __forceinline__ void dmma_m8n8k4(double &c0, double &c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

__device__ __forceinline__ void dmma_16x8x8_k4(double (&c)[4], const double (&a)[4], const double (&b)[2]) {
    dmma_m8n8k4(c[0], c[1], a[0], b[0]);
    dmma_m8n8k4(c[0], c[1], a[2], b[1]);
    dmma_m8n8k4(c[2], c[3], a[1], b[0]);
    dmma_m8n8k4(c[2], c[3], a[3], b[1]);
}

__device__ __forceinline__ void dmma_16x8x8_k8(double (&c)[4], const double (&a)[4], const double (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
        "{%0,%1,%2,%3};\n"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}

__device__ __forceinline__ void dmma_16x8x8(double (&c)[4], const double (&a)[4], const double (&b)[2]) {
#if B200_DMMA_K4
    dmma_16x8x8_k4(c, a, b);
#else
    dmma_16x8x8_k8(c, a, b);
#endif
}

// ---- cp.async ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
// 16-byte async copy global->shared; src_bytes in {0,16}: 0 zero-fills the destination
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gsrc),
                 "r"(src_bytes));
}
// 8-byte async copy global->shared; src_bytes in {0,8}
__device__ __forceinline__ void cp_async8(void *smem_dst, const void *gsrc, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gsrc),
                 "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// ---- reductions ----------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// block-wide sum, result valid in thread 0; `red` = shared array of >= 32 doubles
__device__ __forceinline__ double block_sum(double v, double *red) {
    v = warp_sum(v);
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) red[w] = v;
    __syncthreads();
    int nw = (blockDim.x + 31) >> 5;
    double r = 0.0;
    if (w == 0) {
        r = (lane < nw) ? red[lane] : 0.0;
        r = warp_sum(r);
    }
    __syncthreads();
    return r;
}

}  // namespace b200
