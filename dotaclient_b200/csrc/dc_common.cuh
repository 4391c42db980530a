// Shared helpers for the dotaclient_b200 CUDA sources (sm_90a: H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "dotaclient_b200.h"

// Records a message retrievable through dc_last_error() (thread-local).
void dc_set_error(const char *fmt, ...);

#define DC_REQUIRE(cond, code, ...)        \
    do {                                   \
        if (!(cond)) {                     \
            dc_set_error(__VA_ARGS__);     \
            return (code);                 \
        }                                  \
    } while (0)

#define DC_CUDA(call)                                                                      \
    do {                                                                                   \
        cudaError_t e__ = (call);                                                          \
        if (e__ != cudaSuccess) {                                                          \
            dc_set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,              \
                         cudaGetErrorString(e__));                                         \
            return (int)e__;                                                               \
        }                                                                                  \
    } while (0)

#define DC_LAUNCH_OK() DC_CUDA(cudaGetLastError())

static inline cudaStream_t dc_cu_stream(dc_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// Number of SMs of the current device (cached per device; 132 on H100 SXM).
int dc_sm_count();

// csrc/gemm_tf32x3.cu: split-K wgmma 3xTF32 GEMM writing `ksplit` partial [M, N] products (library-internal).
int dc_gemm_tf32x3_splitk(const float *A, int lda, const float *B, int ldb, float *part, int64_t M, int N, int K, int ksplit,
                          bool first_call, cudaStream_t st);

// csrc/encoder.cu: dW_b / db_b (+)= the fixed-order sum of `nblocks` [128][13] partials (library-internal).
int dc_unit_basic_reduce(const float *partial, int nblocks, float *dw_b, float *db_b, int accumulate, cudaStream_t st);

__device__ __forceinline__ float dc_sigmoid(float x) { return 1.0f / (1.0f + __expf(-x)); }
// tanh via one exp; abs error ~1e-7, saturates cleanly for |x| large.
__device__ __forceinline__ float dc_tanh(float x) { return 1.0f - 2.0f / (__expf(2.0f * x) + 1.0f); }

// Two independent FMAs on (x, y) pairs, each rounded to nearest.
__device__ __forceinline__ float2 dc_ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

// ---- Hopper tensor-core helpers (wgmma) shared by csrc/gemm_tf32x3.cu and csrc/rnn_cluster.cuh ----
__device__ __forceinline__ uint32_t dc_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
// round-to-nearest, ties away from zero, to 10 mantissa bits (cvt.rna.tf32.f32 for finite inputs): the hi half of a
// 3xTF32 split; v - hi is exact in fp32 and is the lo half.
__device__ __forceinline__ float dc_tf32_rna(float v) { return __uint_as_float((__float_as_uint(v) + 0x1000u) & 0xffffe000u); }
// wgmma shared-memory matrix descriptor of a K-major SWIZZLE_128B tile (rows of 128 bytes = 32 tf32, 8-row groups 1024 B
// apart, 1024-byte aligned base): start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major) | SBO>>4 [32,46) |
// layout type 1 = SWIZZLE_128B [62,64).  Advancing K by 8 tf32 (32 bytes) inside the swizzle row adds 2 to the descriptor.
__device__ __forceinline__ uint64_t dc_wgmma_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void dc_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void dc_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void dc_wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of an accumulator register across the asynchronous wgmma and its wait
__device__ __forceinline__ void dc_reg_fence(float &r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void dc_mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(dc_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void dc_mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(dc_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void dc_mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(ok)
                     : "r"(dc_smem_u32(bar)), "r"(parity)
                     : "memory");
    } while (!ok);
}

__device__ __forceinline__ float dc_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double dc_warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
