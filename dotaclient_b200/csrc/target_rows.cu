// The tokens the target-unit head serves, as a row list on the device.
//
// The loss reads a token's target-unit logits only when its mask row or its action row has a bit set (ppo_loss.cu,
// head_token: other rows return before any use and get zero dlogits).  With the reference's data format that is a step at
// which the agent chose to attack (agent.py:665-671), a minority of the tokens.  dc_target_rows lists those tokens in
// ascending order, with their count, both on the device, so that the head and the GEMMs around it (the *_rows entry points)
// run on them alone and a captured graph replays whatever the count.
//
//   pass 1  one block per kTokBlk tokens: flag byte per token (mask | action row non-zero) + the block's count
//   pass 2  block b adds up the counts of blocks < b (its base), scans its flags and writes rows[base + rank]; the last
//           block writes the total.  Two launches, no atomics: the order is the token order, deterministic.
// The GEMMs on the list read their operand rows through it and write their dense outputs at rows[i] themselves
// (gemm_tf32x3.cu, kDevM / kDevT), so no row is copied; dc_rows_zero_inactive writes the zero rows of the inactive
// tokens into such a dense output -- nothing at all when every token is active.
#include "dc_common.cuh"

namespace {

constexpr int kRowBytes = 40;                  // target_unit mask / action row: 40 bool bytes (policy.py:76)
constexpr int kThreadsR = 256;
constexpr int kTokPerThread = 4;
constexpr int kTokBlk = kThreadsR * kTokPerThread;

__device__ __forceinline__ bool row_any(const uint8_t *__restrict__ m, const uint8_t *__restrict__ a, int64_t n) {
    // rows start at 40 n bytes: 8-byte aligned when the base is
    const uint2 *pm = reinterpret_cast<const uint2 *>(m + n * kRowBytes), *pa = reinterpret_cast<const uint2 *>(a + n * kRowBytes);
    uint32_t v = 0;
#pragma unroll
    for (int j = 0; j < kRowBytes / 8; ++j) {
        const uint2 x = __ldg(pm + j), y = __ldg(pa + j);
        v |= x.x | x.y | y.x | y.y;
    }
    return v != 0;
}

__global__ void __launch_bounds__(kThreadsR) target_flags_kernel(const uint8_t *__restrict__ mask, const uint8_t *__restrict__ action,
                                                                 int64_t N, uint8_t *__restrict__ flags, int *__restrict__ block_count) {
    __shared__ int s_warp[kThreadsR / 32];
    const int64_t base = (int64_t)blockIdx.x * kTokBlk;
    int c = 0;
#pragma unroll
    for (int j = 0; j < kTokPerThread; ++j) {
        const int64_t n = base + j * kThreadsR + threadIdx.x;       // consecutive threads, consecutive rows
        if (n < N) {
            const bool f = row_any(mask, action, n);
            flags[n] = f ? 1 : 0;
            c += f ? 1 : 0;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < kThreadsR / 32; ++w) t += s_warp[w];
        block_count[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kThreadsR) target_rows_kernel(const uint8_t *__restrict__ flags, const int *__restrict__ block_count,
                                                                int64_t N, int *__restrict__ rows, int *__restrict__ count) {
    __shared__ int s_warp[kThreadsR / 32];
    __shared__ int s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // base = sum of the counts of the blocks before this one
    int b = 0;
    for (int k = threadIdx.x; k < (int)blockIdx.x; k += kThreadsR) b += block_count[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) b += __shfl_xor_sync(0xffffffffu, b, o);
    if (lane == 0) s_warp[warp] = b;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < kThreadsR / 32; ++w) t += s_warp[w];
        s_base = t;
    }
    __syncthreads();
    // thread t owns tokens base + 4t .. 4t+3: exclusive scan of the per-thread counts over the block
    const int64_t t0 = (int64_t)blockIdx.x * kTokBlk + (int64_t)threadIdx.x * kTokPerThread;
    uint32_t f4 = 0;
    if (t0 + kTokPerThread <= N) {
        f4 = __ldg(reinterpret_cast<const uint32_t *>(flags + t0));    // t0 % 4 == 0: an aligned word
    } else {                                                       // the tail of the last block
        for (int j = 0; j < kTokPerThread; ++j)
            if (t0 + j < N) f4 |= (uint32_t)flags[t0 + j] << (8 * j);
    }
    const int mine = __popc(f4);
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    __syncthreads();                                               // s_warp is reused
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int before = s_base;
    for (int w = 0; w < warp; ++w) before += s_warp[w];
    int r = before + incl - mine;
#pragma unroll
    for (int j = 0; j < kTokPerThread; ++j)
        if ((f4 >> (8 * j)) & 0xffu) rows[r++] = (int)(t0 + j);
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == kThreadsR - 1) *count = r;    // the last thread of the last block ends the list
}

// dst[n, :width] = 0 for every n with flags[n] == 0: one warp per 32 tokens reads their flags, then zeroes the inactive rows
__global__ void __launch_bounds__(kThreadsR) zero_inactive_kernel(const uint8_t *__restrict__ flags, int64_t N, float *__restrict__ dst,
                                                                  int ld, int width) {
    const int lane = threadIdx.x & 31;
    const int64_t base = ((int64_t)blockIdx.x * kThreadsR + threadIdx.x - lane);
    if (base >= N) return;
    const bool mine = base + lane < N && flags[base + lane] == 0;
    uint32_t todo = __ballot_sync(0xffffffffu, mine);
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    while (todo) {
        const int r = __ffs(todo) - 1;
        todo &= todo - 1;
        float4 *d = reinterpret_cast<float4 *>(dst + (base + r) * ld);
        for (int c = lane; c < width / 4; c += 32) d[c] = z;
    }
}

int64_t flag_blocks(int64_t N) { return (N + kTokBlk - 1) / kTokBlk; }

}  // namespace

extern "C" size_t dc_target_rows_workspace_bytes(int64_t N) { return N <= 0 ? 0 : (size_t)flag_blocks(N) * sizeof(int); }

extern "C" int dc_target_rows(const uint8_t *mask, const uint8_t *action, int64_t N, int32_t *rows, int32_t *count, uint8_t *flags,
                              void *workspace, dc_stream_t stream) {
    DC_REQUIRE(mask && action && rows && count && flags && workspace && N > 0 && N < (1ll << 31) - kTokBlk, DC_EINVAL,
               "dc_target_rows: bad arguments");
    DC_REQUIRE((((uintptr_t)mask | (uintptr_t)action) & 7) == 0 && ((uintptr_t)flags & 3) == 0 && ((uintptr_t)workspace & 3) == 0,
               DC_EINVAL, "dc_target_rows: mask / action must be 8-byte aligned, flags and workspace 4-byte aligned");
    cudaStream_t st = dc_cu_stream(stream);
    int *block_count = reinterpret_cast<int *>(workspace);
    const unsigned blocks = (unsigned)flag_blocks(N);
    target_flags_kernel<<<blocks, kThreadsR, 0, st>>>(mask, action, N, flags, block_count);
    DC_LAUNCH_OK();
    target_rows_kernel<<<blocks, kThreadsR, 0, st>>>(flags, block_count, N, rows, count);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_rows_zero_inactive(const uint8_t *flags, int64_t N, float *dst, int ld, int width, dc_stream_t stream) {
    DC_REQUIRE(flags && dst && N > 0 && width > 0 && width % 4 == 0 && ld >= width && ld % 4 == 0 && ((uintptr_t)dst & 15) == 0,
               DC_EINVAL, "dc_rows_zero_inactive: bad arguments");
    zero_inactive_kernel<<<(unsigned)((N + kThreadsR - 1) / kThreadsR), kThreadsR, 0, dc_cu_stream(stream)>>>(flags, N, dst, ld, width);
    DC_LAUNCH_OK();
    return DC_OK;
}
