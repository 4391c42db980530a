// Column gather of many time-major tensors in one launch: the minibatch assembly of PPO epochs (DotaOptimizer.train_epochs).
//
// For every descriptor d, o < outer and j < n_index:
//   dst[(o*n_index + j)*row_bytes + b] = src[(o*src_cols + index[j])*row_bytes + b]
// i.e. torch.index_select(t, 1, index) on a contiguous [outer, src_cols, row] tensor ([S, B, ...] experience tensors and the
// [L, B, H] initial states), for up to DC_GATHER_MAX_TENSORS tensors at once.
//
// Work is counted in copy units of 16, 4 or 1 bytes, chosen per descriptor on the host (16 when row_bytes and both base
// pointers are multiples of 16, else 4 for the same test with 4, else 1).  Each block copies kUnitsPerBlock consecutive
// DESTINATION units of one descriptor; the blocks of all descriptors are numbered by a host prefix sum passed in the
// parameters, so a small tensor occupies a few blocks and no thread waits on another tensor's work.  Consecutive lanes
// write consecutive units (destination rows j..j+k of one o are contiguous), so every warp store is one contiguous run;
// the reads are contiguous within a source row.  Each thread issues its kUnroll loads before its stores.
//
// HBM traffic: outer*n_index*row_bytes read and the same written per descriptor, plus the index (L1/L2 resident).
//
// kFill (dc_gather_columns_fill): an index value < 0 writes a row of zeros and reads nothing.  The state refresh between
// PPO epochs uses it to build the rollout-major [T, R, ...] inputs of each time block from a training batch (rows the
// batch does not hold are zeros, as in experience prep) and to bring rollout-major values back into the batch layout.
// Bytes as above, less the rows a negative index skips on the read side.
#include <climits>
#include "dc_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr int kUnitsPerBlock = kThreads * kUnroll;

struct GatherParams {
    dc_gather_desc d[DC_GATHER_MAX_TENSORS];
    long long block_start[DC_GATHER_MAX_TENSORS + 1];   // first block of descriptor k; block_start[n_desc] = grid size
    int unit[DC_GATHER_MAX_TENSORS];                     // copy unit in bytes: 16, 4 or 1
    int narrow[DC_GATHER_MAX_TENSORS];                   // 1: every unit offset of the descriptor fits in 32 bits
    int n_desc;
};

// Copies units [u0, u0 + kUnitsPerBlock) of the destination, clipped to `total`.  I is the index type of the unit
// arithmetic: 32-bit division is several times cheaper than 64-bit, and the byte path is division-bound.
template <bool kFill, typename V, typename I>
__device__ __forceinline__ void gather_units(const V *__restrict__ src, V *__restrict__ dst, const int64_t *__restrict__ index,
                                             I row_units, I n_index, I src_cols, I total, I u0) {
    V v[kUnroll];
    I at[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
        const I u = u0 + (I)(k * kThreads + threadIdx.x);
        at[k] = u;
        if (u < total) {
            const I row = u / row_units, b = u - row * row_units;
            const I o = row / n_index, j = row - o * n_index;
            if constexpr (kFill) {
                const int64_t s = index[j];
                v[k] = s < 0 ? V{} : src[(o * src_cols + (I)s) * row_units + b];
            } else {
                v[k] = src[(o * src_cols + (I)index[j]) * row_units + b];
            }
        }
    }
#pragma unroll
    for (int k = 0; k < kUnroll; ++k)
        if (at[k] < total) dst[at[k]] = v[k];
}

template <bool kFill, typename V>
__device__ __forceinline__ void gather_desc(const dc_gather_desc &d, int narrow, const int64_t *__restrict__ index,
                                            int64_t n_index, long long block) {
    const int64_t row_units = d.row_bytes / (int64_t)sizeof(V);
    const int64_t total = d.outer * n_index * row_units;
    const int64_t u0 = block * kUnitsPerBlock;
    const V *src = static_cast<const V *>(d.src);
    V *dst = static_cast<V *>(d.dst);
    if (narrow)
        gather_units<kFill, V, uint32_t>(src, dst, index, (uint32_t)row_units, (uint32_t)n_index, (uint32_t)d.src_cols,
                                  (uint32_t)total, (uint32_t)u0);
    else
        gather_units<kFill, V, int64_t>(src, dst, index, row_units, n_index, d.src_cols, total, u0);
}

template <bool kFill>
__global__ void __launch_bounds__(kThreads) gather_columns_kernel(const __grid_constant__ GatherParams p,
                                                                  const int64_t *__restrict__ index, int64_t n_index) {
    const long long b = blockIdx.x;
    int k = 0;
    while (k + 1 < p.n_desc && b >= p.block_start[k + 1]) ++k;      // block-uniform, at most 31 steps
    const long long block = b - p.block_start[k];
    switch (p.unit[k]) {
        case 16: gather_desc<kFill, uint4>(p.d[k], p.narrow[k], index, n_index, block); break;
        case 4: gather_desc<kFill, uint32_t>(p.d[k], p.narrow[k], index, n_index, block); break;
        default: gather_desc<kFill, uint8_t>(p.d[k], p.narrow[k], index, n_index, block); break;
    }
}

bool aligned(const void *p, int64_t a) { return reinterpret_cast<uintptr_t>(p) % (uintptr_t)a == 0; }

template <bool kFill>
int gather_launch(const char *name, const dc_gather_desc *descs, int n_desc, const int64_t *index, int64_t n_index,
                  dc_stream_t stream) {
    DC_REQUIRE(n_desc >= 0 && n_desc <= DC_GATHER_MAX_TENSORS, DC_EINVAL, "%s: n_desc=%d outside [0, %d]", name,
               n_desc, DC_GATHER_MAX_TENSORS);
    DC_REQUIRE(n_index >= 0, DC_EINVAL, "%s: n_index=%lld < 0", name, (long long)n_index);
    if (n_desc == 0) return DC_OK;
    DC_REQUIRE(descs, DC_EINVAL, "%s: null descriptor array", name);
    for (int k = 0; k < n_desc; ++k) {
        const dc_gather_desc &d = descs[k];
        DC_REQUIRE(d.row_bytes > 0 && d.outer >= 0 && d.src_cols >= 0, DC_EINVAL,
                   "%s: descriptor %d has outer=%lld src_cols=%lld row_bytes=%lld (need outer >= 0, "
                   "src_cols >= 0, row_bytes > 0)", name, k, (long long)d.outer, (long long)d.src_cols, (long long)d.row_bytes);
    }
    if (n_index == 0) return DC_OK;
    DC_REQUIRE(index, DC_EINVAL, "%s: null index", name);
    GatherParams p;
    p.n_desc = n_desc;
    long long blocks = 0;
    for (int k = 0; k < n_desc; ++k) {
        const dc_gather_desc &d = descs[k];
        p.d[k] = d;
        p.block_start[k] = blocks;
        p.unit[k] = 1;
        p.narrow[k] = 1;
        if (d.outer == 0) continue;
        DC_REQUIRE(d.src && d.dst, DC_EINVAL, "%s: descriptor %d has a null pointer", name, k);
        DC_REQUIRE(d.src_cols > 0, DC_EINVAL, "%s: descriptor %d has src_cols=0 and %lld indices", name, k,
                   (long long)n_index);
        DC_REQUIRE(n_index <= INT64_MAX / d.outer && d.outer * n_index <= INT64_MAX / d.row_bytes &&
                       d.src_cols <= INT64_MAX / d.outer && d.outer * d.src_cols <= INT64_MAX / d.row_bytes,
                   DC_EINVAL, "%s: descriptor %d is too large", name, k);
        const int64_t dst_bytes = d.outer * n_index * d.row_bytes, src_bytes = d.outer * d.src_cols * d.row_bytes;
        const uintptr_t s = reinterpret_cast<uintptr_t>(d.src), t = reinterpret_cast<uintptr_t>(d.dst);
        DC_REQUIRE(t + (uintptr_t)dst_bytes <= s || s + (uintptr_t)src_bytes <= t, DC_EINVAL,
                   "%s: descriptor %d: dst overlaps src", name, k);
        if (d.row_bytes % 16 == 0 && aligned(d.src, 16) && aligned(d.dst, 16))
            p.unit[k] = 16;
        else if (d.row_bytes % 4 == 0 && aligned(d.src, 4) && aligned(d.dst, 4))
            p.unit[k] = 4;
        const int64_t src_units = src_bytes / p.unit[k], dst_units = dst_bytes / p.unit[k];
        // the last block's unit offsets reach (blocks * kUnitsPerBlock); both must stay below 2^32 for the 32-bit path
        const int64_t nb = (dst_units + kUnitsPerBlock - 1) / kUnitsPerBlock;
        p.narrow[k] = src_units <= (int64_t)UINT32_MAX && nb * kUnitsPerBlock <= (int64_t)UINT32_MAX;
        blocks += nb;
    }
    p.block_start[n_desc] = blocks;
    DC_REQUIRE(blocks <= INT_MAX, DC_EUNSUPPORTED, "%s: %lld blocks exceed the grid limit", name, blocks);
    if (blocks == 0) return DC_OK;
    gather_columns_kernel<kFill><<<(unsigned)blocks, kThreads, 0, dc_cu_stream(stream)>>>(p, index, n_index);
    DC_LAUNCH_OK();
    return DC_OK;
}

}  // namespace

extern "C" int dc_gather_columns(const dc_gather_desc *descs, int n_desc, const int64_t *index, int64_t n_index,
                                 dc_stream_t stream) {
    return gather_launch<false>("dc_gather_columns", descs, n_desc, index, n_index, stream);
}

extern "C" int dc_gather_columns_fill(const dc_gather_desc *descs, int n_desc, const int64_t *index, int64_t n_index,
                                      dc_stream_t stream) {
    return gather_launch<true>("dc_gather_columns_fill", descs, n_desc, index, n_index, stream);
}
