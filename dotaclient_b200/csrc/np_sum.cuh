// numpy's float32 reduction order, shared by the advantage scans (gae_scan.cu, vtrace_scan.cu) so that both reduce the
// per-step sub-rewards bit-identically to np.sum(rewards, axis=1) (optimizer.py:397).
#pragma once

namespace dc {

// numpy's pairwise float32 add-reduce over a contiguous axis of n < 128 elements at(0) .. at(n-1) (8 accumulators,
// combined as ((0+1)+(2+3))+((4+5)+(6+7)), remainder added sequentially).
template <class At>
__device__ __forceinline__ float np_sum(int n, At at) {
    if (n == 1) return at(0);
    if (n < 8) {
        float s = at(0);
        for (int i = 1; i < n; ++i) s = __fadd_rn(s, at(i));
        return s;
    }
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = at(j);
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], at(i + j));
    }
    float s = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                        __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) s = __fadd_rn(s, at(i));
    return s;
}

// np.sum(p[:n]) for a contiguous row.
__device__ __forceinline__ float np_sum_row(const float *__restrict__ p, int n) {
    return np_sum(n, [p](int i) { return p[i]; });
}

}  // namespace dc
