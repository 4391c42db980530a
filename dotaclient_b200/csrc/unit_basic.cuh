// The unit encoder's basic layer, relu(units W_b^T + b_b) (policy.py:100,105,...), as ONE definition of the value of a
// (row, channel) pair.  The activations are rebuilt from the 12 raw features wherever they are read -- the embedding GEMM's
// producers, the target-unit head, the ReLU mask of the fused data gradient -- so every kernel calls this function and the
// value is the same bit for bit everywhere: start from b_b[j], one fmaf per feature in order k = 0..11, then the ReLU.
#pragma once
#include "dc_common.cuh"

constexpr int kUnitFeatures = 12;                  // raw features per unit (policy.py:56)

__device__ __forceinline__ float dc_unit_basic(const float (&u)[kUnitFeatures], const float (&w)[kUnitFeatures], float b) {
    float a = b;
#pragma unroll
    for (int k = 0; k < kUnitFeatures; ++k) a = fmaf(u[k], w[k], a);
    return fmaxf(a, 0.f);
}
