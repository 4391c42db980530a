// Step-wise recurrence for the wide layers (H a multiple of 128 other than 128 / 256, e.g. BASELINE's H = 512).
//
// At H = 512 the fp32 W_hh (4 MB LSTM; 8 MB as tf32 hi + lo) fits neither one SM nor a 16-CTA cluster, so the weights cannot
// stay on chip across steps the way rnn_resident.cuh / rnn_cluster.cuh keep them.  The step is a genuine dense contraction
// ([B, H] x [H, G*H], 1.07 GFLOP per step at B = 512), so every step runs as
//     (1) the split-K wgmma 3xTF32 GEMM of csrc/gemm_tf32x3.cu over all SMs (W_hh streams from L2, where it stays
//         resident: 4 MB of 126 MB), writing `ksplit` partial products, and
//     (2) one elementwise gate kernel that sums the partials in a fixed order (deterministic) and applies the cell.
// 2 launches per time step; same buffers, same saved tensors and the same in-place reuse of the gate buffer as the other
// recurrence kernels (include/dotaclient_b200.h).  fp32-level accuracy like every other dense layer of the step.
#pragma once
#include "rnn_cell.cuh"

namespace dc_rnns {

inline bool stepwise_supported(int H) { return H % 128 == 0 && H != 128 && H != 256; }

// split-K factor: fill the SMs (tiles * ksplit <= #SM) with K ranges that stay multiples of 32 (one swizzle row)
inline int pick_ksplit(int64_t M, int N, int K) {
    const int tiles = (int)((M + 127) / 128) * (N / 128);
    int ks = 1;
    while (ks < 16 && tiles * ks * 2 <= dc_sm_count() && (K / 32) % (ks * 2) == 0) ks *= 2;
    return ks;
}

struct Workspace {
    float *wT, *part_f, *part_b, *dgbuf, *dh_carry, *dc_carry;
    int ksf, ksb;
    size_t total_floats;
};
inline Workspace carve(void *base, int cell, int B, int H) {
    const int G = cell == DC_CELL_GRU ? 3 : 4;
    Workspace w;
    w.ksf = pick_ksplit(B, G * H, H);
    w.ksb = pick_ksplit(B, H, G * H);
    float *p = reinterpret_cast<float *>(base);
    auto take = [&](size_t n) { float *q = p; p += (n + 63) / 64 * 64; return q; };
    w.wT = take((size_t)G * H * H);
    w.part_f = take((size_t)w.ksf * B * G * H);
    w.part_b = take((size_t)w.ksb * B * H);
    w.dgbuf = take((size_t)B * G * H);
    w.dh_carry = take((size_t)B * H);
    w.dc_carry = take((size_t)B * H);
    w.total_floats = (size_t)(p - reinterpret_cast<float *>(base));
    return w;
}
inline size_t workspace_bytes(int cell, int B, int H) { return carve(nullptr, cell, B, H).total_floats * sizeof(float); }

// ---- forward gate kernel: one thread per (sequence, unit) ---------------------------------------------------------------
// kReset: resets of step t from rs (rnn_cell.cuh); pre and prev of a reset token come from its tables, the GEMM's partials
// of the stale state are not read.
template <int G, bool kReset = false>
__global__ void __launch_bounds__(256) fwd_gate_kernel(float *__restrict__ gates_t, const float *__restrict__ part, int ksplit,
                                                       const float *__restrict__ b_hh, const float *__restrict__ h_prev,
                                                       const float *__restrict__ c_prev, float *__restrict__ h_next,
                                                       float *__restrict__ aux_next, int B, int H, dc_rnn::Reset rs, int t) {
    const int idx = blockIdx.x * 256 + threadIdx.x;
    if (idx >= B * H) return;
    const int b = idx / H, u = idx - b * H, GH = G * H;
    const size_t stride = (size_t)B * GH;
    float pre[G];
    float *g = gates_t + (size_t)b * GH + u;
    float act[G];
    if constexpr (kReset) {
        const int k = rs.slot[(size_t)t * B + b];
        float prev;
        if (k >= 0) {
            const size_t r = (size_t)k * B + b;
#pragma unroll
            for (int q = 0; q < G; ++q) pre[q] = rs.pre[r * GH + q * H + u];
            prev = rs.prev[r * H + u];
        } else {
#pragma unroll
            for (int q = 0; q < G; ++q) {
                float a = __ldg(b_hh + q * H + u);
                const float *p = part + (size_t)b * GH + q * H + u;
                for (int s = 0; s < ksplit; ++s) a += p[(size_t)s * stride];
                pre[q] = a;
            }
            prev = G == 3 ? h_prev[idx] : c_prev[idx];
        }
        h_next[idx] = dc_rnn::cell_fwd<G>([&](int q) { return g[q * H]; }, [&](int q) { return pre[q]; }, prev, act, aux_next[idx]);
    } else {
#pragma unroll
        for (int q = 0; q < G; ++q) {
            float a = __ldg(b_hh + q * H + u);
            const float *p = part + (size_t)b * GH + q * H + u;
            for (int s = 0; s < ksplit; ++s) a += p[(size_t)s * stride];
            pre[q] = a;
        }
        h_next[idx] = dc_rnn::cell_fwd<G>([&](int q) { return g[q * H]; }, [&](int q) { return pre[q]; },
                                          G == 3 ? h_prev[idx] : c_prev[idx], act, aux_next[idx]);   // aux: cbuf slot t+1
    }
#pragma unroll
    for (int q = 0; q < G; ++q) g[q * H] = act[q];
}

// ---- backward gate kernel -------------------------------------------------------------------------------------------------
// dh = dy_t + carry + sum of the previous step's partial products; writes dgi (in place of the saved gates), the h2h gate
// gradients (GEMM operand of this step) and the carries.  first != 0: the carries are initialised from dhn / dcn.
// kReset: at a reset token of step t (rs, rnn_cell.cuh) prev comes from the table, and the carries and the GEMM operand are
// zero, so that the next gate kernel (or bwd_final_kernel) receives exactly nothing from this token.
template <int G, bool kReset = false>
__global__ void __launch_bounds__(256) bwd_gate_kernel(float *__restrict__ gates_t, const float *__restrict__ dy_t,
                                                       const float *__restrict__ part, int ksplit, float *__restrict__ dh_carry,
                                                       float *__restrict__ dc_carry, const float *__restrict__ dhn,
                                                       const float *__restrict__ dcn, const float *__restrict__ h_prev,
                                                       const float *__restrict__ c_prev, float *aux_cur, float *__restrict__ dgbuf,
                                                       int first, int B, int H, dc_rnn::Reset rs, int t) {
    const int idx = blockIdx.x * 256 + threadIdx.x;
    if (idx >= B * H) return;
    const int b = idx / H, u = idx - b * H, GH = G * H;
    float dh = dy_t[idx];
    if (first) {
        if (dhn) dh += dhn[idx];
    } else {
        dh += dh_carry[idx];
        const size_t stride = (size_t)B * H;
        for (int s = 0; s < ksplit; ++s) dh += part[(size_t)s * stride + idx];
    }
    float *g = gates_t + (size_t)b * GH + u;
    float *dg = dgbuf + (size_t)b * GH + u;
    float dgi[G], dgh[G];
    float dc = G == 3 ? 0.f : first ? (dcn ? dcn[idx] : 0.f) : dc_carry[idx];
    if constexpr (kReset) {
        const int k = rs.slot[(size_t)t * B + b];
        const float prev = k >= 0 ? rs.prev[((size_t)k * B + b) * H + u] : G == 3 ? h_prev[idx] : c_prev[idx];
        const float dh_direct = dc_rnn::cell_bwd<G>([&](int q) { return g[q * H]; }, aux_cur[idx], prev, dh, dc, dgi, dgh);
        dh_carry[idx] = k >= 0 ? 0.f : dh_direct;
#pragma unroll
        for (int q = 0; q < G; ++q) { g[q * H] = dgi[q]; dg[q * H] = k >= 0 ? 0.f : dgh[q]; }
        if (G == 3) aux_cur[idx] = dgh[2];
        else dc_carry[idx] = k >= 0 ? 0.f : dc;
    } else {
        dh_carry[idx] = dc_rnn::cell_bwd<G>([&](int q) { return g[q * H]; }, aux_cur[idx], G == 3 ? h_prev[idx] : c_prev[idx], dh,
                                            dc, dgi, dgh);
#pragma unroll
        for (int q = 0; q < G; ++q) { g[q * H] = dgi[q]; dg[q * H] = dgh[q]; }
        if (G == 3) aux_cur[idx] = dgh[2];                   // n-gate part of dgh (cbuf slot t+1)
        else dc_carry[idx] = dc;
    }
}

__global__ void __launch_bounds__(256) bwd_final_kernel(const float *__restrict__ part, int ksplit, const float *__restrict__ dh_carry,
                                                        const float *__restrict__ dc_carry, float *__restrict__ dh0,
                                                        float *__restrict__ dc0, int n) {
    const int idx = blockIdx.x * 256 + threadIdx.x;
    if (idx >= n) return;
    float dh = dh_carry[idx];
    for (int s = 0; s < ksplit; ++s) dh += part[(size_t)s * n + idx];
    if (dh0) dh0[idx] = dh;
    if (dc0) dc0[idx] = dc_carry[idx];
}

template <bool kReset>
inline int launch_fwd(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf, float *cbuf, int B, int S, int H,
                      void *workspace, dc_rnn::Reset rs, cudaStream_t st) {
    const int G = cell == DC_CELL_GRU ? 3 : 4, GH = G * H;
    const Workspace w = carve(workspace, cell, B, H);
    const int blocks = (B * H + 255) / 256;
    const size_t BH = (size_t)B * H;
    for (int t = 0; t < S; ++t) {
        int rc = dc_gemm_tf32x3_splitk(ybuf + t * BH, H, w_hh, H, w.part_f, B, GH, H, w.ksf, t == 0, st);
        if (rc) return rc;
        float *gt = gates + (size_t)t * B * GH;
        if (G == 3)
            fwd_gate_kernel<3, kReset><<<blocks, 256, 0, st>>>(gt, w.part_f, w.ksf, b_hh, ybuf + t * BH, nullptr, ybuf + (t + 1) * BH, cbuf + (t + 1) * BH, B, H, rs, t);
        else
            fwd_gate_kernel<4, kReset><<<blocks, 256, 0, st>>>(gt, w.part_f, w.ksf, b_hh, ybuf + t * BH, cbuf + t * BH, ybuf + (t + 1) * BH, cbuf + (t + 1) * BH, B, H, rs, t);
    }
    DC_LAUNCH_OK();
    return DC_OK;
}

template <bool kReset>
inline int launch_bwd(int cell, float *gates, const float *w_hh, const float *ybuf, float *cbuf, const float *dy, const float *dhn,
                      const float *dcn, float *dh0, float *dc0, int B, int S, int H, void *workspace, dc_rnn::Reset rs,
                      cudaStream_t st) {
    const int G = cell == DC_CELL_GRU ? 3 : 4, GH = G * H;
    const Workspace w = carve(workspace, cell, B, H);
    const int blocks = (B * H + 255) / 256;
    const size_t BH = (size_t)B * H;
    int rc = dc_rnn::launch_transpose(w_hh, w.wT, GH, H, st);                  // W_hh^T [H, G*H]: the GEMM's [N, K] operand
    if (rc) return rc;
    for (int it = 0; it < S; ++it) {
        const int t = S - 1 - it;
        float *gt = gates + (size_t)t * B * GH;
        if (G == 3)
            bwd_gate_kernel<3, kReset><<<blocks, 256, 0, st>>>(gt, dy + t * BH, w.part_b, w.ksb, w.dh_carry, w.dc_carry, dhn, nullptr,
                                                               ybuf + t * BH, nullptr, cbuf + (t + 1) * BH, w.dgbuf, it == 0, B, H, rs, t);
        else
            bwd_gate_kernel<4, kReset><<<blocks, 256, 0, st>>>(gt, dy + t * BH, w.part_b, w.ksb, w.dh_carry, w.dc_carry, dhn, dcn, nullptr,
                                                               cbuf + t * BH, cbuf + (t + 1) * BH, w.dgbuf, it == 0, B, H, rs, t);
        rc = dc_gemm_tf32x3_splitk(w.dgbuf, GH, w.wT, GH, w.part_b, B, H, GH, w.ksb, it == 0, st);
        if (rc) return rc;
    }
    bwd_final_kernel<<<blocks, 256, 0, st>>>(w.part_b, w.ksb, w.dh_carry, G == 4 ? w.dc_carry : nullptr, dh0, G == 4 ? dc0 : nullptr, B * H);
    DC_LAUNCH_OK();
    return DC_OK;
}

}  // namespace dc_rnns
