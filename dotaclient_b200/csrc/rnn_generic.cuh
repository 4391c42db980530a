// Shape-generic recurrence kernels (any H that is a multiple of 4, GRU or LSTM).
//
// Fallback for the widths that rnn_resident.cuh, rnn_cluster.cuh and rnn_stepwise.cuh do not cover.
// One CTA owns kBT sequences for all S steps (no inter-CTA communication); h lives in shared
// memory; W_hh is streamed from L2 every step (it is <= 4 MB and stays L2-resident), read with
// fully coalesced loads (forward reads the [H, G*H] transpose held in the workspace, backward
// reads W_hh [G*H, H] as stored).  Correct everywhere, FMA/L2-bound at large H.
#pragma once
#include "rnn_cell.cuh"

namespace dc_rnn {

constexpr int kBT = 4;         // sequences per CTA
constexpr int kThreads = 256;

// The backward's dh mat-vec splits its contraction over kThreads / H slices when H < kThreads (H = 32, 64, 96 here); the
// slices' partial sums go through shared memory and are added in slice order, so that the result is deterministic.
__host__ __device__ constexpr int bwd_slices(int H) { return kThreads >= H ? kThreads / H : 1; }

// Forward.  gates [S,B,G,H] (in: x W_ih^T + b_ih; out: activated gates), wT [H, G*H].  kReset: resets from rs (rnn_cell.cuh).
template <int G, bool kReset = false>
__global__ void __launch_bounds__(kThreads) fwd_generic_kernel(float *__restrict__ gates, const float *__restrict__ wT,
                                                               const float *__restrict__ b_hh, float *__restrict__ ybuf,
                                                               float *__restrict__ cbuf, int B, int S, int H, Reset rs) {
    extern __shared__ __align__(16) float smem[];
    float *h_s = smem;                 // [kBT][H]
    float *pre_s = smem + kBT * H;     // [kBT][G*H]
    const int GH = G * H;
    const int b0 = blockIdx.x * kBT;
    const int nb = min(kBT, B - b0);
    for (int i = threadIdx.x; i < kBT * H; i += kThreads) {
        const int b = i / H, u = i % H;
        h_s[i] = b < nb ? ybuf[(size_t)(b0 + b) * H + u] : 0.f;
    }
    __syncthreads();
    for (int t = 0; t < S; ++t) {
        for (int j = threadIdx.x; j < GH; j += kThreads) {
            float acc[kBT];
            const float bj = b_hh[j];
#pragma unroll
            for (int b = 0; b < kBT; ++b) acc[b] = bj;
            for (int k = 0; k < H; k += 4) {
                float w[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) w[q] = __ldg(wT + (size_t)(k + q) * GH + j);
#pragma unroll
                for (int b = 0; b < kBT; ++b) {
                    const float4 hv = *reinterpret_cast<const float4 *>(h_s + b * H + k);
                    acc[b] = fmaf(hv.x, w[0], acc[b]);
                    acc[b] = fmaf(hv.y, w[1], acc[b]);
                    acc[b] = fmaf(hv.z, w[2], acc[b]);
                    acc[b] = fmaf(hv.w, w[3], acc[b]);
                }
            }
#pragma unroll
            for (int b = 0; b < kBT; ++b) pre_s[b * GH + j] = acc[b];
        }
        __syncthreads();
        for (int i = threadIdx.x; i < nb * H; i += kThreads) {
            const int b = i / H, u = i % H;
            const size_t tok = (size_t)t * B + b0 + b;
            float *g = gates + tok * GH;
            const float *pre = pre_s + b * GH;
            float act[G], aux;
            float prev = G == 3 ? h_s[b * H + u] : cbuf[((size_t)t * B + b0 + b) * H + u];
            if constexpr (kReset) {
                const int k = rs.slot[tok];
                if (k >= 0) {                   // the mat-vec on the stale state is discarded
                    const size_t r = (size_t)k * B + b0 + b;
                    pre = rs.pre + r * GH;
                    prev = rs.prev[r * H + u];
                }
            }
            const float hnew = cell_fwd<G>([&](int q) { return g[q * H + u]; }, [&](int q) { return pre[q * H + u]; }, prev, act, aux);
#pragma unroll
            for (int q = 0; q < G; ++q) g[q * H + u] = act[q];
            cbuf[((size_t)(t + 1) * B + b0 + b) * H + u] = aux;
            ybuf[((size_t)(t + 1) * B + b0 + b) * H + u] = hnew;
            h_s[b * H + u] = hnew;   // each (b,u) is owned by one thread; matvec readers are behind the barrier
        }
        __syncthreads();
    }
}

// Backward.  gates in: activated gates, out: dgi.  w [G*H, H] as stored.  kReset: resets from rs (rnn_cell.cuh).
template <int G, bool kReset = false>
__global__ void __launch_bounds__(kThreads) bwd_generic_kernel(float *__restrict__ gates, const float *__restrict__ w,
                                                               const float *__restrict__ ybuf, float *__restrict__ cbuf,
                                                               const float *__restrict__ dy, const float *__restrict__ dhn,
                                                               const float *__restrict__ dcn, float *__restrict__ dh0,
                                                               float *__restrict__ dc0, int B, int S, int H, Reset rs) {
    extern __shared__ __align__(16) float smem[];
    float *dh_s = smem;                    // [kBT][H] recurrent gradient wrt h
    float *dc_s = smem + kBT * H;          // [kBT][H] (LSTM) recurrent gradient wrt c
    float *dg_s = smem + 2 * kBT * H;      // [kBT][G*H] gradient wrt the hidden-to-hidden pre-activations
    float *part_s = dg_s + kBT * G * H;    // [nslice][kBT][H] partial mat-vec sums (nslice > 1 only)
    const int GH = G * H;
    const int b0 = blockIdx.x * kBT;
    const int nb = min(kBT, B - b0);
    for (int i = threadIdx.x; i < kBT * H; i += kThreads) {
        const int b = i / H, u = i % H;
        dh_s[i] = (b < nb && dhn) ? dhn[(size_t)(b0 + b) * H + u] : 0.f;
        dc_s[i] = (b < nb && dcn) ? dcn[(size_t)(b0 + b) * H + u] : 0.f;
    }
    for (int i = threadIdx.x; i < kBT * GH; i += kThreads) dg_s[i] = 0.f;
    __syncthreads();
    const int nslice = bwd_slices(H);
    for (int t = S - 1; t >= 0; --t) {
        for (int i = threadIdx.x; i < nb * H; i += kThreads) {
            const int b = i / H, u = i % H;
            const size_t tok = (size_t)t * B + b0 + b;
            float *g = gates + tok * GH;
            float *dg = dg_s + b * GH;
            const float dh = dy[tok * H + u] + dh_s[b * H + u];
            const size_t ci = ((size_t)(t + 1) * B + b0 + b) * H + u;
            float dgi[G], dgh[G];
            float prev = G == 3 ? ybuf[tok * H + u] : cbuf[tok * H + u];           // slot t: h_{t-1} | c_{t-1}
            int k = -1;
            if constexpr (kReset) {
                k = rs.slot[tok];
                if (k >= 0) prev = rs.prev[((size_t)k * B + b0 + b) * H + u];
            }
            dh_s[b * H + u] = cell_bwd<G>([&](int q) { return g[q * H + u]; }, cbuf[ci], prev, dh, dc_s[b * H + u], dgi, dgh);   // matvec adds on top
#pragma unroll
            for (int q = 0; q < G; ++q) { g[q * H + u] = dgi[q]; dg[q * H + u] = dgh[q]; }
            if (G == 3) cbuf[ci] = dgh[2];                                            // n-gate part of dgh
            if (kReset && k >= 0) {             // nothing flows into step t-1: zero carries, zero mat-vec operand
                dh_s[b * H + u] = 0.f;
                dc_s[b * H + u] = 0.f;
#pragma unroll
                for (int q = 0; q < G; ++q) dg[q * H + u] = 0.f;
            }
        }
        __syncthreads();
        // dh_{t-1}[b][k] += sum_j dgh[b][j] * W[j][k]
        for (int item = threadIdx.x; item < H * nslice; item += kThreads) {
            const int k = item % H, sl = item / H;
            const int jlo = (int)((long long)GH * sl / nslice), jhi = (int)((long long)GH * (sl + 1) / nslice);
            float acc[kBT];
#pragma unroll
            for (int b = 0; b < kBT; ++b) acc[b] = 0.f;
            for (int j = jlo; j < jhi; ++j) {
                const float wv = __ldg(w + (size_t)j * H + k);
#pragma unroll
                for (int b = 0; b < kBT; ++b) acc[b] = fmaf(dg_s[b * GH + j], wv, acc[b]);
            }
            if (nslice == 1) {                 // the only contribution to dh_s[b][k]
#pragma unroll
                for (int b = 0; b < kBT; ++b) dh_s[b * H + k] += acc[b];
            } else {
#pragma unroll
                for (int b = 0; b < kBT; ++b) part_s[(sl * kBT + b) * H + k] = acc[b];
            }
        }
        __syncthreads();
        if (nslice > 1) {                      // fixed order: cell value, then slice 0, 1, ...
            for (int i = threadIdx.x; i < kBT * H; i += kThreads) {
                float v = dh_s[i];
                for (int sl = 0; sl < nslice; ++sl) v += part_s[sl * kBT * H + i];
                dh_s[i] = v;
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < nb * H; i += kThreads) {
        const int b = i / H, u = i % H;
        if (dh0) dh0[(size_t)(b0 + b) * H + u] = dh_s[b * H + u];
        if (dc0 && G == 4) dc0[(size_t)(b0 + b) * H + u] = dc_s[b * H + u];
    }
}

template <typename K, typename... Args>
inline int launch_generic(K kern, int B, size_t smem, cudaStream_t st, Args... args) {
    DC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(B + kBT - 1) / kBT, kThreads, smem, st>>>(args...);
    DC_LAUNCH_OK();
    return DC_OK;
}

// workspace: W_hh^T [H, G*H] (the forward reads the transpose so that output columns are contiguous)
template <bool kReset>
inline int launch_fwd_generic(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf, float *cbuf, int B, int S,
                              int H, void *workspace, Reset rs, cudaStream_t st) {
    const int G = cell == DC_CELL_GRU ? 3 : 4;
    float *wT = reinterpret_cast<float *>(workspace);
    int rc = launch_transpose(w_hh, wT, G * H, H, st);
    if (rc) return rc;
    const size_t smem = (size_t)kBT * (G + 1) * H * sizeof(float);
    if (G == 3) return launch_generic(fwd_generic_kernel<3, kReset>, B, smem, st, gates, wT, b_hh, ybuf, cbuf, B, S, H, rs);
    return launch_generic(fwd_generic_kernel<4, kReset>, B, smem, st, gates, wT, b_hh, ybuf, cbuf, B, S, H, rs);
}
template <bool kReset>
inline int launch_bwd_generic(int cell, float *gates, const float *w_hh, const float *ybuf, float *cbuf, const float *dy,
                              const float *dhn, const float *dcn, float *dh0, float *dc0, int B, int S, int H, Reset rs,
                              cudaStream_t st) {
    const int G = cell == DC_CELL_GRU ? 3 : 4;
    const int nslice = bwd_slices(H);
    const size_t smem = ((size_t)kBT * (G + 2) * H + (nslice > 1 ? (size_t)nslice * kBT * H : 0)) * sizeof(float);
    if (G == 3) return launch_generic(bwd_generic_kernel<3, kReset>, B, smem, st, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, H, rs);
    return launch_generic(bwd_generic_kernel<4, kReset>, B, smem, st, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, H, rs);
}

}  // namespace dc_rnn
