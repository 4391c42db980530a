// Weight-resident recurrence kernels for H = 128 (GRU and LSTM), forward and backward.
//
// The time loop of nn.GRU / nn.LSTM (policy.py:66,141) is strictly sequential in t, so a launch is
// bound by the latency of ONE step, 2*S times per optimizer step.  Design:
//
//   * one CTA owns kBT sequences for all S steps -- no inter-CTA traffic, no grid sync;
//   * W_hh never leaves the SM: every thread owns a 32 x 4 slab of the [M, Nout] weight matrix,
//     16 rows in REGISTERS (64 regs) and 16 rows in SHARED MEMORY (128 KB LSTM / 96 KB GRU), read
//     as conflict-free 16-byte loads.  (fp32 W_hh is 256 KB for the LSTM: neither the register
//     file nor shared memory alone can hold it, together they can.)
//   * the step's batched mat-vec is FFMA on the fp32 pipe (tensor cores are deliberately not used
//     here: with kBT = 2..4 rows per CTA it is not a dense contraction -- north_star);
//     each warp handles one 32-row slice of the contraction (its input slice is a broadcast
//     shared-memory read) and 128 output columns; the 4 (fwd) / 12-16 (bwd) partial sums per
//     output are combined through shared memory by the gate threads;
//   * the per-step global inputs (i2h pre-activations forward; saved gates, dy, c / hn, h_{t-1}
//     backward) are contiguous [kBT, ...] tiles in the time-major layout and are prefetched
//     kStages steps ahead with 1-D TMA bulk copies (cp.async.bulk + mbarrier complete_tx);
//   * h (fwd) / the gate gradients (bwd) -- the mat-vec input of the next step -- stay in shared
//     memory; c (fwd) and dc (bwd) stay in registers of the thread that owns the (b, unit) pair.
//
// Forward and backward are the same skeleton around one templated mat-vec:
//     fwd: out[b][j] = sum_k h[b][k]   * W_hh^T[k][j]     M = H,   Nout = G*H
//     bwd: out[b][k] = sum_j dg[b][j]  * W_hh[j][k]       M = G*H, Nout = H
//
// Algorithmic HBM bytes per token: fwd reads G*H*4 (gi) and writes (G+2)*H*4 (gates, h, c|hn);
// bwd reads (G+3)*H*4 and writes G*H*4 (+H*4 GRU).
#pragma once
#include "rnn_cell.cuh"

namespace dc_rnn {

constexpr int kH = 128;
constexpr int kStages = 4;

__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(dc_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     dc_smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(dc_smem_u32(bar))
                 : "memory");
}

// Thread layout of the stationary mat-vec: tid = ms * NCG + cg; the thread owns rows [ms*32, ms*32+32) and
// columns [cg*4, cg*4+4) of A [M, NOUT] (row-major in global memory).
template <int NT, int NOUT>
struct Tiling {
    static constexpr int NCG = NOUT / 4;
    static constexpr int NMS = NT / NCG;
    static constexpr int M = NMS * 32;
};

// Weights are held as (row 2j, row 2j+1) PAIRS: the (h[2j], h[2j+1]) operand pairs fall out of the 16-byte
// shared-memory loads for free, and even and odd rows accumulate in two independent FMA chains that are added once
// at the end.
template <int NT, int NOUT>
__device__ __forceinline__ void load_weights(const float *__restrict__ A, float2 (&wr)[8][4], float4 *w_s) {
    using T = Tiling<NT, NOUT>;
    const int cg = threadIdx.x % T::NCG, ms = threadIdx.x / T::NCG;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 r0 = __ldg(reinterpret_cast<const float4 *>(A + (size_t)(ms * 32 + 2 * j) * NOUT) + cg);
        const float4 r1 = __ldg(reinterpret_cast<const float4 *>(A + (size_t)(ms * 32 + 2 * j + 1) * NOUT) + cg);
        wr[j][0] = make_float2(r0.x, r1.x); wr[j][1] = make_float2(r0.y, r1.y);
        wr[j][2] = make_float2(r0.z, r1.z); wr[j][3] = make_float2(r0.w, r1.w);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 r0 = __ldg(reinterpret_cast<const float4 *>(A + (size_t)(ms * 32 + 16 + 2 * j) * NOUT) + cg);
        const float4 r1 = __ldg(reinterpret_cast<const float4 *>(A + (size_t)(ms * 32 + 17 + 2 * j) * NOUT) + cg);
        w_s[((ms * 8 + j) * 2 + 0) * T::NCG + cg] = make_float4(r0.x, r1.x, r0.y, r1.y);
        w_s[((ms * 8 + j) * 2 + 1) * T::NCG + cg] = make_float4(r0.z, r1.z, r0.w, r1.w);
    }
}

// part_s[ms][b][n] = sum over this thread's 32 rows of in_s[b][m] * A[m][n]
template <int NT, int NOUT, int BT>
__device__ __forceinline__ void matvec_partial(const float2 (&wr)[8][4], const float4 *w_s, const float *in_s, float *part_s) {
    using T = Tiling<NT, NOUT>;
    const int cg = threadIdx.x % T::NCG, ms = threadIdx.x / T::NCG;
    float2 acc[BT][4];
#pragma unroll
    for (int b = 0; b < BT; ++b)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[b][c] = make_float2(0.f, 0.f);
    const float *in0 = in_s + ms * 32;
#pragma unroll
    for (int j = 0; j < 8; j += 2) {            // register-resident rows 0..15
        float4 hv[BT];
#pragma unroll
        for (int b = 0; b < BT; ++b) hv[b] = *reinterpret_cast<const float4 *>(in0 + b * T::M + 2 * j);
#pragma unroll
        for (int b = 0; b < BT; ++b) {
            const float2 h0 = make_float2(hv[b].x, hv[b].y), h1 = make_float2(hv[b].z, hv[b].w);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                acc[b][c] = dc_ffma2(h0, wr[j][c], acc[b][c]);
                acc[b][c] = dc_ffma2(h1, wr[j + 1][c], acc[b][c]);
            }
        }
    }
    const float4 *wp = w_s + (ms * 16) * T::NCG + cg;
#pragma unroll
    for (int j = 0; j < 8; j += 2) {            // shared-memory-resident rows 16..31
        float4 hv[BT];
#pragma unroll
        for (int b = 0; b < BT; ++b) hv[b] = *reinterpret_cast<const float4 *>(in0 + b * T::M + 16 + 2 * j);
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const float4 wa = wp[((j + p) * 2 + 0) * T::NCG];
            const float4 wb = wp[((j + p) * 2 + 1) * T::NCG];
            const float2 w0 = make_float2(wa.x, wa.y), w1 = make_float2(wa.z, wa.w);
            const float2 w2 = make_float2(wb.x, wb.y), w3 = make_float2(wb.z, wb.w);
#pragma unroll
            for (int b = 0; b < BT; ++b) {
                const float2 h = p == 0 ? make_float2(hv[b].x, hv[b].y) : make_float2(hv[b].z, hv[b].w);
                acc[b][0] = dc_ffma2(h, w0, acc[b][0]);
                acc[b][1] = dc_ffma2(h, w1, acc[b][1]);
                acc[b][2] = dc_ffma2(h, w2, acc[b][2]);
                acc[b][3] = dc_ffma2(h, w3, acc[b][3]);
            }
        }
    }
#pragma unroll
    for (int b = 0; b < BT; ++b)
        *reinterpret_cast<float4 *>(part_s + ((ms * BT + b) * NOUT) + cg * 4) =
            make_float4(acc[b][0].x + acc[b][0].y, acc[b][1].x + acc[b][1].y, acc[b][2].x + acc[b][2].y, acc[b][3].x + acc[b][3].y);
}

template <int G, int BT>
struct FwdSmem {
    static constexpr int NT = G * kH;
    static constexpr int GH = G * kH;
    static constexpr size_t w_bytes = (size_t)NT * 16 * sizeof(float4);          // smem half of W_hh^T
    static constexpr size_t in_bytes = (size_t)BT * kH * 4;                       // h
    static constexpr size_t part_bytes = (size_t)4 * BT * GH * 4;                 // NMS = 4 partials
    static constexpr size_t stage_bytes = (size_t)BT * GH * 4;                    // gi tile
    static constexpr size_t total = w_bytes + in_bytes + part_bytes + kStages * stage_bytes + kStages * 8 + 16;
};

// ---- forward --------------------------------------------------------------------------------
// kReset: resets from rs (rnn_cell.cuh): the gate thread of a reset token takes pre and prev from the tables instead of the
// mat-vec partials and its own h / c.
template <int G, int BT, bool kReset = false>
__global__ void __launch_bounds__(G *kH, 1) fwd_resident_kernel(float *__restrict__ gates, const float *__restrict__ wT,
                                                                 const float *__restrict__ b_hh, float *__restrict__ ybuf,
                                                                 float *__restrict__ cbuf, int B, int S, Reset rs) {
    using SM = FwdSmem<G, BT>;
    constexpr int NT = SM::NT, GH = SM::GH, H = kH;
    static_assert(BT * kH <= G * kH, "one gate thread per (sequence, unit) pair");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float4 *w_s = reinterpret_cast<float4 *>(smem_raw);
    float *in_s = reinterpret_cast<float *>(smem_raw + SM::w_bytes);
    float *part_s = reinterpret_cast<float *>(smem_raw + SM::w_bytes + SM::in_bytes);
    float *stage_s = reinterpret_cast<float *>(smem_raw + SM::w_bytes + SM::in_bytes + SM::part_bytes);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + SM::w_bytes + SM::in_bytes + SM::part_bytes + kStages * SM::stage_bytes);

    const int tid = threadIdx.x;
    const int b0 = blockIdx.x * BT;
    const int nb = min(BT, B - b0);
    const uint32_t tile_bytes = (uint32_t)nb * GH * 4;

    float2 wr[8][4];
    load_weights<NT, GH>(wT, wr, w_s);
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) dc_mbar_init(&bars[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // unit threads: (b, u) pairs
    const bool unit = tid < BT * H;
    const int ub = tid / H, uu = tid % H;
    const bool live = unit && ub < nb;
    float c_reg = 0.f, bias[G];
    if (unit) {
        in_s[ub * H + uu] = live ? ybuf[(size_t)(b0 + ub) * H + uu] : 0.f;      // h_0
        if (G == 4 && live) c_reg = cbuf[(size_t)(b0 + ub) * H + uu];           // c_0
#pragma unroll
        for (int g = 0; g < G; ++g) bias[g] = b_hh[g * H + uu];
    }
    __syncthreads();
    if (tid == 0) {
        for (int s = 0; s < kStages && s < S; ++s) {
            mbar_expect_tx(&bars[s], tile_bytes);
            bulk_g2s(stage_s + (size_t)s * BT * GH, gates + ((size_t)s * B + b0) * GH, tile_bytes, &bars[s]);
        }
    }
    for (int t = 0; t < S; ++t) {
        int k = -1;                             // loaded ahead of the mat-vec, read after it
        if constexpr (kReset) k = live ? __ldg(rs.slot + (size_t)t * B + b0 + ub) : -1;
        matvec_partial<NT, GH, BT>(wr, w_s, in_s, part_s);
        __syncthreads();
        const int st = t % kStages;
        if (unit) {
            dc_mbar_wait(&bars[st], (t / kStages) & 1);
            if (live) {
                const float *gi = stage_s + (size_t)st * BT * GH + ub * GH;
                float pre[G];
#pragma unroll
                for (int g = 0; g < G; ++g) {
                    float a = bias[g];
#pragma unroll
                    for (int ms = 0; ms < 4; ++ms) a += part_s[(ms * BT + ub) * GH + g * H + uu];
                    pre[g] = a;
                }
                float prev = G == 3 ? in_s[ub * H + uu] : c_reg;
                if (kReset && k >= 0) {
                    const size_t r = (size_t)k * B + b0 + ub;
#pragma unroll
                    for (int g = 0; g < G; ++g) pre[g] = rs.pre[r * GH + g * H + uu];
                    prev = rs.prev[r * H + uu];
                }
                const size_t tok = (size_t)t * B + b0 + ub;
                float *gout = gates + tok * GH;
                float act[G], aux;
                const float hnew = cell_fwd<G, false>([&](int g) { return gi[g * H + uu]; }, [&](int g) { return pre[g]; },
                                               prev, act, aux);
                if (G == 4) c_reg = aux;
#pragma unroll
                for (int g = 0; g < G; ++g) gout[g * H + uu] = act[g];
                cbuf[(tok + B) * H + uu] = aux;                                    // c_t | W_hn h + b_hn, slot t+1
                ybuf[(tok + B) * H + uu] = hnew;
                in_s[ub * H + uu] = hnew;
            }
        }
        __syncthreads();
        if (tid == 0 && t + kStages < S) {      // every reader of this stage is behind the barrier: refill it
            mbar_expect_tx(&bars[st], tile_bytes);
            bulk_g2s(stage_s + (size_t)st * BT * GH, gates + ((size_t)(t + kStages) * B + b0) * GH, tile_bytes, &bars[st]);
        }
    }
}

// ---- backward -------------------------------------------------------------------------------
template <int G, int BT>
struct BwdSmem {
    static constexpr int NT = G * kH;
    static constexpr int GH = G * kH;
    static constexpr int NMS = NT / (kH / 4);                                     // 16 (LSTM) / 12 (GRU)
    static constexpr size_t w_bytes = (size_t)NT * 16 * sizeof(float4);
    static constexpr size_t in_bytes = (size_t)BT * GH * 4;                       // gate gradients (mat-vec input)
    static constexpr size_t part_bytes = (size_t)NMS * BT * kH * 4;
    // stage: gates tile [BT, GH] + dy [BT, H] + aux1 [BT, H] (LSTM c_{t-1} | GRU hn) + aux2 [BT, H] (GRU h_{t-1})
    static constexpr size_t stage_floats = (size_t)BT * (GH + 3 * kH);
    static constexpr size_t total = w_bytes + in_bytes + part_bytes + kStages * stage_floats * 4 + kStages * 8 + 16;
};

// kReset: resets from rs (rnn_cell.cuh): a reset token reads prev from the table and leaves zero carries and a zero mat-vec
// operand, so step t-1 (or dh0 / dc0) receives exactly nothing from it.
template <int G, int BT, bool kReset = false>
__global__ void __launch_bounds__(G *kH, 1) bwd_resident_kernel(float *__restrict__ gates, const float *__restrict__ w,
                                                                 const float *__restrict__ ybuf, float *__restrict__ cbuf,
                                                                 const float *__restrict__ dy, const float *__restrict__ dhn,
                                                                 const float *__restrict__ dcn, float *__restrict__ dh0,
                                                                 float *__restrict__ dc0, int B, int S, Reset rs) {
    using SM = BwdSmem<G, BT>;
    constexpr int NT = SM::NT, GH = SM::GH, H = kH, NMS = SM::NMS;
    static_assert(BT * kH <= G * kH, "one gate thread per (sequence, unit) pair");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float4 *w_s = reinterpret_cast<float4 *>(smem_raw);
    float *in_s = reinterpret_cast<float *>(smem_raw + SM::w_bytes);
    float *part_s = reinterpret_cast<float *>(smem_raw + SM::w_bytes + SM::in_bytes);
    float *stage_s = reinterpret_cast<float *>(smem_raw + SM::w_bytes + SM::in_bytes + SM::part_bytes);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + SM::w_bytes + SM::in_bytes + SM::part_bytes + kStages * SM::stage_floats * 4);

    const int tid = threadIdx.x;
    const int b0 = blockIdx.x * BT;
    const int nb = min(BT, B - b0);
    const uint32_t gate_bytes = (uint32_t)nb * GH * 4, row_bytes = (uint32_t)nb * H * 4;

    float2 wr[8][4];
    load_weights<NT, H>(w, wr, w_s);
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) dc_mbar_init(&bars[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const bool unit = tid < BT * H;
    const int ub = tid / H, uu = tid % H;
    const bool live = unit && ub < nb;
    // recurrent gradients owned by the (b, u) thread
    float dh_carry = 0.f;      // GRU: direct path dh * z;  both: initial dh_n
    float dc_carry = 0.f;      // LSTM: dL/dc flowing to step t-1
    float c_cur = 0.f;         // LSTM: c_t of the step being processed (slot t+1)
    if (live) {
        if (dhn) dh_carry = dhn[(size_t)(b0 + ub) * H + uu];
        if (G == 4) {
            if (dcn) dc_carry = dcn[(size_t)(b0 + ub) * H + uu];
            c_cur = cbuf[((size_t)S * B + b0 + ub) * H + uu];
        }
    }
    for (int i = tid; i < NMS * BT * H; i += NT) part_s[i] = 0.f;
    for (int i = tid; i < BT * GH; i += NT) in_s[i] = 0.f;
    __syncthreads();

    auto issue = [&](int t, int st) {
        float *dst = stage_s + (size_t)st * SM::stage_floats;
        const size_t tok = (size_t)t * B + b0;
        const uint32_t total = gate_bytes + row_bytes * (G == 3 ? 3u : 2u);
        mbar_expect_tx(&bars[st], total);
        bulk_g2s(dst, gates + tok * GH, gate_bytes, &bars[st]);
        bulk_g2s(dst + BT * GH, dy + tok * H, row_bytes, &bars[st]);
        if (G == 4) {
            bulk_g2s(dst + BT * (GH + H), cbuf + tok * H, row_bytes, &bars[st]);            // c_{t-1} (slot t)
        } else {
            bulk_g2s(dst + BT * (GH + H), cbuf + (tok + B) * H, row_bytes, &bars[st]);      // hn (slot t+1)
            bulk_g2s(dst + BT * (GH + 2 * H), ybuf + tok * H, row_bytes, &bars[st]);        // h_{t-1} (slot t)
        }
    };
    if (tid == 0)
        for (int s = 0; s < kStages && s < S; ++s) issue(S - 1 - s, s);

    for (int it = 0; it < S; ++it) {
        const int t = S - 1 - it;
        const int st = it % kStages;
        if (unit) {
            int k = -1;
            if constexpr (kReset) k = live ? __ldg(rs.slot + (size_t)t * B + b0 + ub) : -1;
            dc_mbar_wait(&bars[st], (it / kStages) & 1);
            if (live) {
                const float *sg = stage_s + (size_t)st * SM::stage_floats;
                const float *g = sg + ub * GH;
                float dh = sg[BT * GH + ub * H + uu] + dh_carry;
#pragma unroll
                for (int ms = 0; ms < NMS; ++ms) dh += part_s[(ms * BT + ub) * H + uu];
                const size_t tok = (size_t)t * B + b0 + ub;
                float *gout = gates + tok * GH;
                float *dg = in_s + ub * GH;
                auto act = [&](int q) { return g[q * H + uu]; };
                const float aux1 = sg[BT * (GH + H) + ub * H + uu];                  // LSTM c_{t-1} | GRU hn
                float dgi[G], dgh[G];
                if constexpr (kReset) {
                    float prev = G == 3 ? sg[BT * (GH + 2 * H) + ub * H + uu] : aux1;
                    if (k >= 0) prev = rs.prev[((size_t)k * B + b0 + ub) * H + uu];
                    dh_carry = cell_bwd<G>(act, G == 3 ? aux1 : c_cur, prev, dh, dc_carry, dgi, dgh);
                } else {
                    if (G == 3) dh_carry = cell_bwd<G>(act, aux1, sg[BT * (GH + 2 * H) + ub * H + uu], dh, dc_carry, dgi, dgh);
                    else dh_carry = cell_bwd<G>(act, c_cur, aux1, dh, dc_carry, dgi, dgh);
                }
#pragma unroll
                for (int q = 0; q < G; ++q) gout[q * H + uu] = dgi[q];
                if (G == 3) cbuf[(tok + B) * H + uu] = dgh[2];
                if (kReset && k >= 0) {
                    dh_carry = 0.f;
                    dc_carry = 0.f;
#pragma unroll
                    for (int q = 0; q < G; ++q) dgh[q] = 0.f;
                }
#pragma unroll
                for (int q = 0; q < G; ++q) dg[q * H + uu] = dgh[q];
                if (G == 4) c_cur = aux1;
            }
        }
        __syncthreads();
        if (tid == 0 && it + kStages < S) issue(S - 1 - (it + kStages), st);
        matvec_partial<NT, H, BT>(wr, w_s, in_s, part_s);
        __syncthreads();
    }
    if (live) {
        float dh = dh_carry;
#pragma unroll
        for (int ms = 0; ms < NMS; ++ms) dh += part_s[(ms * BT + ub) * H + uu];
        if (dh0) dh0[(size_t)(b0 + ub) * H + uu] = dh;
        if (G == 4 && dc0) dc0[(size_t)(b0 + ub) * H + uu] = dc_carry;
    }
}

inline bool resident_supported(int H) { return H == kH; }

template <int G, int BT, bool kReset>
int launch_fwd_t(float *gates, const float *wT, const float *b_hh, float *ybuf, float *cbuf, int B, int S, Reset rs, cudaStream_t st) {
    const size_t smem = FwdSmem<G, BT>::total;
    DC_CUDA(cudaFuncSetAttribute(fwd_resident_kernel<G, BT, kReset>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fwd_resident_kernel<G, BT, kReset><<<(B + BT - 1) / BT, G * kH, smem, st>>>(gates, wT, b_hh, ybuf, cbuf, B, S, rs);
    DC_LAUNCH_OK();
    return DC_OK;
}
template <int G, int BT, bool kReset>
int launch_bwd_t(float *gates, const float *w, const float *ybuf, float *cbuf, const float *dy, const float *dhn,
                 const float *dcn, float *dh0, float *dc0, int B, int S, Reset rs, cudaStream_t st) {
    const size_t smem = BwdSmem<G, BT>::total;
    DC_CUDA(cudaFuncSetAttribute(bwd_resident_kernel<G, BT, kReset>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    bwd_resident_kernel<G, BT, kReset><<<(B + BT - 1) / BT, G * kH, smem, st>>>(gates, w, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, rs);
    DC_LAUNCH_OK();
    return DC_OK;
}

// kBT: the smallest batch tile that still fits the batch in one wave of CTAs (1 CTA / SM).  The gate phase maps one
// thread to one (sequence, unit) pair, so kBT * H must not exceed the CTA size G * H: kBT <= 3 (GRU) / 4 (LSTM).
inline bool small_tile(int B) { return (B + 1) / 2 <= dc_sm_count(); }

// workspace: W_hh^T [H, G*H], the [M, NOUT] operand of the forward mat-vec
template <bool kReset>
inline int launch_fwd_resident(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf, float *cbuf, int B,
                               int S, void *workspace, Reset rs, cudaStream_t st) {
    float *wT = reinterpret_cast<float *>(workspace);
    int rc = launch_transpose(w_hh, wT, (cell == DC_CELL_GRU ? 3 : 4) * kH, kH, st);
    if (rc) return rc;
    if (cell == DC_CELL_GRU)
        return small_tile(B) ? launch_fwd_t<3, 2, kReset>(gates, wT, b_hh, ybuf, cbuf, B, S, rs, st)
                             : launch_fwd_t<3, 3, kReset>(gates, wT, b_hh, ybuf, cbuf, B, S, rs, st);
    return small_tile(B) ? launch_fwd_t<4, 2, kReset>(gates, wT, b_hh, ybuf, cbuf, B, S, rs, st)
                         : launch_fwd_t<4, 4, kReset>(gates, wT, b_hh, ybuf, cbuf, B, S, rs, st);
}
template <bool kReset>
inline int launch_bwd_resident(int cell, float *gates, const float *w, const float *ybuf, float *cbuf, const float *dy,
                               const float *dhn, const float *dcn, float *dh0, float *dc0, int B, int S, Reset rs, cudaStream_t st) {
    if (cell == DC_CELL_GRU)
        return small_tile(B) ? launch_bwd_t<3, 2, kReset>(gates, w, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, rs, st)
                             : launch_bwd_t<3, 3, kReset>(gates, w, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, rs, st);
    return small_tile(B) ? launch_bwd_t<4, 2, kReset>(gates, w, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, rs, st)
                         : launch_bwd_t<4, 4, kReset>(gates, w, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, rs, st);
}

}  // namespace dc_rnn
