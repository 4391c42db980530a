// Cluster-resident tensor-core recurrence for H = 256 (GRU and LSTM), forward and backward.
//
// H = 256 is the reference's own width (policy.py:66 nn.GRU(256, 256)); W_hh is 768 KB (GRU) / 1 MB (LSTM) in fp32 and
// cannot live in one SM.  At this width the step IS a dense contraction -- [sequences, 256] x [256, G*256] per step --
// so the mat-vec runs on the tensor cores (wgmma) with the same 3xTF32 split as the other dense layers (fp32-level
// accuracy, ~1e-6).
//
//   * a CLUSTER of 8 CTAs owns kNB = 32 sequences for all S steps; CTA r owns hidden units [32r, 32r+32): its 4 x 32
//     rows of W_hh (forward) / 4 x 32 columns (backward) stay on chip for the whole launch -- the tf32 hi half in
//     REGISTERS as the A fragments of wgmma (64 registers per thread), the lo half in shared memory (128 KB of K-major
//     SWIZZLE_128B tiles).  Both halves in shared memory would need 256 KB, more than an SM has;
//   * forward  D[(g,u)][b] = W_hh[(g,u)][:] . h[b][:]      M = 128 rows, N = 32 sequences, K = 256: every CTA needs the
//     whole h of its 32 sequences -- an all-gather.  h_t is an OUTPUT of the layer anyway (ybuf), so each CTA writes its
//     32-unit slice to ybuf, the cluster barrier (release/acquire) publishes it, and every CTA reads the [32 x 256] tile
//     back from L2, splits it hi/lo and stores the B-operand tiles.  Warpgroup w takes rows [64 (w%2), +64) and K half
//     w/2; the two K halves meet in shared memory;
//   * backward D[k][b] = sum_{j in own 128 gate columns} W_hh[j][k] dg[b][j]   M = 256 (64 rows per warpgroup), N = 32,
//     K = 128: the B operand (this CTA's own gate gradients) is local; the partial sums over the 8 CTAs are exchanged
//     through a small L2-resident scratch (reduce-scatter, fixed summation order => deterministic);
//   * gate math: thread = (unit, 2 sequences), 128-byte coalesced global accesses; the per-step global inputs are
//     loaded while the wgmma run asynchronously.
// Per step and CTA: 48 wgmma m64n32k8 per warpgroup, one cluster barrier, one L2 round trip; the cluster barrier is split
// (arrive.release right after the exchanged slice is stored, wait.acquire after the remaining stores).
// Algorithmic HBM bytes per token: forward 4*(G+1)*H, backward 8*(G+1)*H (SURVEY.md 8d).
#pragma once
#include "rnn_cell.cuh"

namespace dc_rnnc {

constexpr int kH = 256;
constexpr int kCL = 8;                  // CTAs per cluster
constexpr int kNB = 32;                 // sequences per cluster = MMA N
constexpr int kThreads = 512;           // 4 warpgroups
constexpr int kPanelA = 128 * 128;      // bytes of one A tile: 128 rows x 32 tf32 (one SWIZZLE_128B row each)
constexpr int kPanelB = kNB * 128;      // bytes of one B tile:  32 rows x 32 tf32

#define DC_ACC16 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
// d (+)= A[smem desc, 64 x 8] B[smem desc, 32 x 8]^T
__device__ __forceinline__ void wgmma_ss(float (&d)[16], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
        : DC_ACC16
        : "l"(desc_a), "l"(desc_b), "r"(1));
}
// d (+)= A[registers, 64 x 8] B[smem desc, 32 x 8]^T.  Fragment of thread (warp w of the warpgroup, lane l): a[0] = A[16w + l/4][l%4],
// a[1] = A[16w + l/4 + 8][l%4], a[2] = A[16w + l/4][l%4 + 4], a[3] = A[16w + l/4 + 8][l%4 + 4].
__device__ __forceinline__ void wgmma_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}\n"
        : DC_ACC16
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}
#undef DC_ACC16
// accumulator fragment of m64n32: d[i] at row 16*warp + lane/4 + 8*((i/2)%2), column 8*(i/4) + 2*(lane%4) + i%2
__device__ __forceinline__ int acc_row(int i, int wi, int lane) { return 16 * wi + (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int acc_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }
__device__ __forceinline__ void acc_fence(float (&d)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) dc_reg_fence(d[i]);
}
// All threads of all CTAs of the cluster.  release/acquire at cluster scope: global writes made before the barrier by any
// thread of the cluster are visible to every thread of the cluster after it.
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_barrier() { cluster_arrive(); cluster_wait(); }
__device__ __forceinline__ unsigned char *align1024(unsigned char *p) {
    return reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}
// one 16-byte chunk (4 tf32) of row `row`, 16-byte chunk index `c` (0..7) of a K-major SWIZZLE_128B tile
__device__ __forceinline__ int swz(int row, int c) { return row * 128 + ((c ^ (row & 7)) << 4); }

// ---- forward ------------------------------------------------------------------------------------------------------------
// W_hh slice row rho = g*32 + u  <->  row g*H + 32*rank + u of W_hh, column = k.  Registers: the hi half of warpgroup w's
// rows [64 (w%2), +64) and K half w/2.  Shared: W lo half (8 K-panels of [128 rows x 32]), h hi / lo (8 K-panels of
// [32 sequences x 32]), the two K halves' products [2][4 gates][32 sequences][32 units].
struct FwdSmem {
    static constexpr size_t wlo = 0;
    static constexpr size_t hhi = wlo + 8 * kPanelA;
    static constexpr size_t hlo = hhi + 8 * kPanelB;
    static constexpr size_t scratch = hlo + 8 * kPanelB;          // [2 K halves][4 gates][32 sequences][32 units] fp32
    static constexpr size_t total = scratch + 2 * 4 * kNB * 32 * 4 + 1024;   // + alignment slack
};
constexpr int kNP = 2;                                            // (sequence, unit) pairs per thread in the gate phase

// kReset: resets from rs (rnn_cell.cuh).  The all-gather and the MMAs run unchanged on the stale state; the gate math of a
// reset token takes pre and prev from the tables.  Each step's reset slots are prefetched with its i2h inputs.
template <int G, bool kReset = false>
__global__ void __launch_bounds__(kThreads, 1) fwd_cluster_kernel(float *gates, const float *__restrict__ w_hh,
                                                                   const float *__restrict__ b_hh, float *ybuf, float *cbuf,
                                                                   int B, int S, dc_rnn::Reset rs) {
    constexpr int H = kH, GH = G * kH, NP = kNP;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *base = align1024(smem_raw);
    unsigned char *wlo = base + FwdSmem::wlo, *hhi = base + FwdSmem::hhi, *hlo = base + FwdSmem::hlo;
    float *scratch = reinterpret_cast<float *>(base + FwdSmem::scratch);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rank = blockIdx.x % kCL, b0 = (blockIdx.x / kCL) * kNB;

    // MMA roles: warpgroup wg takes rows [64 mh, 64 mh + 64) of the slice and K-panels [4 kh, 4 kh + 4)
    const int wg = warp >> 2, wi = warp & 3, mh = wg & 1, kh = wg >> 1;
    uint32_t ahi[16][4];                                                   // A fragments of the hi half, one per k-step of 8
    {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int rho = 64 * mh + 16 * wi + (lane >> 2) + 8 * h, g = rho >> 5;
            const float *wrow = w_hh + (size_t)(g * H + rank * 32 + (rho & 31)) * H + 128 * kh + (lane & 3);
#pragma unroll
            for (int s = 0; s < 16; ++s) {
                ahi[s][h] = __float_as_uint(g < G ? dc_tf32_rna(__ldg(wrow + 8 * s)) : 0.f);          // GRU has no 4th gate: zero rows
                ahi[s][h + 2] = __float_as_uint(g < G ? dc_tf32_rna(__ldg(wrow + 8 * s + 4)) : 0.f);
            }
        }
    }
    const uint64_t d_alo = dc_wgmma_desc(dc_smem_u32(wlo) + 4 * kh * kPanelA + mh * 64 * 128), d_bhi = dc_wgmma_desc(dc_smem_u32(hhi) + 4 * kh * kPanelB),
                   d_blo = dc_wgmma_desc(dc_smem_u32(hlo) + 4 * kh * kPanelB);
    float *my_scratch = scratch + kh * (4 * kNB * 32);

    {   // resident lo half, once: warp (q, kq) fills rows [32q, 32q+32), columns [64*kq, 64*kq+64)
        const int q = warp & 3, kq = warp >> 2, rho = q * 32 + lane;
        const bool valid = q < G;                                          // q == gate index; GRU has no 4th gate: zero rows
        const float *wrow = w_hh + (size_t)(q * H + rank * 32 + lane) * H;
#pragma unroll 2
        for (int k0 = kq * 64; k0 < kq * 64 + 64; k0 += 8) {
            float w[8], hi[8], lo[8];
            if (valid) {
                const float4 w0 = __ldg(reinterpret_cast<const float4 *>(wrow + k0)), w1 = __ldg(reinterpret_cast<const float4 *>(wrow + k0 + 4));
                w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
            } else {
#pragma unroll
                for (int e = 0; e < 8; ++e) w[e] = 0.f;
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) { hi[e] = dc_tf32_rna(w[e]); lo[e] = w[e] - hi[e]; }
            unsigned char *panel = wlo + (size_t)(k0 >> 5) * kPanelA;
            const int c0 = (k0 & 31) >> 2;
            *reinterpret_cast<float4 *>(panel + swz(rho, c0)) = make_float4(lo[0], lo[1], lo[2], lo[3]);
            *reinterpret_cast<float4 *>(panel + swz(rho, c0 + 1)) = make_float4(lo[4], lo[5], lo[6], lo[7]);
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    // gate phase: thread = (unit ul, sequences sb + 16 i)
    const int ul = lane, unit = rank * 32 + ul, sb = warp;
    float bias[G], c_reg[NP], h_reg[NP], cur[NP][G], nxt[NP][G];
    int cslot[NP], nslot[NP];                                              // reset slots of this step and the next (kReset)
    bool live[NP];
#pragma unroll
    for (int g = 0; g < G; ++g) bias[g] = __ldg(b_hh + g * H + unit);
#pragma unroll
    for (int i = 0; i < NP; ++i) {
        const int b = b0 + sb + 16 * i;
        live[i] = b < B;
        if constexpr (kReset) cslot[i] = nslot[i] = live[i] ? __ldg(rs.slot + b) : -1;
        c_reg[i] = (G == 4 && live[i]) ? cbuf[(size_t)b * H + unit] : 0.f;
        h_reg[i] = (G == 3 && live[i]) ? ybuf[(size_t)b * H + unit] : 0.f;
#pragma unroll
        for (int g = 0; g < G; ++g) {
            cur[i][g] = live[i] ? gates[(size_t)b * GH + g * H + unit] : 0.f;
            nxt[i][g] = 0.f;
        }
    }
    // h-tile loader: thread = (sequence hb, 16-byte chunk hc) of K-panels hp0, hp0+2, hp0+4, hp0+6
    const int hc = tid & 7, hb = (tid >> 3) & 31, hp0 = tid >> 8;
    const bool hlive = b0 + hb < B;
    cluster_barrier();

    for (int t = 0; t < S; ++t) {
        // ---- A: gather h_{t-1} [32 x 256] (ybuf slot t) from L2, split, store the B-operand tiles
        {
            const float *src = ybuf + ((size_t)t * B + b0 + hb) * H + 4 * hc;
            float4 v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                v[j] = hlive ? __ldcg(reinterpret_cast<const float4 *>(src + 32 * (hp0 + 2 * j))) : make_float4(0.f, 0.f, 0.f, 0.f);
            const int off = swz(hb, hc);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int p = hp0 + 2 * j;
                float4 hi, lo;
                hi.x = dc_tf32_rna(v[j].x); hi.y = dc_tf32_rna(v[j].y); hi.z = dc_tf32_rna(v[j].z); hi.w = dc_tf32_rna(v[j].w);
                lo.x = v[j].x - hi.x; lo.y = v[j].y - hi.y; lo.z = v[j].z - hi.z; lo.w = v[j].w - hi.w;
                *reinterpret_cast<float4 *>(hhi + p * kPanelB + off) = hi;
                *reinterpret_cast<float4 *>(hlo + p * kPanelB + off) = lo;
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        // ---- B: 48 wgmma per warpgroup (4 K-panels x 4 k-steps x 3 products), asynchronous until the wait below
        float d[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) d[i] = 0.f;
        acc_fence(d);
        dc_wgmma_fence();
#pragma unroll
        for (int s = 0; s < 16; ++s) {
            const uint64_t adv = (uint64_t)((s & 3) * 2), pa = (uint64_t)(s >> 2) * (kPanelA >> 4), pb = (uint64_t)(s >> 2) * (kPanelB >> 4);
            wgmma_ss(d, d_alo + pa + adv, d_bhi + pb + adv);                                     // small terms first
            wgmma_rs(d, ahi[s], d_blo + pb + adv);
            wgmma_rs(d, ahi[s], d_bhi + pb + adv);
        }
        dc_wgmma_commit();
        // prefetch the next step's i2h pre-activations while the tensor core works
        if (t + 1 < S) {
#pragma unroll
            for (int i = 0; i < NP; ++i) {
#pragma unroll
                for (int g = 0; g < G; ++g)
                    nxt[i][g] = live[i] ? gates[((size_t)(t + 1) * B + b0 + sb + 16 * i) * GH + g * H + unit] : 0.f;
                if constexpr (kReset) nslot[i] = live[i] ? __ldg(rs.slot + (size_t)(t + 1) * B + b0 + sb + 16 * i) : -1;
            }
        }
        dc_wgmma_wait0();
        acc_fence(d);
        // ---- C: this K half's product -> scratch [half][gate][sequence][unit]; the gate math adds the halves in a fixed order
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int rho = 64 * mh + acc_row(i, wi, lane);
            my_scratch[((rho >> 5) * kNB + acc_col(i, lane)) * 32 + (rho & 31)] = d[i];
        }
        __syncthreads();
        float act[NP][G], aux[NP];                                                 // activated gates, c | hn -> cbuf slot t+1
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            const int bb = sb + 16 * i;
            float pre[G];
#pragma unroll
            for (int g = 0; g < G; ++g) pre[g] = bias[g] + (scratch[(g * kNB + bb) * 32 + ul] + scratch[((4 + g) * kNB + bb) * 32 + ul]);
            float prev = G == 3 ? h_reg[i] : c_reg[i];
            if (kReset && cslot[i] >= 0) {
                const size_t r = (size_t)cslot[i] * B + b0 + bb;
#pragma unroll
                for (int g = 0; g < G; ++g) pre[g] = rs.pre[r * GH + g * H + unit];
                prev = rs.prev[r * H + unit];
            }
            const float hnew = dc_rnn::cell_fwd<G>([&](int g) { return cur[i][g]; }, [&](int g) { return pre[g]; },
                                                   prev, act[i], aux[i]);
            if (G == 3) h_reg[i] = hnew;
            else c_reg[i] = aux[i];
            if (live[i]) ybuf[((size_t)(t + 1) * B + b0 + bb) * H + unit] = hnew;  // the slice the other CTAs wait for
        }
        // ---- D: publish this CTA's slice of h_t (release), then write the rest of the step's outputs behind the barrier
        cluster_arrive();
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            if (live[i]) {
                const size_t tok = (size_t)t * B + b0 + sb + 16 * i;
                float *gout = gates + tok * GH + unit;
#pragma unroll
                for (int g = 0; g < G; ++g) gout[g * H] = act[i][g];
                cbuf[(tok + B) * H + unit] = aux[i];
            }
#pragma unroll
            for (int g = 0; g < G; ++g) cur[i][g] = nxt[i][g];
            if constexpr (kReset) cslot[i] = nslot[i];
        }
        cluster_wait();
    }
}

// ---- backward -----------------------------------------------------------------------------------------------------------
// W_hh^T slice: row k (two M tiles of 128), column kappa = g*32 + u <-> j = g*H + 32*rank + u.  Registers: the hi half of
// warpgroup w's rows [64 w, 64 w + 64), all G K-panels.  Shared: lo half (2 x 4 K-panels), gate-gradient tile hi / lo.
struct BwdSmem {
    static constexpr size_t wlo = 0;
    static constexpr size_t ghi = wlo + 8 * kPanelA;
    static constexpr size_t glo = ghi + 4 * kPanelB;
    static constexpr size_t total = glo + 4 * kPanelB + 1024;
};

inline size_t bwd_workspace_bytes(int B) { return (size_t)2 * ((B + kNB - 1) / kNB) * kCL * kNB * kH * sizeof(float); }

// kReset: resets from rs (rnn_cell.cuh).  A reset token reads prev from the table and puts zero carries and a zero column into
// the B operand, so every CTA's partial for that sequence -- and so the reduce-scatter into step t-1 -- is exactly zero.
template <int G, bool kReset = false>
__global__ void __launch_bounds__(kThreads, 1) bwd_cluster_kernel(float *gates, const float *__restrict__ w_hh, const float *ybuf,
                                                                   float *cbuf, const float *__restrict__ dy,
                                                                   const float *__restrict__ dhn, const float *__restrict__ dcn,
                                                                   float *__restrict__ dh0, float *__restrict__ dc0, float *part,
                                                                   int B, int S, dc_rnn::Reset rs) {
    constexpr int H = kH, GH = G * kH, NP = kNP;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *base = align1024(smem_raw);
    unsigned char *wlo = base + BwdSmem::wlo, *ghi = base + BwdSmem::ghi, *glo = base + BwdSmem::glo;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rank = blockIdx.x % kCL, cl = blockIdx.x / kCL, ncl = gridDim.x / kCL, b0 = cl * kNB;

    // MMA roles: warpgroup wg takes rows k in [64 wg, 64 wg + 64) (M tile wg / 2), all of this CTA's G K-panels
    const int wg = warp >> 2, wi = warp & 3;
    uint32_t ahi[4 * G][4];                                                // A fragments of the hi half, one per k-step of 8
#pragma unroll
    for (int s = 0; s < 4 * G; ++s) {
        const int g = s >> 2, u = 8 * (s & 3) + (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int k = 64 * wg + 16 * wi + (lane >> 2) + 8 * h;
            ahi[s][h] = __float_as_uint(dc_tf32_rna(__ldg(w_hh + (size_t)(g * H + rank * 32 + u) * H + k)));
            ahi[s][h + 2] = __float_as_uint(dc_tf32_rna(__ldg(w_hh + (size_t)(g * H + rank * 32 + u + 4) * H + k)));
        }
    }
    const uint64_t d_alo = dc_wgmma_desc(dc_smem_u32(wlo) + (wg >> 1) * 4 * kPanelA + (wg & 1) * 64 * 128), d_bhi = dc_wgmma_desc(dc_smem_u32(ghi)),
                   d_blo = dc_wgmma_desc(dc_smem_u32(glo));

    {   // resident lo half of the W_hh^T slice, once: row rho of tile mt <-> k; a warp reads 32 consecutive k of one row j (128 B)
        const int q = warp & 3, mt = (warp >> 2) & 1, wh = warp >> 3;      // row quadrant, M tile, half of the columns
        const int rho = q * 32 + lane, k = mt * 128 + rho;
#pragma unroll 2
        for (int kap0 = wh * 64; kap0 < wh * 64 + 64; kap0 += 8) {
            float w[8], hi[8], lo[8];
            const int g = kap0 >> 5;
#pragma unroll
            for (int e = 0; e < 8; ++e)
                w[e] = g < G ? __ldg(w_hh + (size_t)(g * H + rank * 32 + (kap0 & 31) + e) * H + k) : 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) { hi[e] = dc_tf32_rna(w[e]); lo[e] = w[e] - hi[e]; }
            unsigned char *panel = wlo + (size_t)(mt * 4 + g) * kPanelA;
            const int c0 = (kap0 & 31) >> 2;
            *reinterpret_cast<float4 *>(panel + swz(rho, c0)) = make_float4(lo[0], lo[1], lo[2], lo[3]);
            *reinterpret_cast<float4 *>(panel + swz(rho, c0 + 1)) = make_float4(lo[4], lo[5], lo[6], lo[7]);
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    // gate phase: thread = (unit ul, sequences sb + 16 i)
    const int ul = lane, unit = rank * 32 + ul, sb = warp;
    bool live[NP];
    float dh_carry[NP], dc_carry[NP], c_cur[NP];
    // per-step inputs, prefetched one step ahead: saved gates, dy, aux0 (LSTM c_{t-1} | GRU hn), aux1 (GRU h_{t-1})
    float cg[NP][G], cdy[NP], ca0[NP], ca1[NP], ng[NP][G], ndy[NP], na0[NP], na1[NP];
    int cslot[NP], nslot[NP];                                                      // reset slots (kReset)
    auto fetch = [&](int t, float (&fg)[NP][G], float (&fdy)[NP], float (&fa0)[NP], float (&fa1)[NP], int (&fsl)[NP]) {
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            const size_t tok = (size_t)t * B + b0 + sb + 16 * i;
            if constexpr (kReset) fsl[i] = live[i] ? __ldg(rs.slot + tok) : -1;
            if (live[i]) {
#pragma unroll
                for (int g = 0; g < G; ++g) fg[i][g] = gates[tok * GH + g * H + unit];
                fdy[i] = __ldg(dy + tok * H + unit);
                if (G == 4) {
                    fa0[i] = cbuf[tok * H + unit];                                 // c_{t-1} (slot t)
                    fa1[i] = 0.f;
                } else {
                    fa0[i] = cbuf[(tok + B) * H + unit];                           // hn (slot t+1)
                    fa1[i] = ybuf[tok * H + unit];                                 // h_{t-1} (slot t)
                }
            } else {
#pragma unroll
                for (int g = 0; g < G; ++g) fg[i][g] = 0.f;
                fdy[i] = fa0[i] = fa1[i] = 0.f;
            }
        }
    };
#pragma unroll
    for (int i = 0; i < NP; ++i) {
        const int b = b0 + sb + 16 * i;
        live[i] = b < B;
        dh_carry[i] = (live[i] && dhn) ? dhn[(size_t)b * H + unit] : 0.f;
        dc_carry[i] = (G == 4 && live[i] && dcn) ? dcn[(size_t)b * H + unit] : 0.f;
        c_cur[i] = (G == 4 && live[i]) ? cbuf[((size_t)S * B + b) * H + unit] : 0.f;
    }
    fetch(S - 1, cg, cdy, ca0, ca1, cslot);
    fetch(S - 1, ng, ndy, na0, na1, nslot);                                        // (initialises the second buffer)
    cluster_barrier();

    for (int it = 0; it < S; ++it) {
        const int t = S - 1 - it;
        // ---- recurrent gradient: fixed-order sum of the 8 CTAs' partials of the previous step, then the gate gradients
        const float *pprev = part + ((size_t)(((it + 1) & 1) * ncl + cl) * kCL) * kNB * H;
        float dgi[NP][G], daux[NP];                                                // global outputs of this step, stored behind the MMAs
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            const int bb = sb + 16 * i;
            float dh = cdy[i] + dh_carry[i];
            if (it > 0) {
                float pv[kCL];
#pragma unroll
                for (int r = 0; r < kCL; ++r) pv[r] = __ldcg(pprev + ((size_t)r * kNB + bb) * H + unit);
#pragma unroll
                for (int r = 0; r < kCL; ++r) dh += pv[r];
            }
            float d[G];                                                            // gradients wrt the h2h pre-activations
#pragma unroll
            for (int g = 0; g < G; ++g) dgi[i][g] = d[g] = 0.f;
            if (live[i]) {
                float prev = G == 3 ? ca1[i] : ca0[i];                             // h_{t-1} | c_{t-1}
                if (kReset && cslot[i] >= 0) prev = rs.prev[((size_t)cslot[i] * B + b0 + bb) * H + unit];
                dh_carry[i] = dc_rnn::cell_bwd<G>([&](int g) { return cg[i][g]; }, G == 3 ? ca0[i] : c_cur[i],   // hn | c_t
                                                  prev, dh, dc_carry[i], dgi[i], d);
                if (G == 4) c_cur[i] = ca0[i];
            }
            daux[i] = d[2];                                                        // GRU: dghn -> cbuf slot t+1
            if (kReset && cslot[i] >= 0) {                                         // nothing flows into step t-1
                dh_carry[i] = dc_carry[i] = 0.f;
#pragma unroll
                for (int g = 0; g < G; ++g) d[g] = 0.f;
            }
            // B operand: row = sequence bb, column kappa = g*32 + ul  ->  K-panel g, 16-byte chunk ul/4, word ul%4
            const int off = swz(bb, ul >> 2) + (ul & 3) * 4;
#pragma unroll
            for (int g = 0; g < G; ++g) {
                const float hi = dc_tf32_rna(d[g]);
                *reinterpret_cast<float *>(ghi + g * kPanelB + off) = hi;
                *reinterpret_cast<float *>(glo + g * kPanelB + off) = d[g] - hi;
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        // 12 G wgmma per warpgroup (G K-panels x 4 k-steps x 3 products), asynchronous until the wait below
        float d[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) d[i] = 0.f;
        acc_fence(d);
        dc_wgmma_fence();
#pragma unroll
        for (int s = 0; s < 4 * G; ++s) {
            const uint64_t adv = (uint64_t)((s & 3) * 2), pa = (uint64_t)(s >> 2) * (kPanelA >> 4), pb = (uint64_t)(s >> 2) * (kPanelB >> 4);
            wgmma_ss(d, d_alo + pa + adv, d_bhi + pb + adv);
            wgmma_rs(d, ahi[s], d_blo + pb + adv);
            wgmma_rs(d, ahi[s], d_bhi + pb + adv);
        }
        dc_wgmma_commit();
        // behind the MMAs: this step's global outputs, then the next step's inputs
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            if (!live[i]) continue;
            const size_t tok = (size_t)t * B + b0 + sb + 16 * i;
            float *gout = gates + tok * GH + unit;
#pragma unroll
            for (int g = 0; g < G; ++g) gout[g * H] = dgi[i][g];
            if (G == 3) cbuf[(tok + B) * H + unit] = daux[i];
        }
        if (t > 0) fetch(t - 1, ng, ndy, na0, na1, nslot);
        dc_wgmma_wait0();
        acc_fence(d);
        {   // partial dh_{t-1}[b][k] of this CTA's 128 gate columns -> scratch [buffer][cluster][rank][b][k]
            float *dst = part + ((size_t)((it & 1) * ncl + cl) * kCL + rank) * kNB * H + 64 * wg;
#pragma unroll
            for (int i = 0; i < 16; ++i) __stcg(dst + (size_t)acc_col(i, lane) * H + acc_row(i, wi, lane), d[i]);
        }
        cluster_arrive();
#pragma unroll
        for (int i = 0; i < NP; ++i) {
#pragma unroll
            for (int g = 0; g < G; ++g) cg[i][g] = ng[i][g];
            cdy[i] = ndy[i]; ca0[i] = na0[i]; ca1[i] = na1[i];
            if constexpr (kReset) cslot[i] = nslot[i];
        }
        cluster_wait();
    }
    // gradient of the initial state
    const float *plast = part + ((size_t)(((S - 1) & 1) * ncl + cl) * kCL) * kNB * H;
#pragma unroll
    for (int i = 0; i < NP; ++i) {
        if (!live[i]) continue;
        const int bb = sb + 16 * i;
        float dh = dh_carry[i];
#pragma unroll
        for (int r = 0; r < kCL; ++r) dh += __ldcg(plast + ((size_t)r * kNB + bb) * H + unit);
        if (dh0) dh0[(size_t)(b0 + bb) * H + unit] = dh;
        if (G == 4 && dc0) dc0[(size_t)(b0 + bb) * H + unit] = dc_carry[i];
    }
}

inline bool cluster_supported(int H) { return H == kH; }

template <typename K, typename... Args>
inline int launch_cluster(K kern, int B, size_t smem, cudaStream_t st, Args... args) {
    DC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(((B + kNB - 1) / kNB) * kCL));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kCL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    DC_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
    return DC_OK;
}

template <bool kReset>
inline int launch_fwd(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf, float *cbuf, int B, int S,
                      dc_rnn::Reset rs, cudaStream_t st) {
    if (cell == DC_CELL_GRU)
        return launch_cluster(fwd_cluster_kernel<3, kReset>, B, FwdSmem::total, st, gates, w_hh, b_hh, ybuf, cbuf, B, S, rs);
    return launch_cluster(fwd_cluster_kernel<4, kReset>, B, FwdSmem::total, st, gates, w_hh, b_hh, ybuf, cbuf, B, S, rs);
}
template <bool kReset>
inline int launch_bwd(int cell, float *gates, const float *w_hh, const float *ybuf, float *cbuf, const float *dy, const float *dhn,
                      const float *dcn, float *dh0, float *dc0, float *part, int B, int S, dc_rnn::Reset rs, cudaStream_t st) {
    if (cell == DC_CELL_GRU)
        return launch_cluster(bwd_cluster_kernel<3, kReset>, B, BwdSmem::total, st, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0,
                              part, B, S, rs);
    return launch_cluster(bwd_cluster_kernel<4, kReset>, B, BwdSmem::total, st, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0,
                          part, B, S, rs);
}

}  // namespace dc_rnnc
