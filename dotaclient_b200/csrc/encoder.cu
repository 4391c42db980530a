// Memory-bound pieces of the unit encoder and the target-unit attention head (policy.py:99-136,144-153).
//
// The 128x128 unit-embedding GEMMs run on the tensor cores (gemm_tf32x3.cu); everything around them is
// bandwidth work on ~20 KB/token of activations and is written here so that each tensor crosses HBM once:
//
//   env_fwd / env_bwd   relu(env W_e^T + b_e), 3 -> 128, written into / read from columns [0,128) of the concatenated
//                       [N, 896] pre-rnn input row (no torch.cat), policy.py:55,97
//   unit_basic reduce   fixed-order sum of the dW_b / db_b partials of the fused data-gradient kernel (gemm_tf32x3.cu)
//   target_unit_q_fwd   logits[n,u] = <att[n] W_g, basic[n,u]> + <att[n], b_g>: the head WITHOUT the [N,40,128] embedding
//   target_unit_q_bwd   s_g[n] = sum_u dlogits[n,u] basic_g[n,u] (-> d_att and the head's share of dW_g as token-level GEMMs)
// The basic layer relu(units W_b^T + b_b) ([R,12] -> [R,128], K = 12: not a tensor-core shape) has no kernel of its own: the
// embedding GEMM's producers (dc_unit_embed_fwd) and the target-unit head rebuild it from the raw unit features
// (unit_basic.cuh).  The max-pool over a group's units lives in the embedding GEMM's epilogue and its backward routing is
// generated inside the weight- / data-gradient kernels (dc_unit_wgrad_routed, dc_unit_dgrad_fused), all in gemm_tf32x3.cu.
//
// Thread mapping everywhere: one warp per row of 128 channels, lane l owns channels 4l..4l+3 -> every global access
// is a fully coalesced 512-byte row segment (16 bytes per lane).
#include "dc_common.cuh"
#include "unit_basic.cuh"

namespace {

constexpr int kC = 128;          // embedding width (policy.py:56-63)
constexpr int kIn = kUnitFeatures;
constexpr int kWarps = 8;
constexpr int kThreadsE = kWarps * 32;
constexpr int kMaxUnits = 40;

// ---- dW_b, db_b: fixed-order sum of the [128][13] partials of dc_unit_dgrad_fused (12 weight-gradient columns + the bias gradient)
__global__ void unit_basic_bwd_reduce_kernel(const float *__restrict__ partial, int nblocks, float *__restrict__ dw_b,
                                             float *__restrict__ db_b, int accumulate) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;          // over 128 x 13
    if (i >= kC * (kIn + 1)) return;
    float s = 0.f;
    for (int b = 0; b < nblocks; ++b) s += partial[(size_t)b * kC * (kIn + 1) + i];
    const int o = i / (kIn + 1), k = i % (kIn + 1);
    float *dst = k < kIn ? dw_b + o * kIn + k : db_b + o;
    *dst = accumulate ? *dst + s : s;
}

// ---- environment encoder: relu(env W_e^T + b_e), 3 -> 128 (policy.py:55,97) ---------------------------------------
// Written straight into columns [0,128) of the concatenated pre-rnn input row (row pitch ld), next to the group maxima
// that dc_gemm_unit_max puts in columns [128,896): the reference's torch.cat (policy.py:129-136) never materialises.
constexpr int kEnvIn = 3;
__global__ void __launch_bounds__(kThreadsE) env_fwd_kernel(const float *__restrict__ env, const float *__restrict__ w_e,
                                                            const float *__restrict__ b_e, float *__restrict__ out, int ld,
                                                            int64_t N) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w[4][kEnvIn], b[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        b[c] = b_e[lane * 4 + c];
#pragma unroll
        for (int k = 0; k < kEnvIn; ++k) w[c][k] = w_e[(lane * 4 + c) * kEnvIn + k];
    }
    const int64_t rows_per_iter = (int64_t)gridDim.x * kWarps * 32;
    for (int64_t base = ((int64_t)blockIdx.x * kWarps + warp) * 32; base < N; base += rows_per_iter) {
        const int nrows = (int)min((int64_t)32, N - base);
        float e[kEnvIn];                                           // lane r holds row base+r, rows are broadcast by shuffle
#pragma unroll
        for (int k = 0; k < kEnvIn; ++k) e[k] = lane < nrows ? env[(base + lane) * kEnvIn + k] : 0.f;
        for (int r = 0; r < nrows; ++r) {
            float a[4] = {b[0], b[1], b[2], b[3]};
#pragma unroll
            for (int k = 0; k < kEnvIn; ++k) {
                const float u = __shfl_sync(0xffffffffu, e[k], r);
#pragma unroll
                for (int c = 0; c < 4; ++c) a[c] = fmaf(u, w[c][k], a[c]);
            }
            *reinterpret_cast<float4 *>(out + (base + r) * ld + lane * 4) =
                make_float4(fmaxf(a[0], 0.f), fmaxf(a[1], 0.f), fmaxf(a[2], 0.f), fmaxf(a[3], 0.f));
        }
    }
}

// dW_e, db_e from d_out, the ReLU mask (out > 0) and env: partial[block][128][4] (3 weight columns + bias), then reduced.
__global__ void __launch_bounds__(kThreadsE) env_bwd_kernel(const float *__restrict__ d_out, const float *__restrict__ out, int ld,
                                                            const float *__restrict__ env, int64_t N,
                                                            float *__restrict__ partial) {
    __shared__ float s_red[kC][kEnvIn + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float acc[4][kEnvIn + 1];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int k = 0; k <= kEnvIn; ++k) acc[c][k] = 0.f;
    const int64_t rows_per_iter = (int64_t)gridDim.x * kWarps * 32;
    for (int64_t base = ((int64_t)blockIdx.x * kWarps + warp) * 32; base < N; base += rows_per_iter) {
        const int nrows = (int)min((int64_t)32, N - base);
        float e[kEnvIn];
#pragma unroll
        for (int k = 0; k < kEnvIn; ++k) e[k] = lane < nrows ? env[(base + lane) * kEnvIn + k] : 0.f;
        for (int r0 = 0; r0 < nrows; r0 += 8) {                    // 8 rows per trip: 16 independent 16-byte loads per lane
            float4 g4[8], y4[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int r = min(r0 + j, nrows - 1);
                g4[j] = __ldg(reinterpret_cast<const float4 *>(d_out + (base + r) * ld) + lane);
                y4[j] = __ldg(reinterpret_cast<const float4 *>(out + (base + r) * ld) + lane);
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const bool live = r0 + j < nrows;                  // uniform across the warp
                const float g[4] = {live && y4[j].x > 0.f ? g4[j].x : 0.f, live && y4[j].y > 0.f ? g4[j].y : 0.f,
                                    live && y4[j].z > 0.f ? g4[j].z : 0.f, live && y4[j].w > 0.f ? g4[j].w : 0.f};
#pragma unroll
                for (int k = 0; k < kEnvIn; ++k) {
                    const float u = __shfl_sync(0xffffffffu, e[k], min(r0 + j, 31));
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[c][k] = fmaf(g[c], u, acc[c][k]);
                }
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[c][kEnvIn] += g[c];
            }
        }
    }
    for (int w = 0; w < kWarps; ++w) {                             // fixed fold order: deterministic
        if (warp == w) {
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int k = 0; k <= kEnvIn; ++k) {
                    float *dst = &s_red[lane * 4 + c][k];
                    *dst = (w == 0 ? 0.f : *dst) + acc[c][k];
                }
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < kC * (kEnvIn + 1); i += kThreadsE)
        partial[(size_t)blockIdx.x * kC * (kEnvIn + 1) + i] = (&s_red[0][0])[i];
}

// 32 outputs x 8 block-groups per CTA: group y sums blocks y, y+8, ...; the groups are then added in order.
__global__ void __launch_bounds__(256) env_bwd_reduce_kernel(const float *__restrict__ partial, int nblocks, float *__restrict__ dw_e,
                                                             float *__restrict__ db_e) {
    __shared__ float sh[8][32];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + x;                             // over 128 x 4
    float s = 0.f;
    if (i < kC * (kEnvIn + 1))
        for (int b = y; b < nblocks; b += 8) s += partial[(size_t)b * kC * (kEnvIn + 1) + i];
    sh[y][x] = s;
    __syncthreads();
    if (y == 0 && i < kC * (kEnvIn + 1)) {
        float t = 0.f;
#pragma unroll
        for (int r = 0; r < 8; ++r) t += sh[r][x];
        const int o = i / (kEnvIn + 1), k = i % (kEnvIn + 1);
        if (k < kEnvIn) dw_e[o * kEnvIn + k] = t; else db_e[o] = t;
    }
}

// ---- target-unit head without the unit embedding ------------------------------------------------------------------------
// logits[n,u] = <att[n], W_g basic[n,u] + b_g> = <att[n] W_g, basic[n,u]> + <att[n], b_g> (policy.py:144-153; algebra pinned in
// tests/test_oracle.py): with q[n, g*128 + j] = (att W_g)[n, j] and q[n, 768 + g] = <att[n], b_g> from ONE small GEMM over tokens,
// the head rebuilds the `basic` rows from the raw unit features and the [N, 40, 128] embedding is never materialised.
// A warp owns one token at a time (grid-stride over tokens, so that a lane loads the W_b rows of its 4 channels once): the
// token's 40 raw unit rows (1.9 KB) are staged in the warp's shared-memory slot, every lane reads a row as a broadcast and
// regenerates its 4 channels in registers -- 20 KB per token that are not read from HBM, for 48 FMAs per lane and row.
struct UnitPtrs { const float *p[6]; };
__host__ __device__ constexpr int group_units(int g) { return g == 1 ? 5 : (g == 2 || g == 3) ? 16 : 1; }
__host__ __device__ constexpr int group_offset(int g) { return g == 0 ? 0 : g == 1 ? 1 : g == 2 ? 6 : g == 3 ? 22 : g == 4 ? 38 : 39; }
constexpr int kTokenU4 = kMaxUnits * kIn / 4;                      // 16-byte pieces of a token's raw unit rows

// W_b / b_b of the lane's channels 4l..4l+3
__device__ __forceinline__ void load_basic_weights(float (&w)[4][kIn], float (&b)[4], const float *__restrict__ w_b,
                                                   const float *__restrict__ b_b, int lane) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        b[c] = __ldg(b_b + 4 * lane + c);
#pragma unroll
        for (int k = 0; k < kIn; ++k) w[c][k] = __ldg(w_b + (4 * lane + c) * kIn + k);
    }
}

// token n's unit rows, group after group (row off_g + u at su + 3 (off_g + u)); the caller brackets it with __syncwarp()
__device__ __forceinline__ void stage_token_units(float4 *su, const UnitPtrs &units, int64_t n, int lane) {
#pragma unroll
    for (int g = 0; g < 6; ++g) {
        const int cnt = 3 * group_units(g);
        const float4 *src = reinterpret_cast<const float4 *>(units.p[g]) + n * cnt;
        for (int j = lane; j < cnt; j += 32) su[3 * group_offset(g) + j] = __ldg(src + j);
    }
}

// the lane's 4 channels of the basic row whose raw features are at `row`
__device__ __forceinline__ float4 basic_row(const float4 *row, const float (&w)[4][kIn], const float (&b)[4]) {
    const float4 u0 = row[0], u1 = row[1], u2 = row[2];
    const float u[kIn] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w, u2.x, u2.y, u2.z, u2.w};
    return make_float4(dc_unit_basic(u, w[0], b[0]), dc_unit_basic(u, w[1], b[1]), dc_unit_basic(u, w[2], b[2]),
                       dc_unit_basic(u, w[3], b[3]));
}

// kRows: the head on a row list -- item i < *count is token rows[i], whose q row is row i of the compact q; the logits go to
// row rows[i] and other rows are not written.
template <bool kRows = false>
__global__ void __launch_bounds__(kThreadsE) target_unit_q_fwd_kernel(const float *__restrict__ q, int ld_q, UnitPtrs units,
                                                                      const float *__restrict__ w_b, const float *__restrict__ b_b,
                                                                      float *__restrict__ logits, int64_t N,
                                                                      const int *__restrict__ rows = nullptr,
                                                                      const int *__restrict__ count = nullptr) {
    __shared__ float4 s_u[kWarps][kTokenU4];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w[4][kIn], b[4];
    load_basic_weights(w, b, w_b, b_b, lane);
    float4 *su = s_u[warp];
    if constexpr (kRows) N = min(N, (int64_t)__ldg(count));
    for (int64_t i = (int64_t)blockIdx.x * kWarps + warp; i < N; i += (int64_t)gridDim.x * kWarps) {
        const int64_t n = kRows ? (int64_t)__ldg(rows + i) : i;
        const float *qrow = q + i * ld_q;
        __syncwarp();                                              // the previous token's rows have been read
        stage_token_units(su, units, n, lane);
        __syncwarp();
        float mine = 0.f, mine_hi = 0.f;                          // lane u keeps logit u (u < 32), lanes 0..7 also u+32
#pragma unroll
        for (int g = 0; g < 6; ++g) {
            const float4 a = __ldg(reinterpret_cast<const float4 *>(qrow + g * kC) + lane);
            const float c = __ldg(qrow + 6 * kC + g);
            const int nu = group_units(g), off = group_offset(g);
            for (int u = 0; u < nu; ++u) {
                const float4 v = basic_row(su + 3 * (off + u), w, b);
                float d = v.x * a.x + v.y * a.y + v.z * a.z + v.w * a.w;
                d = dc_warp_sum(d) + c;
                const int o = off + u;
                if (o < 32) { if (lane == o) mine = d; } else { if (lane == o - 32) mine_hi = d; }
            }
        }
        logits[n * kMaxUnits + lane] = mine;
        if (lane < kMaxUnits - 32) logits[n * kMaxUnits + 32 + lane] = mine_hi;
    }
}

// s[n, g*128 + j] = sum_u dlogits[n, off_g + u] basic_g[n,u,j],  s[n, 768 + g] = sum_u dlogits[n, off_g + u]  (zeros elsewhere):
// d_att = s [W_0 | ... | W_5 | b_0..b_5]^T is then one GEMM over tokens.  Tokens that did not use the head write zeros, read nothing.
// kRows: item i < *count is token rows[i]; its s row is row i of the compact s, and no row past the count is written.
template <bool kRows = false>
__global__ void __launch_bounds__(kThreadsE) target_unit_q_bwd_kernel(const float *__restrict__ dlogits, UnitPtrs units,
                                                                      const float *__restrict__ w_b, const float *__restrict__ b_b,
                                                                      float *__restrict__ s, int ld_s, int64_t N,
                                                                      const int *__restrict__ rows = nullptr,
                                                                      const int *__restrict__ count = nullptr) {
    __shared__ float4 s_u[kWarps][kTokenU4];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w[4][kIn], b[4];
    load_basic_weights(w, b, w_b, b_b, lane);
    float4 *su = s_u[warp];
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (kRows) N = min(N, (int64_t)__ldg(count));
    for (int64_t i = (int64_t)blockIdx.x * kWarps + warp; i < N; i += (int64_t)gridDim.x * kWarps) {
        const int64_t n = kRows ? (int64_t)__ldg(rows + i) : i;
        const float g_lo = dlogits[n * kMaxUnits + lane];
        const float g_hi = lane < kMaxUnits - 32 ? dlogits[n * kMaxUnits + 32 + lane] : 0.f;
        const bool any = __any_sync(0xffffffffu, g_lo != 0.f || g_hi != 0.f);
        float4 *srow = reinterpret_cast<float4 *>(s + i * ld_s) + lane;
        if (!any) {
#pragma unroll
            for (int g = 0; g < 7; ++g) srow[g * (kC / 4)] = zero;
            continue;
        }
        __syncwarp();
        stage_token_units(su, units, n, lane);
        __syncwarp();
        float sig[6];
#pragma unroll
        for (int g = 0; g < 6; ++g) {
            const int nu = group_units(g), off = group_offset(g);
            float4 acc = zero;
            float sg = 0.f;
            for (int u = 0; u < nu; ++u) {
                const int o = off + u;
                const float gv = __shfl_sync(0xffffffffu, o < 32 ? g_lo : g_hi, o & 31);
                const float4 v = basic_row(su + 3 * o, w, b);
                acc.x = fmaf(gv, v.x, acc.x); acc.y = fmaf(gv, v.y, acc.y); acc.z = fmaf(gv, v.z, acc.z); acc.w = fmaf(gv, v.w, acc.w);
                sg += gv;
            }
            srow[g * (kC / 4)] = acc;
            sig[g] = sg;
        }
        float4 tail = zero;                                        // columns 768..895: the six sums, then zeros
        if (lane == 0) tail = make_float4(sig[0], sig[1], sig[2], sig[3]);
        if (lane == 1) tail = make_float4(sig[4], sig[5], 0.f, 0.f);
        srow[6 * (kC / 4)] = tail;
    }
}

// Grid of the two head kernels: one warp per token, at most as many blocks as are resident at once (per_sm per SM).
static unsigned head_grid(int per_sm, int64_t N) {
    const int64_t want = (N + kWarps - 1) / kWarps, cap = (int64_t)(per_sm < 1 ? 1 : per_sm) * dc_sm_count();
    return (unsigned)(want < cap ? want : cap);
}

// the six unit arrays of the head: non-null, 16-byte aligned (rows are read as 3 x 16 bytes)
static int unit_ptrs(const float *const units[6], UnitPtrs *up, const char *who) {
    DC_REQUIRE(units != nullptr, DC_EINVAL, "%s: units is NULL", who);
    for (int g = 0; g < 6; ++g) {
        DC_REQUIRE(units[g] && ((uintptr_t)units[g] & 15) == 0, DC_EINVAL, "%s: units[%d] null / not 16-byte aligned", who, g);
        up->p[g] = units[g];
    }
    return DC_OK;
}

}  // namespace

extern "C" size_t dc_unit_basic_bwd_workspace_bytes(void) { return (size_t)4 * 1024 * kC * (kIn + 1) * sizeof(float); }

int dc_unit_basic_reduce(const float *partial, int nblocks, float *dw_b, float *db_b, int accumulate, cudaStream_t st) {
    unit_basic_bwd_reduce_kernel<<<(kC * (kIn + 1) + 255) / 256, 256, 0, st>>>(partial, nblocks, dw_b, db_b, accumulate);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_env_fwd(const float *env, const float *w_e, const float *b_e, float *out, int ld_out, int64_t N,
                          dc_stream_t stream) {
    DC_REQUIRE(env && w_e && b_e && out && N > 0 && ld_out >= kC && ld_out % 4 == 0 && ((uintptr_t)out & 15) == 0, DC_EINVAL,
               "dc_env_fwd: bad arguments");
    env_fwd_kernel<<<4 * dc_sm_count(), kThreadsE, 0, dc_cu_stream(stream)>>>(env, w_e, b_e, out, ld_out, N);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" size_t dc_env_bwd_workspace_bytes(void) { return (size_t)1024 * kC * (kEnvIn + 1) * sizeof(float); }

extern "C" int dc_env_bwd(const float *d_out, const float *out, int ld, const float *env, float *dw_e, float *db_e, int64_t N,
                          void *workspace, dc_stream_t stream) {
    DC_REQUIRE(d_out && out && env && dw_e && db_e && workspace && N > 0 && ld >= kC && ld % 4 == 0, DC_EINVAL,
               "dc_env_bwd: bad arguments");
    DC_REQUIRE((((uintptr_t)d_out | (uintptr_t)out) & 15) == 0, DC_EINVAL, "dc_env_bwd: inputs must be 16-byte aligned");
    cudaStream_t st = dc_cu_stream(stream);
    float *partial = reinterpret_cast<float *>(workspace);
    const int blocks = 2 * dc_sm_count();                          // <= 1024 (workspace bound)
    env_bwd_kernel<<<blocks, kThreadsE, 0, st>>>(d_out, out, ld, env, N, partial);
    DC_LAUNCH_OK();
    env_bwd_reduce_kernel<<<(kC * (kEnvIn + 1) + 31) / 32, 256, 0, st>>>(partial, blocks, dw_e, db_e);
    DC_LAUNCH_OK();
    return DC_OK;
}

template <bool kRows>
static int q_fwd(const float *q, int ld_q, const float *const units[6], const float *w_b, const float *b_b, float *logits, int64_t N,
                 const int32_t *rows, const int32_t *count, dc_stream_t stream, const char *who) {
    DC_REQUIRE(q && w_b && b_b && logits && N > 0 && ld_q >= 7 * kC && ld_q % 4 == 0 && (!kRows || (rows && count)), DC_EINVAL,
               "%s: bad arguments", who);
    UnitPtrs up;
    const int rc = unit_ptrs(units, &up, who);
    if (rc != DC_OK) return rc;
    DC_REQUIRE(((uintptr_t)q & 15) == 0, DC_EINVAL, "%s: alignment", who);
    int per_sm = 0;
    DC_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, target_unit_q_fwd_kernel<kRows>, kThreadsE, 0));
    target_unit_q_fwd_kernel<kRows><<<head_grid(per_sm, N), kThreadsE, 0, dc_cu_stream(stream)>>>(q, ld_q, up, w_b, b_b, logits, N, rows,
                                                                                                  count);
    DC_LAUNCH_OK();
    return DC_OK;
}

template <bool kRows>
static int q_bwd(const float *dlogits, const float *const units[6], const float *w_b, const float *b_b, float *s, int ld_s, int64_t N,
                 const int32_t *rows, const int32_t *count, dc_stream_t stream, const char *who) {
    DC_REQUIRE(dlogits && w_b && b_b && s && N > 0 && ld_s >= 7 * kC && ld_s % 4 == 0 && (!kRows || (rows && count)), DC_EINVAL,
               "%s: bad arguments", who);
    UnitPtrs up;
    const int rc = unit_ptrs(units, &up, who);
    if (rc != DC_OK) return rc;
    DC_REQUIRE(((uintptr_t)s & 15) == 0, DC_EINVAL, "%s: alignment", who);
    int per_sm = 0;
    DC_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, target_unit_q_bwd_kernel<kRows>, kThreadsE, 0));
    target_unit_q_bwd_kernel<kRows><<<head_grid(per_sm, N), kThreadsE, 0, dc_cu_stream(stream)>>>(dlogits, up, w_b, b_b, s, ld_s, N, rows,
                                                                                                  count);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_target_unit_q_fwd(const float *q, int ld_q, const float *const units[6], const float *w_b, const float *b_b,
                                    float *logits, int64_t N, dc_stream_t stream) {
    return q_fwd<false>(q, ld_q, units, w_b, b_b, logits, N, nullptr, nullptr, stream, "dc_target_unit_q_fwd");
}

extern "C" int dc_target_unit_q_bwd(const float *dlogits, const float *const units[6], const float *w_b, const float *b_b, float *s,
                                    int ld_s, int64_t N, dc_stream_t stream) {
    return q_bwd<false>(dlogits, units, w_b, b_b, s, ld_s, N, nullptr, nullptr, stream, "dc_target_unit_q_bwd");
}

extern "C" int dc_target_unit_q_fwd_rows(const float *q, int ld_q, const float *const units[6], const float *w_b, const float *b_b,
                                         float *logits, int64_t N, const int32_t *rows, const int32_t *count, dc_stream_t stream) {
    return q_fwd<true>(q, ld_q, units, w_b, b_b, logits, N, rows, count, stream, "dc_target_unit_q_fwd_rows");
}

extern "C" int dc_target_unit_q_bwd_rows(const float *dlogits, const float *const units[6], const float *w_b, const float *b_b, float *s,
                                         int ld_s, int64_t N, const int32_t *rows, const int32_t *count, dc_stream_t stream) {
    return q_bwd<true>(dlogits, units, w_b, b_b, s, ld_s, N, rows, count, stream, "dc_target_unit_q_bwd_rows");
}

