// GAE-lambda advantages and rewards-to-go as a warp-shuffle segmented reverse scan.
//
// Replaces optimizer.py:53-64 (discount / advantage_returns), the per-step reward reduction
// np.sum(s_rewards, axis=1) (optimizer.py:397) and the zero bootstrap (optimizer.py:417-420).
//
// One warp per rollout (segment).  The warp walks the rollout backwards in 32-row tiles aligned
// to the END of the segment: loads are coalesced, the in-tile recurrence y_t = x_t + c*y_{t+1}
// is a 5-step Kogge-Stone scan over shuffles (multiplier c^d squared each step), and the carry
// of the later tile enters as c^(32-lane) * carry.  Accumulation is float64 and rounded once to
// fp32, like scipy.signal.lfilter (float64) + astype(float32); the TD residuals are formed in
// fp32 with the three roundings numpy applies (no FMA contraction).
//
// HBM traffic: (4*n_sub + 4) read + 8 written bytes per row -- 16 B/row with pre-summed rewards.
//
// kIndexed (dc_gae_scan_indexed): the rows stay rollout-major for the rewards, the segments and the bootstraps, but the
// values are read from, and the outputs written to, a token layout of their own: row r reads values[tok[r] * ld_values]
// and writes adv[tok[r]], ret[tok[r]].  tok[r] < 0 reads a value of 0 and writes nothing.  This lets the advantages of a
// training batch ([S, B], one rollout spread over several columns or sharing one) be recomputed where the batch holds
// them, from values read where the head GEMM wrote them.  (4*n_sub + 8 + 4) read + 8 written bytes per row; the value
// and output accesses are gathers.  The arithmetic is the non-indexed kernel's.
//
// Value heads (dc_gae_scan_heads, _indexed): K <= DC_VALUE_HEADS_MAX channels per segment, one per reward group, each with
// its own discount, value column and carries, in the same pass over the tiles; every channel runs the single-value
// kernel's step (gae_tile_channel), and the row's advantage is the channel sum in float64, rounded once.
// (40 + 4K) read + (4 + 4K) written bytes per row (+ 8 read for the token when indexed).
#include "dc_common.cuh"
#include "np_sum.cuh"

namespace {

using dc::np_sum_row;

// c^(32-lane): the weight of the incoming carry for this lane.
__device__ __forceinline__ double carry_weight(int lane, double c) {
    double p = 1.0;
    for (int i = 0; i < 32 - lane; ++i) p *= c;
    return p;
}

// One channel of one 32-row tile, shared by the single-value and the multi-head scans: the TD residual of this lane's
// row from its reward r, its value v and the next row's value (v_after past the tile's last row), then both reverse
// scans with the later tile's carries.  On return a / q are the row's advantage and return (float64, not yet rounded),
// and carry_a, carry_r, v_after hold what the next (earlier) tile needs.
__device__ __forceinline__ void gae_tile_channel(int lane, float r, float v, float gf, double ca, double cr, double pa,
                                                 double pr, float &v_after, double &carry_a, double &carry_r, double &a,
                                                 double &q) {
    float v_next = __shfl_down_sync(0xffffffffu, v, 1);
    if (lane == 31) v_next = v_after;
    // deltas = rewards[:-1] + gamma*values[1:] - values[:-1], three fp32 roundings (optimizer.py:60)
    const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(gf, v_next)), v);
    a = (double)delta;
    q = (double)r;
    double ma = ca, mr = cr;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const double ua = __shfl_down_sync(0xffffffffu, a, d);
        const double uq = __shfl_down_sync(0xffffffffu, q, d);
        if (lane + d < 32) { a += ma * ua; q += mr * uq; }
        ma *= ma; mr *= mr;
    }
    a += pa * carry_a;
    q += pr * carry_r;
    carry_a = __shfl_sync(0xffffffffu, a, 0);
    carry_r = __shfl_sync(0xffffffffu, q, 0);
    v_after = __shfl_sync(0xffffffffu, v, 0);
}

template <bool kIndexed>
__global__ void __launch_bounds__(128) gae_scan_kernel(const float *__restrict__ rewards, int n_sub,
                                                        const float *__restrict__ values,
                                                        const int64_t *__restrict__ seg_off, int n_seg,
                                                        const float *__restrict__ boot_value,
                                                        const float *__restrict__ boot_reward, double gamma,
                                                        double lam, float *__restrict__ adv,
                                                        float *__restrict__ ret, const int64_t *__restrict__ tok,
                                                        int64_t ld_values) {
    const int lane = threadIdx.x & 31;
    const int seg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (seg >= n_seg) return;
    const int64_t lo = seg_off[seg], hi = seg_off[seg + 1];
    if (hi <= lo) return;
    const float gf = (float)gamma;
    const double ca = gamma * lam, cr = gamma;
    const double pa = carry_weight(lane, ca), pr = carry_weight(lane, cr);
    const float boot = boot_value ? boot_value[seg] : 0.0f;
    // discount(rewards)[:-1] starts from the trailing reward element (optimizer.py:63, :419-420: 0)
    double carry_a = 0.0, carry_r = boot_reward ? (double)boot_reward[seg] : 0.0;
    float v_after = boot;  // value of the row following the current tile
    for (int64_t end = hi; end > lo; end -= 32) {
        const int64_t row = end - 32 + lane;
        const bool ok = row >= lo;
        float v = 0.f, r = 0.f;
        int64_t t = row;  // where the row's value and outputs live (the row itself unless kIndexed)
        if (ok) {
            if constexpr (kIndexed) {
                t = tok[row];
                if (t >= 0) v = values[t * ld_values];
            } else {
                v = values[row];
            }
            r = np_sum_row(rewards + row * (int64_t)n_sub, n_sub);
        }
        double a, q;
        gae_tile_channel(lane, r, v, gf, ca, cr, pa, pr, v_after, carry_a, carry_r, a, q);
        if constexpr (kIndexed) {
            if (ok && t >= 0) { adv[t] = (float)a; ret[t] = (float)q; }
        } else {
            if (ok) { adv[row] = (float)a; ret[row] = (float)q; }
        }
    }
}

// The reward groups and discounts of the multi-head scan, passed by value (validated on the host).  Group k sums the
// columns col[off[k]] .. col[off[k+1]-1] of a row, ascending.
struct HeadsArgs {
    double gamma[DC_VALUE_HEADS_MAX];
    int K;
    int8_t off[DC_VALUE_HEADS_MAX + 1];
    int8_t col[128];
};

// K channels per segment in one pass over the tiles: every row's rewards are reduced into the K group sums, every
// channel runs gae_tile_channel with its own discount, value and carries (registers), and the row's advantage is the
// channel sum in float64, rounded once.  Row r of every channel reads its value at values[t * ld_values + k] (t = r, or
// tok[r] when kIndexed) and writes ret[t * K + k]; adv[t].
template <bool kIndexed>
__global__ void __launch_bounds__(128) gae_scan_heads_kernel(const float *__restrict__ rewards, int n_sub,
                                                              const HeadsArgs h, const float *__restrict__ values,
                                                              int64_t ld_values, const int64_t *__restrict__ seg_off,
                                                              int n_seg, const float *__restrict__ boot_value,
                                                              const float *__restrict__ boot_reward, double lam,
                                                              float *__restrict__ adv, float *__restrict__ ret,
                                                              const int64_t *__restrict__ tok) {
    constexpr int kMax = DC_VALUE_HEADS_MAX;
    const int lane = threadIdx.x & 31;
    const int seg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (seg >= n_seg) return;
    const int64_t lo = seg_off[seg], hi = seg_off[seg + 1];
    if (hi <= lo) return;
    const int K = h.K;
    double pa[kMax], pr[kMax], carry_a[kMax], carry_r[kMax];
    float v_after[kMax];
#pragma unroll
    for (int k = 0; k < kMax; ++k) {
        if (k < K) {
            pa[k] = carry_weight(lane, h.gamma[k] * lam);
            pr[k] = carry_weight(lane, h.gamma[k]);
            carry_a[k] = 0.0;
            carry_r[k] = boot_reward ? (double)boot_reward[seg * (int64_t)K + k] : 0.0;
            v_after[k] = boot_value ? boot_value[seg * (int64_t)K + k] : 0.0f;
        }
    }
    for (int64_t end = hi; end > lo; end -= 32) {
        const int64_t row = end - 32 + lane;
        const bool ok = row >= lo;
        int64_t t = row;
        if (ok && kIndexed) t = tok[row];
        const bool has_value = ok && t >= 0;
        const float *rw = rewards + (ok ? row : lo) * (int64_t)n_sub;
        double asum = 0.0;
#pragma unroll
        for (int k = 0; k < kMax; ++k) {
            if (k < K) {
                const float v = has_value ? values[t * ld_values + k] : 0.f;
                float r = 0.f;
                if (ok) {
                    const int8_t *c = h.col + h.off[k];
                    r = dc::np_sum(h.off[k + 1] - h.off[k], [&](int i) { return rw[c[i]]; });
                }
                double a, q;
                gae_tile_channel(lane, r, v, (float)h.gamma[k], h.gamma[k] * lam, h.gamma[k], pa[k], pr[k], v_after[k],
                                 carry_a[k], carry_r[k], a, q);
                asum = k == 0 ? a : asum + a;
                if (has_value) ret[t * K + k] = (float)q;
            }
        }
        if (has_value) adv[t] = (float)asum;
    }
}

}  // namespace

extern "C" int dc_gae_scan(const float *rewards, int n_sub, const float *values, const int64_t *seg_off,
                           int n_seg, const float *boot_value, const float *boot_reward, double gamma, double lam,
                           float *adv, float *ret, dc_stream_t stream) {
    DC_REQUIRE(n_seg >= 0 && n_sub >= 1 && n_sub < 128, DC_EINVAL, "dc_gae_scan: n_seg=%d n_sub=%d", n_seg, n_sub);
    if (n_seg == 0) return DC_OK;
    DC_REQUIRE(rewards && values && seg_off && adv && ret, DC_EINVAL, "dc_gae_scan: null pointer");
    const int warps = 4;
    gae_scan_kernel<false><<<(n_seg + warps - 1) / warps, warps * 32, 0, dc_cu_stream(stream)>>>(
        rewards, n_sub, values, seg_off, n_seg, boot_value, boot_reward, gamma, lam, adv, ret, nullptr, 1);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_gae_scan_indexed(const float *rewards, int n_sub, const float *values, int64_t ld_values,
                                   const int64_t *tok, const int64_t *seg_off, int n_seg, const float *boot_value,
                                   const float *boot_reward, double gamma, double lam, float *adv, float *ret,
                                   dc_stream_t stream) {
    DC_REQUIRE(n_seg >= 0 && n_sub >= 1 && n_sub < 128, DC_EINVAL, "dc_gae_scan_indexed: n_seg=%d n_sub=%d", n_seg,
               n_sub);
    DC_REQUIRE(ld_values >= 1, DC_EINVAL, "dc_gae_scan_indexed: ld_values=%lld must be >= 1", (long long)ld_values);
    if (n_seg == 0) return DC_OK;
    DC_REQUIRE(rewards && values && tok && seg_off && adv && ret, DC_EINVAL, "dc_gae_scan_indexed: null pointer");
    const int warps = 4;
    gae_scan_kernel<true><<<(n_seg + warps - 1) / warps, warps * 32, 0, dc_cu_stream(stream)>>>(
        rewards, n_sub, values, seg_off, n_seg, boot_value, boot_reward, gamma, lam, adv, ret, tok, ld_values);
    DC_LAUNCH_OK();
    return DC_OK;
}

namespace {

// Host-side checks of the multi-head scan's shape arguments; fills the kernel's by-value group table.
int heads_args(const char *fn, int n_sub, const int32_t *group, int K, const double *gammas, double lam, HeadsArgs *h) {
    DC_REQUIRE(K >= 1 && K <= DC_VALUE_HEADS_MAX, DC_EINVAL, "%s: K=%d value heads (1 .. %d)", fn, K, DC_VALUE_HEADS_MAX);
    DC_REQUIRE(n_sub >= 1 && n_sub < 128, DC_EINVAL, "%s: n_sub=%d", fn, n_sub);
    DC_REQUIRE(group && gammas, DC_EINVAL, "%s: null group map or gammas", fn);
    DC_REQUIRE(lam >= 0.0 && lam <= 1.0, DC_EINVAL, "%s: lam=%g outside [0, 1]", fn, lam);
    int n = 0;
    h->K = K;
    for (int k = 0; k < K; ++k) {
        DC_REQUIRE(gammas[k] > 0.0 && gammas[k] <= 1.0, DC_EINVAL, "%s: gammas[%d]=%g outside (0, 1]", fn, k, gammas[k]);
        h->gamma[k] = gammas[k];
        h->off[k] = (int8_t)n;
        for (int i = 0; i < n_sub; ++i)
            if (group[i] == k) h->col[n++] = (int8_t)i;
        DC_REQUIRE(n > h->off[k], DC_EINVAL, "%s: value head %d has no reward column", fn, k);
    }
    h->off[K] = (int8_t)n;
    DC_REQUIRE(n == n_sub, DC_EINVAL, "%s: the group map puts a reward column outside groups 0 .. %d", fn, K - 1);
    return DC_OK;
}

}  // namespace

extern "C" int dc_gae_scan_heads(const float *rewards, int n_sub, const int32_t *group, int K, const float *values,
                                 const int64_t *seg_off, int n_seg, const float *boot_value, const float *boot_reward,
                                 const double *gammas, double lam, float *adv, float *ret, dc_stream_t stream) {
    HeadsArgs h;
    const int rc = heads_args("dc_gae_scan_heads", n_sub, group, K, gammas, lam, &h);
    if (rc != DC_OK) return rc;
    DC_REQUIRE(n_seg >= 0, DC_EINVAL, "dc_gae_scan_heads: n_seg=%d", n_seg);
    if (n_seg == 0) return DC_OK;
    DC_REQUIRE(rewards && values && seg_off && adv && ret, DC_EINVAL, "dc_gae_scan_heads: null pointer");
    const int warps = 4;
    gae_scan_heads_kernel<false><<<(n_seg + warps - 1) / warps, warps * 32, 0, dc_cu_stream(stream)>>>(
        rewards, n_sub, h, values, K, seg_off, n_seg, boot_value, boot_reward, lam, adv, ret, nullptr);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_gae_scan_heads_indexed(const float *rewards, int n_sub, const int32_t *group, int K,
                                         const float *values, int64_t ld_values, const int64_t *tok,
                                         const int64_t *seg_off, int n_seg, const float *boot_value,
                                         const float *boot_reward, const double *gammas, double lam, float *adv,
                                         float *ret, dc_stream_t stream) {
    HeadsArgs h;
    const int rc = heads_args("dc_gae_scan_heads_indexed", n_sub, group, K, gammas, lam, &h);
    if (rc != DC_OK) return rc;
    DC_REQUIRE(n_seg >= 0, DC_EINVAL, "dc_gae_scan_heads_indexed: n_seg=%d", n_seg);
    DC_REQUIRE(ld_values >= K, DC_EINVAL, "dc_gae_scan_heads_indexed: ld_values=%lld must be >= K=%d",
               (long long)ld_values, K);
    if (n_seg == 0) return DC_OK;
    DC_REQUIRE(rewards && values && tok && seg_off && adv && ret, DC_EINVAL, "dc_gae_scan_heads_indexed: null pointer");
    const int warps = 4;
    gae_scan_heads_kernel<true><<<(n_seg + warps - 1) / warps, warps * 32, 0, dc_cu_stream(stream)>>>(
        rewards, n_sub, h, values, ld_values, seg_off, n_seg, boot_value, boot_reward, lam, adv, ret, tok);
    DC_LAUNCH_OK();
    return DC_OK;
}
