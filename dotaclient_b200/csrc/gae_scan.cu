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
#include "dc_common.cuh"
#include "np_sum.cuh"

namespace {

using dc::np_sum_row;

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
    // c^(32-lane): weight of the incoming carry for this lane.
    double pa = 1.0, pr = 1.0;
    for (int i = 0; i < 32 - lane; ++i) { pa *= ca; pr *= cr; }
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
        float v_next = __shfl_down_sync(0xffffffffu, v, 1);
        if (lane == 31) v_next = v_after;
        // deltas = rewards[:-1] + gamma*values[1:] - values[:-1], three fp32 roundings (optimizer.py:60)
        const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(gf, v_next)), v);
        double a = (double)delta, q = (double)r;
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
        if constexpr (kIndexed) {
            if (ok && t >= 0) { adv[t] = (float)a; ret[t] = (float)q; }
        } else {
            if (ok) { adv[row] = (float)a; ret[row] = (float)q; }
        }
        carry_a = __shfl_sync(0xffffffffu, a, 0);
        carry_r = __shfl_sync(0xffffffffu, q, 0);
        v_after = __shfl_sync(0xffffffffu, v, 0);
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
