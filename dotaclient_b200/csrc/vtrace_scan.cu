// V-trace (Espeholt et al. 2018, IMPALA) value targets and policy-gradient advantages as a warp-shuffle segmented
// reverse scan: the off-policy counterpart of gae_scan.cu for rollouts an actor sampled with older weights.
//
// Per row t of a rollout, with the behaviour (actor) and target (prep-time) log-probs of the taken actions:
//   log rho_t = sum_h (lp_target[t,h] - lp_behaviour[t,h])        float64, heads in order
//   rhob_t    = min(rho_clip, exp(log rho_t)),  c_t = lam * min(c_clip, exp(log rho_t))
//   delta_t   = rhob_t * (r_t + gamma V_{t+1} - V_t)
//   vs_t      = V_t + delta_t + gamma c_t (vs_{t+1} - V_{t+1}),    vs_L = V_L = boot
//   A_t       = rhob_t * (r_t + gamma vs_{t+1} - V_t)
// With log rho = 0 and c_clip >= 1 this is GAE(lambda): vs - V is dc_gae_scan's advantage.
//
// One warp per rollout (segment), walking it backwards in 32-row tiles aligned to the END of the segment, like
// gae_scan_kernel.  The recurrence y_t = x_t + a_t y_{t+1} (y = vs - V, x = delta, a = gamma c) has a per-row
// coefficient, so the in-tile scan is a 5-step Kogge-Stone scan over (a, x) pairs composed as
// (a1, x1) o (a2, x2) = (a1 a2, x1 + a1 x2); the later tile's carry enters as x += a_prefix * carry.  Everything after
// the fp32 reward reduction is float64; each output is rounded once to fp32.
//
// HBM traffic per row: 4*n_sub + 4 + 2*20 bytes read, 8 written.  The two [rows, 5] log-prob inputs are read as one
// contiguous 640-byte block per tile each (coalesced) through shared memory.
//
// kIndexed (dc_vtrace_scan_indexed): as gae_scan_kernel<true>, row r reads its value at values[tok[r] * ld_values] and
// its target log-probs at logp_target[tok[r] * 5 + h], and writes pg_adv[tok[r]], vs[tok[r]]; tok[r] < 0 reads 0 for
// both and writes nothing.  Rewards, segments, bootstraps, behaviour log-probs and valid_len stay rollout-major.  Each
// lane stages its own row's five target log-probs into the same shared-memory tile, so the arithmetic is unchanged.
// (4*n_sub + 8 + 4 + 2*20) bytes read, 8 written per row.
#include "dc_common.cuh"
#include "np_sum.cuh"

namespace {

constexpr int kWarps = 4;
constexpr int kHeads = DC_NUM_HEADS;
constexpr int kTileLp = 32 * kHeads;   // log-prob floats per 32-row tile

template <bool kIndexed>
__global__ void __launch_bounds__(kWarps * 32) vtrace_scan_kernel(
    const float *__restrict__ rewards, int n_sub, const float *__restrict__ values,
    const float *__restrict__ logp_target, const float *__restrict__ logp_behaviour,
    const int64_t *__restrict__ seg_off, int n_seg, const int64_t *__restrict__ valid_len,
    const float *__restrict__ boot_value, double gamma, double lam, double rho_clip, double c_clip,
    float *__restrict__ pg_adv, float *__restrict__ vs_out, double *__restrict__ seg_stats,
    const int64_t *__restrict__ tok, int64_t ld_values) {
    __shared__ float s_lt[kWarps][kTileLp];
    __shared__ float s_lb[kWarps][kTileLp];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int seg = blockIdx.x * kWarps + warp;
    if (seg >= n_seg) return;
    const int64_t lo = seg_off[seg], hi = seg_off[seg + 1];
    // rows [lo, valid_end) are real steps; the rest of the segment is padding, left out of the statistics
    const int64_t valid_end = valid_len ? min(hi, lo + max(valid_len[seg], (int64_t)0)) : hi;
    double st_n = 0.0, st_logrho = 0.0, st_rhob = 0.0, st_rho_clipped = 0.0, st_c_clipped = 0.0;
    const double boot = boot_value ? (double)boot_value[seg] : 0.0;
    double carry_y = 0.0;        // vs - V of the row following the current tile (0 at the bootstrap)
    double carry_vs = boot;      // vs of that row
    double v_after = boot;       // V of that row
    for (int64_t end = hi; end > lo; end -= 32) {
        const int64_t base = end - 32;
        // coalesced loads of the tile's two [32, 5] log-prob blocks (rows before lo are not read)
        __syncwarp();
#pragma unroll
        for (int j = 0; j < kHeads; ++j) {
            const int e = j * 32 + lane;
            const int64_t idx = base * kHeads + e;
            const bool in = idx >= lo * kHeads;
            if constexpr (!kIndexed) s_lt[warp][e] = in ? logp_target[idx] : 0.f;
            s_lb[warp][e] = in ? logp_behaviour[idx] : 0.f;
        }
        int64_t t = -1;  // kIndexed: the token of this lane's row, where its value, target log-probs and outputs live
        if constexpr (kIndexed) {
            t = base + lane >= lo ? tok[base + lane] : -1;
#pragma unroll
            for (int h = 0; h < kHeads; ++h) s_lt[warp][lane * kHeads + h] = t >= 0 ? logp_target[t * kHeads + h] : 0.f;
        }
        __syncwarp();
        const int64_t row = base + lane;
        const bool ok = row >= lo;
        double v = 0.0, r = 0.0, logrho = 0.0;
        if (ok) {
            if constexpr (kIndexed) {
                if (t >= 0) v = (double)values[t * ld_values];
            } else {
                v = (double)values[row];
            }
            r = (double)dc::np_sum_row(rewards + row * (int64_t)n_sub, n_sub);
#pragma unroll
            for (int h = 0; h < kHeads; ++h)
                logrho += (double)s_lt[warp][lane * kHeads + h] - (double)s_lb[warp][lane * kHeads + h];
        }
        // min(clip, rho) written so that a NaN log-prob stays NaN (fmin would drop it) and trips the step's NaN guard
        const double rho = exp(logrho);
        const double rhob = rho > rho_clip ? rho_clip : rho;
        const double c = lam * (rho > c_clip ? c_clip : rho);
        double v_next = __shfl_down_sync(0xffffffffu, v, 1);
        if (lane == 31) v_next = v_after;
        double x = ok ? rhob * (r + gamma * v_next - v) : 0.0;
        double a = ok ? gamma * c : 1.0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const double ua = __shfl_down_sync(0xffffffffu, a, d);
            const double ux = __shfl_down_sync(0xffffffffu, x, d);
            if (lane + d < 32) { x += a * ux; a *= ua; }
        }
        const double y = x + a * carry_y;        // vs_t - V_t
        const double vs = v + y;
        double vs_next = __shfl_down_sync(0xffffffffu, vs, 1);
        if (lane == 31) vs_next = carry_vs;
        if (ok) {
            if constexpr (kIndexed) {
                if (t >= 0) {
                    vs_out[t] = (float)vs;
                    pg_adv[t] = (float)(rhob * (r + gamma * vs_next - v));
                }
            } else {
                vs_out[row] = (float)vs;
                pg_adv[row] = (float)(rhob * (r + gamma * vs_next - v));
            }
            if (row < valid_end) {
                st_n += 1.0;
                st_logrho += logrho;
                st_rhob += rhob;
                st_rho_clipped += rho > rho_clip ? 1.0 : 0.0;
                st_c_clipped += rho > c_clip ? 1.0 : 0.0;
            }
        }
        carry_y = __shfl_sync(0xffffffffu, y, 0);
        carry_vs = __shfl_sync(0xffffffffu, vs, 0);
        v_after = __shfl_sync(0xffffffffu, v, 0);
    }
    if (seg_stats) {
        st_n = dc_warp_sum(st_n);
        st_logrho = dc_warp_sum(st_logrho);
        st_rhob = dc_warp_sum(st_rhob);
        st_rho_clipped = dc_warp_sum(st_rho_clipped);
        st_c_clipped = dc_warp_sum(st_c_clipped);
        if (lane < DC_VTRACE_STATS_SLOTS) {
            const double out = lane == 0 ? st_n : lane == 1 ? st_logrho : lane == 2 ? st_rhob
                             : lane == 3 ? st_rho_clipped : lane == 4 ? st_c_clipped : 0.0;
            seg_stats[(int64_t)seg * DC_VTRACE_STATS_SLOTS + lane] = out;
        }
    }
}

}  // namespace

extern "C" int dc_vtrace_scan(const float *rewards, int n_sub, const float *values, const float *logp_target,
                              const float *logp_behaviour, const int64_t *seg_off, int n_seg, const int64_t *valid_len,
                              const float *boot_value, double gamma, double lam, double rho_clip, double c_clip,
                              float *pg_adv, float *vs, double *seg_stats, dc_stream_t stream) {
    DC_REQUIRE(n_seg >= 0 && n_sub >= 1 && n_sub < 128, DC_EINVAL, "dc_vtrace_scan: n_seg=%d n_sub=%d", n_seg, n_sub);
    DC_REQUIRE(rho_clip > 0.0 && c_clip > 0.0, DC_EINVAL, "dc_vtrace_scan: rho_clip=%g c_clip=%g must be > 0", rho_clip,
               c_clip);
    if (n_seg == 0) return DC_OK;
    DC_REQUIRE(rewards && values && logp_target && logp_behaviour && seg_off && pg_adv && vs, DC_EINVAL,
               "dc_vtrace_scan: null pointer");
    vtrace_scan_kernel<false><<<(n_seg + kWarps - 1) / kWarps, kWarps * 32, 0, dc_cu_stream(stream)>>>(
        rewards, n_sub, values, logp_target, logp_behaviour, seg_off, n_seg, valid_len, boot_value, gamma, lam, rho_clip,
        c_clip, pg_adv, vs, seg_stats, nullptr, 1);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_vtrace_scan_indexed(const float *rewards, int n_sub, const float *values, int64_t ld_values,
                                      const float *logp_target, const float *logp_behaviour, const int64_t *tok,
                                      const int64_t *seg_off, int n_seg, const int64_t *valid_len,
                                      const float *boot_value, double gamma, double lam, double rho_clip,
                                      double c_clip, float *pg_adv, float *vs, double *seg_stats,
                                      dc_stream_t stream) {
    DC_REQUIRE(n_seg >= 0 && n_sub >= 1 && n_sub < 128, DC_EINVAL, "dc_vtrace_scan_indexed: n_seg=%d n_sub=%d", n_seg,
               n_sub);
    DC_REQUIRE(ld_values >= 1, DC_EINVAL, "dc_vtrace_scan_indexed: ld_values=%lld must be >= 1", (long long)ld_values);
    DC_REQUIRE(rho_clip > 0.0 && c_clip > 0.0, DC_EINVAL, "dc_vtrace_scan_indexed: rho_clip=%g c_clip=%g must be > 0",
               rho_clip, c_clip);
    if (n_seg == 0) return DC_OK;
    DC_REQUIRE(rewards && values && logp_target && logp_behaviour && tok && seg_off && pg_adv && vs, DC_EINVAL,
               "dc_vtrace_scan_indexed: null pointer");
    vtrace_scan_kernel<true><<<(n_seg + kWarps - 1) / kWarps, kWarps * 32, 0, dc_cu_stream(stream)>>>(
        rewards, n_sub, values, logp_target, logp_behaviour, seg_off, n_seg, valid_len, boot_value, gamma, lam, rho_clip,
        c_clip, pg_adv, vs, seg_stats, tok, ld_values);
    DC_LAUNCH_OK();
    return DC_OK;
}
