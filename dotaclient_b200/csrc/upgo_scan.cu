// Upgoing policy update (UPGO; Vinyals et al. 2019, AlphaStar, Methods) as a warp-shuffle segmented reverse scan that
// ADDS coef * A^U into the advantages a base scan (dc_gae_scan / dc_vtrace_scan or their _indexed forms) wrote.
//
// For the rows lo .. hi-1 of one segment, with V_hi := boot (0 or V(s_L) of a cut rollout) and r_t the fp32 reward sum
// of dc_gae_scan:
//   delta_t   = r_t + gamma V_{t+1} - V_t                             float64, three explicit roundings (no FMA)
//   through_t = (t + 1 < hi) and (delta_{t+1} >= 0)                   the next step did at least as well as expected
//   G_t       = r_t + gamma * (through_t ? G_{t+1} : V_{t+1})
//   A^U_t     = rhob_t * (G_t - V_t)
//   adv_t     = fp32((double)adv_t + coef * A^U_t)
// rhob_t = 1 without log-probs (GAE); with them (V-trace) rhob_t = min(rho_clip, exp(sum_h (lp_target - lp_behaviour)))
// computed as vtrace_scan.cu computes it (heads in order, float64, a NaN stays NaN).
//
// One warp per segment, walking it backwards in 32-row tiles aligned to the END of the segment, like vtrace_scan_kernel.
// G_t = x_t + a_t G_{t+1} with x_t = r_t + gamma (1 - through_t) V_{t+1} and a_t = gamma through_t is a 5-step
// Kogge-Stone scan over (a, x) pairs composed as (a1, x1) o (a2, x2) = (a1 a2, x1 + a1 x2); the later tile's G enters as
// x += a_prefix * carry.  Each lane forms its own delta from its row and the next row's value (shuffled down, the later
// tile's first value past the tile's last row); through_t then reads delta_{t+1} the same way.  Everything after the fp32
// reward reduction is float64; each output is rounded once.
//
// Statistics (seg_stats non-NULL): per segment, over its first valid_len rows (all without valid_len), float64 sums in a
// fixed order: 0 the row count, 1 the rows with through_t, 2 the sum of A^U_t (before coef).  Bitwise reproducible.
//
// HBM traffic per row: GAE form 4*n_sub (40) + 4 value + 4 advantage read, 4 advantage written; the V-trace form reads
// 2*20 bytes of log-probs more (each a contiguous 640-byte block per tile, through shared memory); the indexed form reads
// 8 more for the token.
//
// kIndexed (dc_upgo_scan_indexed): the token layout of dc_vtrace_scan_indexed -- row r reads its value at
// values[tok[r] * ld_values], its target log-probs at logp_target[tok[r] * 5 + h] and adds into adv[tok[r]]; tok[r] < 0
// reads 0 for both and writes nothing.  Rewards, segments, bootstraps, behaviour log-probs and valid_len stay
// rollout-major.  The arithmetic is the non-indexed kernel's, so on the same rows both forms agree bit for bit.
#include "dc_common.cuh"
#include "np_sum.cuh"

namespace {

constexpr int kWarps = 4;
constexpr int kHeads = DC_NUM_HEADS;
constexpr int kTileLp = 32 * kHeads;   // log-prob floats per 32-row tile

template <bool kIndexed>
__global__ void __launch_bounds__(kWarps * 32) upgo_scan_kernel(
    const float *__restrict__ rewards, int n_sub, const float *__restrict__ values,
    const float *__restrict__ logp_target, const float *__restrict__ logp_behaviour,
    const int64_t *__restrict__ seg_off, int n_seg, const int64_t *__restrict__ valid_len,
    const float *__restrict__ boot_value, double gamma, double rho_clip, double coef, float *__restrict__ adv,
    double *__restrict__ seg_stats, const int64_t *__restrict__ tok, int64_t ld_values) {
    __shared__ float s_lt[kWarps][kTileLp];
    __shared__ float s_lb[kWarps][kTileLp];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int seg = blockIdx.x * kWarps + warp;
    if (seg >= n_seg) return;
    const bool vtrace = logp_target != nullptr;     // uniform: both log-prob arrays or neither (checked on the host)
    const int64_t lo = seg_off[seg], hi = seg_off[seg + 1];
    // rows [lo, valid_end) are real steps; the rest of the segment is padding, left out of the statistics
    const int64_t valid_end = valid_len ? min(hi, lo + max(valid_len[seg], (int64_t)0)) : hi;
    double st_n = 0.0, st_through = 0.0, st_adv = 0.0;
    double carry_g = 0.0;                                     // G of the row after the tile (the segment's last row never
                                                              // goes through, so its value at the end does not matter)
    double v_after = boot_value ? (double)boot_value[seg] : 0.0;   // V of that row
    double d_after = 0.0;                                     // delta of that row
    for (int64_t end = hi; end > lo; end -= 32) {
        const int64_t base = end - 32;
        const int64_t row = base + lane;
        const bool ok = row >= lo;
        int64_t t = -1;  // kIndexed: the token of this lane's row, where its value, target log-probs and output live
        if constexpr (kIndexed) t = ok ? tok[row] : -1;
        if (vtrace) {
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
            if constexpr (kIndexed) {
#pragma unroll
                for (int h = 0; h < kHeads; ++h)
                    s_lt[warp][lane * kHeads + h] = t >= 0 ? logp_target[t * kHeads + h] : 0.f;
            }
            __syncwarp();
        }
        double v = 0.0, r = 0.0, logrho = 0.0;
        if (ok) {
            if constexpr (kIndexed) {
                if (t >= 0) v = (double)values[t * ld_values];
            } else {
                v = (double)values[row];
            }
            r = (double)dc::np_sum_row(rewards + row * (int64_t)n_sub, n_sub);
            if (vtrace) {
#pragma unroll
                for (int h = 0; h < kHeads; ++h)
                    logrho += (double)s_lt[warp][lane * kHeads + h] - (double)s_lb[warp][lane * kHeads + h];
            }
        }
        // min(clip, rho) written so that a NaN log-prob stays NaN, as vtrace_scan_kernel
        const double rho = exp(logrho);
        const double rhob = vtrace ? (rho > rho_clip ? rho_clip : rho) : 1.0;
        double v_next = __shfl_down_sync(0xffffffffu, v, 1);
        if (lane == 31) v_next = v_after;
        const double q = __dadd_rn(r, __dmul_rn(gamma, v_next));    // r_t + gamma V_{t+1}
        const double delta = __dsub_rn(q, v);
        double d_next = __shfl_down_sync(0xffffffffu, delta, 1);
        if (lane == 31) d_next = d_after;
        const bool through = ok && row + 1 < hi && d_next >= 0.0;
        double x = ok ? (through ? r : q) : 0.0;
        double a = ok ? (through ? gamma : 0.0) : 1.0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const double ua = __shfl_down_sync(0xffffffffu, a, d);
            const double ux = __shfl_down_sync(0xffffffffu, x, d);
            if (lane + d < 32) { x += a * ux; a *= ua; }
        }
        const double g = x + a * carry_g;
        const double au = rhob * (g - v);
        if (ok) {
            if constexpr (kIndexed) {
                if (t >= 0) adv[t] = (float)((double)adv[t] + coef * au);
            } else {
                adv[row] = (float)((double)adv[row] + coef * au);
            }
            if (row < valid_end) {
                st_n += 1.0;
                st_through += through ? 1.0 : 0.0;
                st_adv += au;
            }
        }
        carry_g = __shfl_sync(0xffffffffu, g, 0);
        v_after = __shfl_sync(0xffffffffu, v, 0);
        d_after = __shfl_sync(0xffffffffu, delta, 0);
    }
    if (seg_stats) {
        st_n = dc_warp_sum(st_n);
        st_through = dc_warp_sum(st_through);
        st_adv = dc_warp_sum(st_adv);
        if (lane < DC_UPGO_STATS_SLOTS) {
            const double out = lane == 0 ? st_n : lane == 1 ? st_through : st_adv;
            seg_stats[(int64_t)seg * DC_UPGO_STATS_SLOTS + lane] = out;
        }
    }
}

// The checks both entry points share, before any CUDA call.
int upgo_args(const char *fn, int n_seg, int n_sub, const float *logp_target, const float *logp_behaviour,
              double rho_clip) {
    DC_REQUIRE(n_seg >= 0 && n_sub >= 1 && n_sub < 128, DC_EINVAL, "%s: n_seg=%d n_sub=%d", fn, n_seg, n_sub);
    DC_REQUIRE((logp_target == nullptr) == (logp_behaviour == nullptr), DC_EINVAL,
               "%s: give both log-prob arrays (V-trace) or neither (GAE)", fn);
    DC_REQUIRE(!logp_target || rho_clip > 0.0, DC_EINVAL, "%s: rho_clip=%g must be > 0", fn, rho_clip);
    return DC_OK;
}

}  // namespace

extern "C" int dc_upgo_scan(const float *rewards, int n_sub, const float *values, const float *logp_target,
                            const float *logp_behaviour, const int64_t *seg_off, int n_seg, const int64_t *valid_len,
                            const float *boot_value, double gamma, double rho_clip, double coef, float *adv,
                            double *seg_stats, dc_stream_t stream) {
    const int rc = upgo_args("dc_upgo_scan", n_seg, n_sub, logp_target, logp_behaviour, rho_clip);
    if (rc != DC_OK) return rc;
    if (n_seg == 0) return DC_OK;
    DC_REQUIRE(rewards && values && seg_off && adv, DC_EINVAL, "dc_upgo_scan: null pointer");
    upgo_scan_kernel<false><<<(n_seg + kWarps - 1) / kWarps, kWarps * 32, 0, dc_cu_stream(stream)>>>(
        rewards, n_sub, values, logp_target, logp_behaviour, seg_off, n_seg, valid_len, boot_value, gamma, rho_clip, coef,
        adv, seg_stats, nullptr, 1);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_upgo_scan_indexed(const float *rewards, int n_sub, const float *values, int64_t ld_values,
                                    const float *logp_target, const float *logp_behaviour, const int64_t *tok,
                                    const int64_t *seg_off, int n_seg, const int64_t *valid_len,
                                    const float *boot_value, double gamma, double rho_clip, double coef, float *adv,
                                    double *seg_stats, dc_stream_t stream) {
    const int rc = upgo_args("dc_upgo_scan_indexed", n_seg, n_sub, logp_target, logp_behaviour, rho_clip);
    if (rc != DC_OK) return rc;
    DC_REQUIRE(ld_values >= 1, DC_EINVAL, "dc_upgo_scan_indexed: ld_values=%lld must be >= 1", (long long)ld_values);
    if (n_seg == 0) return DC_OK;
    DC_REQUIRE(rewards && values && tok && seg_off && adv, DC_EINVAL, "dc_upgo_scan_indexed: null pointer");
    upgo_scan_kernel<true><<<(n_seg + kWarps - 1) / kWarps, kWarps * 32, 0, dc_cu_stream(stream)>>>(
        rewards, n_sub, values, logp_target, logp_behaviour, seg_off, n_seg, valid_len, boot_value, gamma, rho_clip, coef,
        adv, seg_stats, tok, ld_values);
    DC_LAUNCH_OK();
    return DC_OK;
}
