/* dotaclient_b200 -- C-ABI of the CUDA-native DotaClient optimizer hot path (H100, sm_90a).
 *
 * The reference (TimZaman/dotaclient @ 8615b90) is pure Python on torch CPU; it has no FFI
 * layer.  Each entry point below replaces a stock-torch/scipy op sequence of the reference's
 * optimizer step and names it (file:line in the reference tree).  A maintainer binds these
 * with ctypes from optimizer.py / policy.py (see INTEGRATION.md).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer (fp32 unless stated), owned by the caller; nothing is
 *     allocated or freed by the library, nothing is synchronised: work is enqueued on `stream`
 *     (a cudaStream_t passed as void*; NULL = legacy default stream).
 *   - return value: 0 = ok; >0 = cudaError_t; <0 = argument error (DC_EINVAL ...).
 *     dc_last_error() returns a thread-local human-readable message for the last failure.
 *   - bool tensors (masks / actions) are bytes holding 0 or 1 (torch.bool layout).
 *   - "time-major" = [S, B, ...]: token (t, b) lives at row t*B + b.
 *   - compiled for sm_90a (H100) only; there is no CPU fallback.
 */
#ifndef DOTACLIENT_B200_H
#define DOTACLIENT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DC_OK 0
#define DC_EINVAL (-1)      /* bad argument */
#define DC_EUNSUPPORTED (-2) /* shape outside what the kernels are built for */

#define DC_CELL_GRU 0  /* gate order r,z,n  (torch.nn.GRU,  policy.py:66) */
#define DC_CELL_LSTM 1 /* gate order i,f,g,o (torch.nn.LSTM; the cell BASELINE.json names) */

#define DC_NUM_HEADS 5    /* enum,x,y,target_unit,ability  (policy.py:46) */
#define DC_LOSS_SLOTS 16  /* layout of the `out` vector of dc_ppo_loss_fwd_bwd, see below */

typedef void *dc_stream_t;

/* Library / device introspection. */
int dc_version(void);
const char *dc_last_error(void);
/* sm count, compute capability of the current device; >0 cudaError_t if there is none. */
int dc_device_info(int *sm_count, int *cc_major, int *cc_minor);

/* ---- GAE -----------------------------------------------------------------------------
 * Replaces advantage_returns()/discount() (optimizer.py:53-64) and the reward reduction that
 * feeds them (optimizer.py:397,417-421) for n_seg rollouts at once.
 *   rewards  [n_rows, n_sub]   sub-rewards per step (n_sub = 10, policy.py:20) or n_sub = 1
 *   values   [n_rows]          critic values (padded steps included, optimizer.py:396)
 *   seg_off  [n_seg+1] int64   rollout r covers rows seg_off[r] .. seg_off[r+1]-1
 *   boot_value [n_seg] or NULL value of the state after the last row   } the trailing elements the
 *   boot_reward[n_seg] or NULL start of the rewards-to-go recursion    } reference appends, both 0
 *                              (NULL = 0: terminated rollouts, optimizer.py:413-420)
 *   adv, ret [n_rows]          outputs
 * deltas in fp32, the two reverse scans accumulate in float64 and round to fp32 exactly like
 * scipy.signal.lfilter + astype(float32) does.  Warp-shuffle segmented scan, one warp / rollout.
 */
int dc_gae_scan(const float *rewards, int n_sub, const float *values, const int64_t *seg_off,
                int n_seg, const float *boot_value, const float *boot_reward, double gamma,
                double lam, float *adv, float *ret, dc_stream_t stream);

/* ---- V-trace -----------------------------------------------------------------------------
 * Off-policy counterpart of dc_gae_scan (Espeholt et al. 2018, IMPALA) for rollouts an actor sampled with older
 * weights: truncated importance weights correct the value targets and the policy-gradient advantages.
 *   rewards, n_sub, values, seg_off, boot_value: as dc_gae_scan (boot_value NULL = 0; there is no boot_reward)
 *   logp_target    [n_rows, 5]  log-prob of the taken action per head under the policy being trained (the dense
 *                               old_logp of dc_selected_logp); 0 where the head took no action
 *   logp_behaviour [n_rows, 5]  the same under the policy the actor sampled with; 0 where the head took no action
 *   valid_len [n_seg] int64 or NULL  the first valid_len[r] rows of segment r are real steps (NULL: all rows)
 *   rho_clip, c_clip > 0        the truncation levels rho-bar and c-bar
 *   pg_adv, vs [n_rows]         outputs: A_t and vs_t below
 *   seg_stats [n_seg][DC_VTRACE_STATS_SLOTS] fp64 or NULL  per-segment sums over the real steps:
 *       0 token count, 1 sum log rho, 2 sum rho-bar_t, 3 #(rho > rho_clip), 4 #(rho > c_clip), 5..7 zero
 * Per row: log rho_t = sum_h (logp_target - logp_behaviour) (fp64, heads in order), rho-bar_t = min(rho_clip, rho_t),
 * c_t = lam min(c_clip, rho_t), r_t = the sub-rewards summed as dc_gae_scan does, and
 *   vs_t = V_t + rho-bar_t (r_t + gamma V_{t+1} - V_t) + gamma c_t (vs_{t+1} - V_{t+1}),   vs_{end} = V_{end} = boot
 *   A_t  = rho-bar_t (r_t + gamma vs_{t+1} - V_t)
 * Float64 throughout after the reward reduction, each output rounded once to fp32.  One warp per segment.
 */
#define DC_VTRACE_STATS_SLOTS 8
int dc_vtrace_scan(const float *rewards, int n_sub, const float *values, const float *logp_target,
                   const float *logp_behaviour, const int64_t *seg_off, int n_seg, const int64_t *valid_len,
                   const float *boot_value, double gamma, double lam, double rho_clip, double c_clip, float *pg_adv,
                   float *vs, double *seg_stats, dc_stream_t stream);

/* ---- GAE / V-trace over a token layout of their own -----------------------------------------
 * The advantage refresh between PPO epochs (DotaOptimizer(recompute_advantages=True)): the same scans, with the same
 * arithmetic, where the rows -- rewards, seg_off, boot_value, boot_reward, logp_behaviour and valid_len, all as above
 * -- stay rollout-major, while each row's value and outputs live at a token of a [S, B] training batch:
 *   tok       [n_rows] int64   the token of row r; tok[r] < 0: the row's value (and target log-probs) read as 0, and
 *                              nothing is written for it
 *   values    value of row r at values[tok[r] * ld_values]; ld_values >= 1 (the packed head output's value column:
 *             ld_values = its row width)
 *   logp_target  [n_tokens, 5] (V-trace) the target log-probs of row r at logp_target[tok[r] * 5 + h]
 *   adv / pg_adv, ret / vs   written at [tok[r]] only; every other element keeps its contents
 * Preconditions the library cannot check (tok is on the device): every tok[r] >= 0 indexes the token arrays, and no
 * two rows share a token.  The caller builds tok on the host and checks it there.
 * Checked: as dc_gae_scan / dc_vtrace_scan, ld_values >= 1 and tok non-null -> DC_EINVAL before any CUDA call.
 */
int dc_gae_scan_indexed(const float *rewards, int n_sub, const float *values, int64_t ld_values, const int64_t *tok,
                        const int64_t *seg_off, int n_seg, const float *boot_value, const float *boot_reward,
                        double gamma, double lam, float *adv, float *ret, dc_stream_t stream);
int dc_vtrace_scan_indexed(const float *rewards, int n_sub, const float *values, int64_t ld_values,
                           const float *logp_target, const float *logp_behaviour, const int64_t *tok,
                           const int64_t *seg_off, int n_seg, const int64_t *valid_len, const float *boot_value,
                           double gamma, double lam, double rho_clip, double c_clip, float *pg_adv, float *vs,
                           double *seg_stats, dc_stream_t stream);

/* ---- UPGO: the upgoing policy update ----------------------------------------------------------
 * DotaOptimizer(upgo_coef=c) (Vinyals et al. 2019, AlphaStar): ADDS c * A^U into the advantages `adv` that one of the
 * scans above wrote, over the same rows and segments.  For the rows lo .. hi-1 of a segment, with V_hi = boot:
 *   delta_t   = r_t + gamma V_{t+1} - V_t                       float64, three roundings, no FMA
 *   through_t = (t + 1 < hi) and (delta_{t+1} >= 0)
 *   G_t       = r_t + gamma * (through_t ? G_{t+1} : V_{t+1})
 *   A^U_t     = rho-bar_t (G_t - V_t),      adv_t = fp32((double)adv_t + coef * A^U_t)
 *   rewards, n_sub, values, seg_off, boot_value (NULL = 0), valid_len: as dc_vtrace_scan
 *   logp_target, logp_behaviour  both NULL (GAE: rho-bar_t = 1) or both given (V-trace: rho-bar_t as dc_vtrace_scan)
 *   rho_clip > 0                 the truncation rho-bar when the log-probs are given
 *   seg_stats [n_seg][DC_UPGO_STATS_SLOTS] fp64 or NULL  per-segment sums over the real steps:
 *       0 token count, 1 #(through_t), 2 sum A^U_t (before coef)
 * The _indexed form has dc_vtrace_scan_indexed's token layout: row r reads values[tok[r] * ld_values] (ld_values >= 1)
 * and logp_target[tok[r] * 5 + h] and adds into adv[tok[r]]; tok[r] < 0 reads 0 and writes nothing.
 * Checked before any CUDA call (DC_EINVAL): n_seg >= 0, 1 <= n_sub < 128, ld_values >= 1, rho_clip > 0 with log-probs,
 * one log-prob array without the other, and null pointers.  Float64 after the reward reduction; one warp per segment.
 */
#define DC_UPGO_STATS_SLOTS 3
int dc_upgo_scan(const float *rewards, int n_sub, const float *values, const float *logp_target,
                 const float *logp_behaviour, const int64_t *seg_off, int n_seg, const int64_t *valid_len,
                 const float *boot_value, double gamma, double rho_clip, double coef, float *adv, double *seg_stats,
                 dc_stream_t stream);
int dc_upgo_scan_indexed(const float *rewards, int n_sub, const float *values, int64_t ld_values,
                         const float *logp_target, const float *logp_behaviour, const int64_t *tok,
                         const int64_t *seg_off, int n_seg, const int64_t *valid_len, const float *boot_value,
                         double gamma, double rho_clip, double coef, float *adv, double *seg_stats, dc_stream_t stream);

/* ---- GAE with one value head per reward group ------------------------------------------------
 * DotaOptimizer(value_heads=...): the sub-rewards of a row are split into K groups, each with its own critic column and
 * discount, all sharing lam.  Per segment, as dc_gae_scan, and per group k:
 *   r_k,t = the fp32 sum of the row's columns in group k, ascending, in the pairwise order np.sum(rewards, axis=1)
 *           applies to a row (np.ascontiguousarray(rewards[:, idx_k]).sum(axis=1))
 *   delta_k,t in fp32 (three roundings), A_k,t = delta_k,t + gamma_k lam A_k,t+1 and R_k,t = r_k,t + gamma_k R_k,t+1
 *   in float64, from the segment's bootstraps boot_value[seg * K + k] / boot_reward[seg * K + k] (NULL = 0)
 * outputs: adv[row] = fp32(sum_k A_k,t) (float64 sum in head order, rounded once), ret[row * K + k] = fp32(R_k,t).
 *   group   [n_sub] int32, HOST: the group 0 .. K-1 of every reward column; every group holds at least one column
 *   gammas  [K] float64, HOST: the discounts, each in (0, 1]
 *   values  [n_rows, K]: head k's value of row r at values[r * K + k]
 * With K = 1 and one group of all columns the results are dc_gae_scan's, bit for bit (the same per-channel step).
 * The _indexed form has dc_gae_scan_indexed's token layout: row r reads values[tok[r] * ld_values + k] (ld_values >= K;
 * the packed head output: its row width) and writes adv[tok[r]] and ret[tok[r] * K + k]; tok[r] < 0 reads 0, writes nothing.
 * Checked before any CUDA call (DC_EINVAL): 1 <= K <= DC_VALUE_HEADS_MAX, 1 <= n_sub < 128, the group map, the gammas,
 * 0 <= lam <= 1, and null pointers.  One warp per segment, every group's channel in the same pass over the tiles.
 */
#define DC_VALUE_HEADS_MAX 10
int dc_gae_scan_heads(const float *rewards, int n_sub, const int32_t *group, int K, const float *values,
                      const int64_t *seg_off, int n_seg, const float *boot_value, const float *boot_reward,
                      const double *gammas, double lam, float *adv, float *ret, dc_stream_t stream);
int dc_gae_scan_heads_indexed(const float *rewards, int n_sub, const int32_t *group, int K, const float *values,
                              int64_t ld_values, const int64_t *tok, const int64_t *seg_off, int n_seg,
                              const float *boot_value, const float *boot_reward, const double *gammas, double lam,
                              float *adv, float *ret, dc_stream_t stream);

/* ---- value loss of K value heads ----------------------------------------------------------------
 * Runs after one of the dc_ppo_loss_fwd_bwd_* entry points that was given a hparams block with DC_HP_VF_COEF = 0 and
 * DC_HP_VALUE_CLIP = 0, on the same stream, and adds the value term of K heads:
 *   value   head k of token t at value[t * ld_value + k] (ld_value >= K: the packed head output's value columns)
 *   ret     [N, K] the value targets; old_value [N, K] or NULL: the prep-time values (clipped loss when
 *           hparams[DC_HP_VALUE_CLIP] > 0); valid [N] or NULL: the tokens that count (NULL: all)
 *   hparams the step's block: DC_HP_VF_COEF and DC_HP_VALUE_CLIP are read
 *   dvalue  written at [t * ld_dvalue + k] for every token: vf_coef (v - R) / N_v (or the clipped term's gradient), 0
 *           on tokens that do not count; N_v = the number of counting tokens (N without a mask)
 *   out     out[3] = vf_coef * 0.5 * sum_k mean (R_k - V_k)^2 (each head PPO2-clipped as the PPO loss clips one), and
 *           out[0] += out[3]
 *   stats   [DC_PPO_STATS_SLOTS] or NULL: DC_STAT_EXPLAINED_VAR = the explained variance of sum_k V_k against sum_k R_k
 *   head_stats [DC_VALUE_HEADS_STATS_SLOTS]: [k] head k's value loss (vf_coef * 0.5 * mean), [DC_VALUE_HEADS_MAX + k]
 *           its explained variance; 0 for k >= K
 *   workspace  DC_VALUE_HEADS_WORKSPACE_BYTES of scratch (zeroed by the call itself)
 * Float64 reductions in a fixed order (bitwise reproducible).  Checked: N > 0, 1 <= K <= DC_VALUE_HEADS_MAX, pitches,
 * null pointers -> DC_EINVAL before any CUDA call.
 */
#define DC_VALUE_HEADS_STATS_SLOTS 20
#define DC_VALUE_HEADS_WORKSPACE_BYTES 131072
int dc_value_heads_loss(const float *value, int64_t ld_value, const float *ret, const float *old_value,
                        const uint8_t *valid, int64_t N, int K, const double *hparams, float *dvalue, int64_t ld_dvalue,
                        float *out, float *stats, float *head_stats, void *workspace, dc_stream_t stream);

/* ---- minibatch assembly: column gather ----------------------------------------------------
 * Picks the sequence columns `index` out of many time-major tensors in ONE launch (the minibatches of PPO epochs,
 * DotaOptimizer.train_epochs; the reference trains on the whole batch and has no counterpart).  Descriptor d describes a
 * contiguous [outer, src_cols, row_bytes] source and a contiguous [outer, n_index, row_bytes] destination; for every
 * o < outer and j < n_index:
 *   dst[(o*n_index + j)*row_bytes + b] = src[(o*src_cols + index[j])*row_bytes + b]         (b < row_bytes)
 * which is torch.index_select(t, 1, index) for each tensor.
 *   descs    host array of n_desc descriptors (0 <= n_desc <= DC_GATHER_MAX_TENSORS), passed by value to the kernel
 *   index    [n_index] int64, DEVICE; repeats allowed
 * Preconditions the library cannot check (the index is on the device): 0 <= index[j] < src_cols for every j.  The
 * caller validates the index where it is made, on the host, before uploading it.
 * Checked: n_desc range, n_index >= 0, outer >= 0, src_cols >= 0, row_bytes > 0, non-null pointers where there is work
 * (src_cols > 0 there too), dst not overlapping src -> DC_EINVAL before any CUDA call.  n_desc == 0 or n_index == 0:
 * nothing to do, returns 0.  Copies in 16-byte units when row_bytes and both base pointers are multiples of 16, else in
 * 4-byte units under the same test, else bytes.
 */
typedef struct {
    const void *src;
    void *dst;
    int64_t outer;
    int64_t src_cols;
    int64_t row_bytes;
} dc_gather_desc;
#define DC_GATHER_MAX_TENSORS 32
int dc_gather_columns(const dc_gather_desc *descs, int n_desc, const int64_t *index, int64_t n_index,
                      dc_stream_t stream);
/* dc_gather_columns_fill: dc_gather_columns, except that index[j] < 0 writes zeros to column j (and reads nothing).
 * Preconditions the library cannot check: -1 <= index[j] < src_cols.  Checked as dc_gather_columns. */
int dc_gather_columns_fill(const dc_gather_desc *descs, int n_desc, const int64_t *index, int64_t n_index,
                           dc_stream_t stream);

/* ---- state refresh between PPO epochs (DotaOptimizer(recompute_states=True)) -------------------------------------
 * After a no-grad forward over time steps [t0, t0 + T) of R rollouts (every layer l's state buffers h_bufs[l] /
 * c_bufs[l], [T + 1, R, H]: slot s holds the state entering step t0 + s), for each destination d < n:
 *   new = h_bufs[l][(step[d] - t0) * R + rollout[d]]  (every layer l; and the c buffer for the LSTM)
 *   slot[d] <  B: written over h0[l, slot[d], :] (and c0), h0 [L, B, H]
 *   slot[d] >= B: written over reset_h[slot[d] - B, l*H : (l+1)*H] (and reset_c), the [K, B, L*H] reset tables
 * and acc[0] += sum (new - old)^2, acc[1] += sum old^2 over every float written, in float64, in a fixed order (no atomics;
 * two calls on the same data give the same bits).  partial: device workspace of 2 * n * n_layers doubles.
 * c_bufs / c0 / reset_c: NULL for the GRU.  All state pointers 16-byte aligned.
 * Preconditions the library cannot check (the tables are on the device): t0 <= step[d] <= t0 + T, 0 <= rollout[d] < R,
 * 0 <= slot[d] < B + K*B, and no slot twice.  The caller builds and checks them on the host.
 * Checked: 1 <= n_layers <= DC_REFRESH_MAX_LAYERS, H a positive multiple of 32, R, B >= 1, K, n, t0 >= 0, non-null and
 * aligned pointers where there is work -> DC_EINVAL before any CUDA call.  n = 0 does nothing.
 */
#define DC_REFRESH_MAX_LAYERS 16
int dc_refresh_states(int n_layers, int H, const float *const *h_bufs, const float *const *c_bufs, int64_t R, int64_t t0,
                      const int64_t *step, const int64_t *rollout, const int64_t *slot, int64_t n, int64_t B, int64_t K,
                      float *h0, float *c0, float *reset_h, float *reset_c, double *partial, double *acc,
                      dc_stream_t stream);

/* ---- recurrent core --------------------------------------------------------------------
 * Replaces the time recurrence inside nn.GRU / nn.LSTM (policy.py:66,141) -- forward and
 * backward -- given the input-to-hidden pre-activations of all steps.
 *
 * Forward
 *   gates  [S, B, G, H] in : x_t W_ih^T + b_ih (time-major)      G = 3 (GRU) / 4 (LSTM)
 *                       out: activated gates (r,z,n | i,f,g,o), saved for backward (in place)
 *   w_hh   [G*H, H], b_hh [G*H]   rnn.weight_hh_l0 / rnn.bias_hh_l0
 *   ybuf   [S+1, B, H]  slot 0 = h_0 (in), slot t+1 = h_t (out)   -> y = ybuf[1:], h_n = ybuf[S]
 *   cbuf   [S+1, B, H]  LSTM: slot 0 = c_0 (in), slot t+1 = c_t (out)
 *                       GRU : slot t+1 = W_hn h_{t-1} + b_hn (out, saved for backward)
 *   workspace: dc_rnn_workspace_bytes(cell, B, H) bytes of scratch; the same buffer serves forward and backward.  It holds
 *              W_hh^T at H = 128 and for the generic kernels, the partial-sum exchange of the cluster backward kernel at
 *              H = 256, and W_hh^T plus the split-K partials and carries of the step-wise kernels at the other multiples of 128.
 * Kernels by width: H = 128 one-SM weight-resident FFMA kernels; H = 256 (the reference's width) 8-CTA-cluster
 * weight-resident wgmma 3xTF32 kernels; other multiples of 128 (384, 512, ...) step-wise kernels: per step a split-K
 * wgmma 3xTF32 GEMM over all SMs that streams W_hh from L2, then a gate kernel; any other H % 4 == 0 a generic kernel
 * that streams W_hh from L2 (through the Python layers: every other H % 32 == 0, e.g. 64, 96, 160, 192).
 * Backward (consumes what forward left behind)
 *   gates  in: activated gates   out: dL/d(gates pre-activation wrt the i2h branch) = dgi
 *   cbuf   LSTM: unchanged.  GRU: slot t+1 out = dL/d(W_hn h + b_hn) (the n-gate part of dgh)
 *   dy     [S, B, H]  dL/dy (time-major); dhn/dcn [B, H] or NULL (gradient of the final state)
 *   dh0/dc0 [B, H] or NULL outputs.
 */
size_t dc_rnn_workspace_bytes(int cell, int B, int H);
int dc_rnn_seq_fwd(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf,
                   float *cbuf, int B, int S, int H, void *workspace, dc_stream_t stream);
int dc_rnn_seq_bwd(int cell, float *gates, const float *w_hh, const float *ybuf, float *cbuf,
                   const float *dy, const float *dhn, const float *dcn, float *dh0, float *dc0,
                   int B, int S, int H, void *workspace, dc_stream_t stream);

/* Same recurrence with recurrent-state RESETS inside a sequence: several segments (e.g. the tails of different rollouts
 * packed into one training sequence) share one column, and each later segment restarts from its own state.
 *   reset_slot [S, B] int32   k = reset_slot[t*B + b]: -1 carries the state; k >= 0 replaces the state entering step t of
 *                             sequence b (at t = 0 it overrides h_0 / c_0) with row k*B + b of the tables below
 *   reset_prev [K, B, H]      GRU: the reset h; LSTM: the reset c (the cell's previous-state operand)
 *   reset_pre  [K, B, G*H]    forward only: h_reset W_hh^T + b_hh of the reset h (the caller computes it once, a GEMM of
 *                             K*B rows)
 *   K >= 0                    rows per column of the tables (NULL tables are allowed when K = 0)
 * Forward: at a reset token the cell reads its h2h pre-activation from reset_pre and its previous state from reset_prev; the
 * step's mat-vec on the stale state is discarded.  The saved tensors keep their meaning (ybuf slot t+1 = h_t, the GRU's cbuf
 * aux = the W_hn h + b_hn the cell used).  Backward: at a reset token prev comes from reset_prev and no gradient flows into
 * step t-1 (neither through W_hh nor through the direct dh z / dc f path); a reset at t = 0 leaves dh0 / dc0 zero for b.
 * The weight gradient dW_hh = dgh^T ybuf[:S] that the caller forms is then wrong at the reset tokens by
 * dgh_t^T (h_reset - ybuf[t]): the caller adds that correction.  db_hh needs none.  The reset states get no gradient.
 * Every design (H = 128, 256, other multiples of 128, generic) has a reset instantiation; the plain entry points above run
 * the instantiations without it.  With every slot at -1 the results are bit-identical to dc_rnn_seq_fwd / _bwd.
 * Preconditions the library cannot check (the slots are on the device): -1 <= reset_slot < K.  Checked before any CUDA
 * call: the arguments of dc_rnn_seq_fwd / _bwd, reset_slot != NULL, K >= 0, non-null tables when K > 0 -> DC_EINVAL. */
int dc_rnn_seq_fwd_reset(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf, float *cbuf,
                         const int32_t *reset_slot, const float *reset_prev, const float *reset_pre, int K,
                         int B, int S, int H, void *workspace, dc_stream_t stream);
int dc_rnn_seq_bwd_reset(int cell, float *gates, const float *w_hh, const float *ybuf, float *cbuf,
                         const float *dy, const float *dhn, const float *dcn, float *dh0, float *dc0,
                         const int32_t *reset_slot, const float *reset_prev, int K,
                         int B, int S, int H, void *workspace, dc_stream_t stream);

/* ---- fp32-accurate tensor-core GEMM (wgmma, 3xTF32) ---------------------------------------
 * C[M,N] = A[M,K] * B[N,K]^T (+ bias[N]) (ReLU if relu != 0); row-major fp32 with leading dimensions lda/ldb/ldc.
 * Replaces the library SGEMM of the input-to-hidden projection inside nn.GRU / nn.LSTM (policy.py:66,141:
 * gates = x W_ih^T + b_ih) and of the other dense layers (policy.py:101-126,138).  Each product is
 * evaluated as a_lo*b_hi + a_hi*b_lo + a_hi*b_hi with tf32 hi/lo splits (fp32-level accuracy, ~1e-6 relative).
 * Requirements: N % 32 == 0, K % 32 == 0, 16-byte aligned pointers, ld* % 4 == 0 (dc_gemm_tf32x3_supported).  With N % 128 != 0
 * the last 128-column tile is partly filled; nothing is stored past column N.  So every layer of a Policy whose width H is a
 * multiple of 32 has a GEMM here (N or K = H, 3H, 4H, 128, 896).
 */
int dc_gemm_tf32x3_supported(int64_t M, int N, int K);
int dc_gemm_tf32x3(const float *A, int lda, const float *B, int ldb, const float *bias, float *C, int ldc,
                   int64_t M, int N, int K, int relu, dc_stream_t stream);

/* Weight gradient of the same layers: dW[No,Ni] (+)= dY[T,No]^T X[T,Ni], db[No] (+)= column sums of dY (NULL = skip).
 * Replaces the dW/db part of AddmmBackward for those layers (loss.backward(), optimizer.py:672).  Contraction over the
 * token dimension (operands transposed to K-major on the way into shared memory), split-K over the SMs, deterministic two-stage reduction.
 * Requirements: No % 32 == 0, Ni % 32 == 0; workspace of dc_gemm_wgrad_workspace_bytes(No, Ni) bytes (one full 128 x 128
 * partial per output tile and split, tiles = ceil(No/128) * ceil(Ni/128)). */
size_t dc_gemm_wgrad_workspace_bytes(int No, int Ni);
int dc_gemm_wgrad_tf32x3(const float *dY, int ldy, const float *X, int ldx, int64_t T, int No, int Ni,
                         float *dW, int ldw, float *db, int accumulate, void *workspace, dc_stream_t stream);
/* The same two GEMMs on a row list held on the device (dc_target_rows; a graph replays them whatever the count):
 * dc_gemm_tf32x3_rows computes rows i < min(M, *count) of a A'^T B (+ bias) with A' row i = A row (gather_a ? rows[i] : i); row i goes
 * to C row i (C may be NULL) and to C_rows row rows[i] (C_rows may be NULL; not both NULL), both with pitch ldc.  No other row is
 * read or written; M sizes the grid.  dc_gemm_wgrad_tf32x3_rows contracts tokens t < min(T, *t_dev) with X row x_rows[t] (x_rows NULL:
 * row t), split over every split-K range; at count 0, dW = 0, db = 0 (accumulate = 0).  The same requirements and workspace as above. */
int dc_gemm_tf32x3_rows(const float *A, int lda, const float *B, int ldb, const float *bias, float *C, float *C_rows, int ldc,
                        int64_t M, const int32_t *count, const int32_t *rows, int gather_a, int N, int K, int relu, dc_stream_t stream);
int dc_gemm_wgrad_tf32x3_rows(const float *dY, int ldy, const float *X, int ldx, const int32_t *x_rows, int64_t T, const int32_t *t_dev,
                              int No, int Ni, float *dW, int ldw, float *db, int accumulate, void *workspace, dc_stream_t stream);

/* ---- unit encoder / target-unit head ------------------------------------------------------------
 * (policy.py:99-136,144-153).  The basic layer basic[R,128] = relu(units[R,12] W_b^T + b_b) (policy.py:100,105,...) is
 * rebuilt from the raw unit features by every kernel that reads it, bit for bit the same value everywhere. */
size_t dc_unit_basic_bwd_workspace_bytes(void);   /* partial sums of dW_b / db_b: the workspace of dc_unit_dgrad_fused */
/* Environment encoder (policy.py:55,97): out[n*ld_out + c] = relu(env[n,:3] . W_e[c,:] + b_e[c]), c < 128 -- written into
 * columns [0,128) of the concatenated pre-rnn input row (ld_out = 896), so the reference's torch.cat (policy.py:129-136)
 * is never materialised.  dc_env_bwd: dW_e[128,3] = (d_out * (out>0))^T env, db_e[128] = column sums (deterministic). */
int dc_env_fwd(const float *env, const float *w_e, const float *b_e, float *out, int ld_out, int64_t N,
               dc_stream_t stream);
size_t dc_env_bwd_workspace_bytes(void);
int dc_env_bwd(const float *d_out, const float *out, int ld, const float *env, float *dw_e, float *db_e, int64_t N,
               void *workspace, dc_stream_t stream);
/* Unit-embedding layer with the max-pool fused into the GEMM epilogue (policy.py:101-127): emb = basic[N*n_units,128] W^T is
 * reduced per token to xmax[n*ld_x + c] = max_u emb[n,u,c] + b[c] (also written to xmax_copy when not NULL, policy.py:127) and
 * argmax[n*128 + c] (first maximum wins, like torch.max); the embedding itself is never stored.  n_units = 5 or 16. */
int dc_gemm_unit_max(const float *basic, const float *w, const float *bias, float *xmax, float *xmax_copy, int ld_x,
                     uint8_t *argmax, int64_t n_tokens, int n_units, dc_stream_t stream);
/* One unit-embedding group's forward in one launch: the basic layer of units [N*n_units, 12] (w_b [128,12], b_b [128]) is
 * generated inside the embedding GEMM and, when basic_out is not NULL, also stored there ([N*n_units, 128], what the weight
 * gradients read).  n_units 5, 16: the max-pool epilogue of dc_gemm_unit_max (xmax, xmax_copy, argmax; same results bit for
 * bit as dc_gemm_unit_max on the stored basic).  n_units 1: xmax[n*ld_x + c] = (basic W^T)[n,c] + b[c], argmax and
 * xmax_copy NULL.  units, basic_out, w, bias, xmax, xmax_copy 16-byte aligned; ld_x >= 128, a multiple of 4. */
int dc_unit_embed_fwd(const float *units, const float *w_b, const float *b_b, float *basic_out, const float *w, const float *bias,
                      float *xmax, float *xmax_copy, int ld_x, uint8_t *argmax, int64_t n_tokens, int n_units, dc_stream_t stream);
/* dc_unit_embed_fwd that also stores the basic layer's ReLU mask when mask_out is not NULL: mask_out[row*4 + c%4] bit c/4
 * = (basic[row][c] > 0), 16 bytes per unit row ([N*n_units][4] words, 16-byte aligned) -- what dc_unit_dgrad_fused_mask reads. */
int dc_unit_embed_fwd_mask(const float *units, const float *w_b, const float *b_b, float *basic_out, uint32_t *mask_out, const float *w,
                           const float *bias, float *xmax, float *xmax_copy, int ld_x, uint8_t *argmax, int64_t n_tokens, int n_units,
                           dc_stream_t stream);
/* Target-unit head without the embedding (policy.py:144-153): logits[n,u] = <q[n, g*128 ..], basic_g[n,u,:]> + q[n, 768+g]
 * with q = att [W_0|...|W_5|b_0..b_5] (ld_q >= 896) and basic_g = relu(units[g] W_b^T + b_b) rebuilt from the raw unit
 * features units[g] [N*units_g, 12] (units 1,5,16,16,1,1; 16-byte aligned).  Backward: s[n, g*128 + j] = sum_u dlogits[n,u]
 * basic_g[n,u,j], s[n, 768+g] = sum_u dlogits[n,u] (zeros in 774..895), so that d_att = s [W_0|...|W_5|b]^T is one GEMM;
 * tokens whose dlogits row is all zero get a zero row of s. */
int dc_target_unit_q_fwd(const float *q, int ld_q, const float *const units[6], const float *w_b, const float *b_b, float *logits,
                         int64_t N, dc_stream_t stream);
int dc_target_unit_q_bwd(const float *dlogits, const float *const units[6], const float *w_b, const float *b_b, float *s, int ld_s,
                         int64_t N, dc_stream_t stream);
/* The head on the tokens of a row list (dc_target_rows): item i < min(N, *count) is token rows[i].  _fwd reads row i of q
 * and writes logits row rows[i] (no other row is written); _bwd reads dlogits row rows[i] and writes row i of s (no row
 * past the count is written).  N: the capacity of rows, q and s. */
int dc_target_unit_q_fwd_rows(const float *q, int ld_q, const float *const units[6], const float *w_b, const float *b_b, float *logits,
                              int64_t N, const int32_t *rows, const int32_t *count, dc_stream_t stream);
int dc_target_unit_q_bwd_rows(const float *dlogits, const float *const units[6], const float *w_b, const float *b_b, float *s, int ld_s,
                              int64_t N, const int32_t *rows, const int32_t *count, dc_stream_t stream);
/* The tokens that use the target-unit head: rows[0 .. *count) = the n < N, ascending, whose target_unit mask row or action
 * row (mask, action: [N, 40] bool bytes, 8-byte aligned) has a byte set -- the rows the PPO loss reads -- and flags[n] = 1 for
 * them, 0 for the others ([N] bytes, 4-byte aligned).  All outputs stay on the device.  Workspace:
 * dc_target_rows_workspace_bytes(N) bytes, 4-byte aligned.
 * dc_rows_zero_inactive: dst[n, :width] = 0 for every n < N with flags[n] == 0 (width % 4 == 0, 16-byte aligned rows). */
size_t dc_target_rows_workspace_bytes(int64_t N);
int dc_target_rows(const uint8_t *mask, const uint8_t *action, int64_t N, int32_t *rows, int32_t *count, uint8_t *flags,
                   void *workspace, dc_stream_t stream);
int dc_rows_zero_inactive(const uint8_t *flags, int64_t N, float *dst, int ld, int width, dc_stream_t stream);
/* Backward of one unit-embedding layer WITHOUT the dense [N*units, 128] gradient of the embedding (what the reference's autograd
 * materialises behind policy.py:100-127,152-153).  R[(n,u), c] = (argmax[n*128 + c] == u) ? d_xmax[n*ld_dx + c] (+ d_xmax2[..]) : 0 is
 * the max-pool routing, generated inside the kernels.
 *   dc_unit_wgrad_routed  dW[128,128] = R^T basic,  db[128] = column sums of R            (n_units = 5 or 16; a 1-unit group is
 *                         dc_gemm_wgrad_tf32x3 on d_xmax itself; workspace: dc_gemm_wgrad_workspace_bytes(128, 128))
 *   dc_unit_dgrad_fused   dW_b[128,12] (+)= G^T units, db_b[128] (+)= column sums of G, with
 *                         G[(n,u), j] = (basic[(n,u), j] > 0) * sum_c (R[(n,u), c] + dlogits[n*ld_dl + u] att[n*128 + c]) W[c, j]:
 *                         the whole gradient of the embedding (routing + the target-unit head's rank-1 part) is generated inside
 *                         the kernel; w_t = W^T [128,128]; the ReLU mask is recomputed from units/w_b/b_b (bit-identical to
 *                         the forward value); dlogits (already offset to the group's first unit) and att [N,128] are NULL when the
 *                         head was not used; d_xmax NULL = no routing (the enemy-tower layer, policy.py:127).  n_units = 1, 5 or
 *                         16; units, att, d_xmax 16-byte aligned; workspace: dc_unit_basic_bwd_workspace_bytes().
 *   dc_unit_dgrad_fused_mask  the same with the ReLU mask read from `mask` (the words dc_unit_embed_fwd_mask stored for these
 *                         unit rows, 16-byte aligned) instead of recomputed; mask NULL = dc_unit_dgrad_fused.  dW_b / db_b are
 *                         bitwise the same either way.
 * The head's share of dW / db is a token-level product (att^T s, s from dc_target_unit_q_bwd) the caller adds. */
int dc_unit_wgrad_routed(const float *d_xmax, const float *d_xmax2, int ld_dx, const uint8_t *argmax, const float *basic,
                         int64_t n_tokens, int n_units, float *dW, float *db, void *workspace, dc_stream_t stream);
int dc_unit_dgrad_fused(const float *d_xmax, const float *d_xmax2, int ld_dx, const uint8_t *argmax, const float *dlogits,
                        int ld_dl, const float *att, const float *w_t, const float *units, const float *w_b,
                        const float *b_b, int64_t n_tokens, int n_units, float *dw_b, float *db_b, int accumulate,
                        void *workspace, dc_stream_t stream);
int dc_unit_dgrad_fused_mask(const float *d_xmax, const float *d_xmax2, int ld_dx, const uint8_t *argmax, const float *dlogits,
                             int ld_dl, const float *att, const float *w_t, const float *units, const uint32_t *mask, const float *w_b,
                             const float *b_b, int64_t n_tokens, int n_units, float *dw_b, float *db_b, int accumulate,
                             void *workspace, dc_stream_t stream);

/* ---- fused PPO loss + gradient ----------------------------------------------------------
 * Replaces optimizer.py:587-589 (advantage normalisation) and :621-665 (masked log-softmax x5,
 * ratio, clipped surrogate, entropy, value loss) AND their autograd backward, for N tokens.
 *   logits[h]  [N, n_h] fp32   n_h = 4,9,9,40,3     masks[h], actions[h] [N, n_h] bytes
 *   old_logp   [N, 5]   log-prob of the taken action per head at prep time (dense form of
 *                       Sequence.log_probs_sel, optimizer.py:387-390); ignored where no action
 *   adv_raw, ret, value [N]
 *   dlogits[h] [N, n_h], dvalue [N]   gradients of the total loss (loss.backward(), :672)
 *   out [DC_LOSS_SLOTS] fp32: 0 loss, 1 policy_loss, 2 entropy_loss, 3 value_loss,
 *       4..8 entropy per head, 9..13 policy loss per head, 14 adv mean, 15 adv std (unbiased)
 *   n_actions [5] int32: rows with a taken action per head (optimizer.py:626,643)
 *   workspace: DC_PPO_WORKSPACE_BYTES of scratch (zeroed by the call itself).
 * Two launches: statistics (counts, advantage mean/std), then loss+grad.
 */
#define DC_PPO_WORKSPACE_BYTES 512
int dc_ppo_loss_fwd_bwd(const float *const logits[DC_NUM_HEADS],
                        const uint8_t *const masks[DC_NUM_HEADS],
                        const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                        const float *adv_raw, const float *ret, const float *value, int64_t N,
                        float e_clip, float entropy_coef, float vf_coef,
                        float *const dlogits[DC_NUM_HEADS], float *dvalue, float *out,
                        int32_t *n_actions, void *workspace, dc_stream_t stream);

/* Same, with row pitches (floats) for logits[h], dlogits[h], value and dvalue: a pitch of 128 lets the four small heads
 * and the value head be column ranges of ONE packed [N,128] tensor-core GEMM output and of its gradient. */
int dc_ppo_loss_fwd_bwd_strided(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                const uint8_t *const masks[DC_NUM_HEADS],
                                const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                                const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                int64_t N, float e_clip, float entropy_coef, float vf_coef,
                                float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                                float *dvalue, int64_t ld_dvalue, float *out, int32_t *n_actions,
                                void *workspace, dc_stream_t stream);

/* ---- device-resident hyper-parameters --------------------------------------------------
 * The `_dev` entry points read their scalar hyper-parameters from a small DEVICE block of DC_HPARAM_SLOTS fp64 values
 * instead of from kernel arguments, so a CUDA graph that captured them sees new values on every replay (the caller
 * rewrites the block with an asynchronous copy before launching).  Each value is rounded to the type the scalar-argument
 * entry point uses: e_clip, entropy_coef, vf_coef, value_clip to float, lr to double, max_grad_norm to float, so at the
 * same values the results are bit-identical to dc_ppo_loss_fwd_bwd_strided / dc_grad_finish.
 */
#define DC_HPARAM_SLOTS 10
#define DC_HP_LR 0             /* Adam learning rate                                               */
#define DC_HP_E_CLIP 1         /* PPO ratio clip range epsilon                                     */
#define DC_HP_ENTROPY_COEF 2
#define DC_HP_VF_COEF 3
#define DC_HP_MAX_GRAD_NORM 4  /* global gradient-norm clip                                        */
#define DC_HP_VALUE_CLIP 5     /* PPO2 value clip range; <= 0: unclipped value loss                 */
#define DC_HP_VALUE_NORM_MEAN 6 /* value normalisation mu (read only when slot 7 > 0)               */
#define DC_HP_VALUE_NORM_STD 7  /* value normalisation sigma; <= 0: off (the plain value loss)      */
#define DC_HP_KL_COEF 8        /* KL penalty coefficient beta (read by dc_ppo_loss_fwd_bwd_kl only) */
#define DC_HP_KL_STOP 9        /* KL limit of dc_grad_finish_kl; <= 0: no limit                    */

/* Loss + gradient as dc_ppo_loss_fwd_bwd_strided, hyper-parameters from `hparams` [DC_HPARAM_SLOTS] (device), plus:
 *   old_value [N] fp32 or NULL: critic values at experience prep.  When hparams[DC_HP_VALUE_CLIP] = eps > 0 and
 *       old_value is not NULL, the value loss is 0.5*vf_coef*mean(max((v-R)^2, (v_old + clip(v-v_old, -eps, eps) - R)^2))
 *       and its gradient goes through the larger branch; otherwise it is exactly the unclipped loss.
 *   stats [DC_PPO_STATS_SLOTS] fp32 out, or NULL to skip: accumulated in the same pass over the tokens, in float64:
 *       0 approximate KL (k3 estimator (r-1) - log r, r = exp(logp - old_logp)), the mean over the heads with action rows;
 *       1..5 per head, averaged over the head's action rows (0 for a head without any);
 *       6 clip fraction (share of action rows with |r-1| > e_clip), the same mean; 7..11 per head;
 *       12 explained variance 1 - Var(ret - v) / Var(ret) over all N tokens, padding included (NaN if Var(ret) = 0;
 *          over the valid tokens only under dc_ppo_loss_fwd_bwd_masked);
 *       13..23 zero (dc_ppo_loss_fwd_bwd_joint: 13, 14 see there; dc_ppo_loss_fwd_bwd_kl: 16..22 see there).
 * Value normalisation (PopArt; this entry point, _masked and _joint): when hparams[DC_HP_VALUE_NORM_STD] = sigma > 0, the
 *   value head's output `value` is in normalised units and the raw targets are read as r_n = fp32((r - mu) / sigma) and,
 *   for the clipped value loss, v_old,n = fp32((v_old - mu) / sigma), both computed in float64 with
 *   mu = hparams[DC_HP_VALUE_NORM_MEAN].  The value loss, dvalue and the explained-variance sums use them in place of r and
 *   v_old.  Slot 7 = 0 runs the plain arithmetic; (mu, sigma) = (0, 1) gives the same bits, as x - 0 and x / 1 are exact.
 */
#define DC_PPO_STATS_SLOTS 24
#define DC_STAT_APPROX_KL 0
#define DC_STAT_CLIP_FRACTION 6
#define DC_STAT_EXPLAINED_VAR 12
#define DC_STAT_JOINT_APPROX_KL 13
#define DC_STAT_JOINT_CLIP_FRACTION 14
#define DC_STAT_KL 16           /* dc_ppo_loss_fwd_bwd_kl: exact KL; 17..21 per head                  */
#define DC_STAT_KL_PENALTY 22   /* dc_ppo_loss_fwd_bwd_kl: beta * KL, the term added to the loss      */
int dc_ppo_loss_fwd_bwd_dev(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                            const uint8_t *const masks[DC_NUM_HEADS],
                            const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                            const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                            const float *old_value, int64_t N, const double *hparams,
                            float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                            float *dvalue, int64_t ld_dvalue, float *out, float *stats, int32_t *n_actions,
                            void *workspace, dc_stream_t stream);

/* Same as dc_ppo_loss_fwd_bwd_dev, plus a per-token mask (no counterpart in the reference, which trains on its zero
 * padding: optimizer.py:587-589,660 average over all tokens and :417-421 bootstrap after the padded length):
 *   valid [N] bytes (0/1) or NULL.  A token with valid = 0 contributes to nothing and gets exactly zero dlogits rows
 *       and dvalue.  With N_v the number of valid tokens: n_actions counts valid rows only (and so drives the
 *       has-gradient flags); out[14] / out[15] are the mean and unbiased std over the valid tokens; policy and entropy
 *       are per-head means over valid action rows; the value loss is 0.5*vf_coef*sum_valid(...)/N_v (clipped or not) and
 *       dvalue = vf_coef*g/N_v; the KL / clip-fraction statistics use valid action rows and the explained variance the
 *       valid tokens.  So the result over N tokens is the unmasked result over the valid tokens alone.
 *   valid NULL or all 1: bit-identical to dc_ppo_loss_fwd_bwd_dev (N_v = N, same summation order).
 *   N_v = 0 or 1: the advantage std is NaN, as torch.std gives, and so is the loss when a head has an action row.
 * Algorithmic bytes: 1 more per token read by each of the two passes.
 */
int dc_ppo_loss_fwd_bwd_masked(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                               const uint8_t *const masks[DC_NUM_HEADS],
                               const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                               const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                               const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                               float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                               float *dvalue, int64_t ld_dvalue, float *out, float *stats, int32_t *n_actions,
                               void *workspace, dc_stream_t stream);

/* Same arguments as dc_ppo_loss_fwd_bwd_masked (valid may be NULL), with the PPO ratio of the whole hierarchical action
 * instead of one ratio per head (no counterpart in the reference, optimizer.py:621-650).  Per token t that counts, S_t is
 * the set of heads with an action row at t and T_a the number of counting tokens with S_t not empty:
 *   log r_t = sum over h in S_t, in head order, of (logp_new[t,h,a_h] - old_logp[t,h])   (fp32; old_logp of a head not
 *             in S_t is ignored)
 *   policy  = -(1/T_a) sum_t min(r_t A_t, clamp(r_t, 1-eps, 1+eps) A_t)                  (0 when T_a = 0)
 * A_t is normalised as by dc_ppo_loss_fwd_bwd_masked.  d loss / d logp_new[t,h,a_h] is the same for every h in S_t,
 * -(1/T_a) A_t (g1 + g2 [r_t in range]) r_t with the autograd rules of torch.min and clamp, and reaches the logits
 * through each head's masked log-softmax.  The entropy term, the value loss (clipped or not), n_actions, the skipping of a
 * head without action rows and the empty-mask rows are as in dc_ppo_loss_fwd_bwd_masked.
 *   out: 1 is the joint policy loss (not divided by 5), and 0 also adds it; 9..13 (policy per head) are 0.
 *   stats: 0..12 as dc_ppo_loss_fwd_bwd_dev (per-head KL / clip fraction of the per-head ratios); 13 the k3 KL and 14 the
 *          clip fraction of the joint ratio, averaged over the T_a tokens (0 when T_a = 0); 15..23 zero.
 * Algorithmic bytes: as dc_ppo_loss_fwd_bwd_masked; the statistics pass also counts T_a.
 */
int dc_ppo_loss_fwd_bwd_joint(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                              const uint8_t *const masks[DC_NUM_HEADS],
                              const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                              const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                              const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                              float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                              float *dvalue, int64_t ld_dvalue, float *out, float *stats, int32_t *n_actions,
                              void *workspace, dc_stream_t stream);

/* ---- KL control: a penalty on the exact KL to the prep-time policy, and an early stop at a KL limit ----------------------
 * No counterpart in the reference.  For a token t that counts (valid, or every token), S_t is the set of heads with an
 * action row at t and T_a the number of counting tokens with S_t not empty.  p_old is the masked softmax of experience
 * prep and p the current one, both over the legal entries of the head's mask, in the reference's form:
 *   KL_t = sum over h in S_t, a legal, of p_old(a) (log p_old(a) - log p(a)),    KL = (1 / T_a) sum_t KL_t (0 if T_a = 0)
 *   loss += beta KL,   dlogits[t, h, a] += (beta / T_a)(p(a) - p_old(a)) for a legal (0 elsewhere)
 * with beta = hparams[DC_HP_KL_COEF].  One definition for both ratio modes.
 *
 * dc_selected_logp_rows: dc_selected_logp's [N,5] output, bit for bit, plus logp_rows [N, DC_KL_ROW_FLOATS] fp32, every
 *   head's full masked log-prob row in head order (columns 0-3 enum, 4-12 x, 13-21 y, 22-61 target_unit, 62-64 ability),
 *   0 at illegal entries.  The selected entry of a row equals logp_out bit for bit.
 * dc_ppo_loss_fwd_bwd_kl: the arguments of dc_ppo_loss_fwd_bwd_masked (valid may be NULL), plus
 *   old_log_probs [N, DC_KL_ROW_FLOATS]  the rows dc_selected_logp_rows wrote at prep
 *   joint          0: the per-head ratios of dc_ppo_loss_fwd_bwd_masked; 1: the joint ratio of dc_ppo_loss_fwd_bwd_joint
 *   kl_out [2] fp32 or NULL  this call's (sum_t KL_t, T_a), e.g. the two floats behind the has-grad flags of the flat
 *                  gradient (dc_grad_finish_kl), so that the gradient all-reduce sums them over the ranks
 *   stats: as the entry point of the chosen ratio mode, plus DC_STAT_KL = KL, 17..21 the per-head KL (sum over the head's
 *          action rows of its row's KL, over their count; 0 for a head without any), DC_STAT_KL_PENALTY = beta KL.
 *   With beta = 0 the loss, dlogits, dvalue and the other stats are those of _masked / _joint bit for bit.
 * Algorithmic bytes: those of the ratio mode's entry point + 260 per token (the old rows).  Checked before any CUDA call:
 * the arguments of _masked, a non-null hparams and old_log_probs -> DC_EINVAL.
 */
#define DC_KL_ROW_FLOATS 65
int dc_selected_logp_rows(const float *const logits[DC_NUM_HEADS], const uint8_t *const masks[DC_NUM_HEADS],
                          const uint8_t *const actions[DC_NUM_HEADS], int64_t N, float *logp_out, float *logp_rows,
                          dc_stream_t stream);
int dc_ppo_loss_fwd_bwd_kl(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                           const uint8_t *const masks[DC_NUM_HEADS], const uint8_t *const actions[DC_NUM_HEADS],
                           const float *old_logp, const float *old_log_probs, const float *adv_raw, const float *ret,
                           const float *value, int64_t ld_value, const float *old_value, const uint8_t *valid, int64_t N,
                           const double *hparams, int joint, float *const dlogits[DC_NUM_HEADS],
                           const int64_t ld_dlogits[DC_NUM_HEADS], float *dvalue, int64_t ld_dvalue, float *out,
                           float *stats, float *kl_out, int32_t *n_actions, void *workspace, dc_stream_t stream);

/* ---- kickstarting: a KL term to a frozen teacher policy (Schmitt et al. 2018) -----------------------------------------
 * No counterpart in the reference.  With S_t and T_a as for KL control (the counting tokens, their heads with an action
 * row, and the number of counting tokens with S_t not empty), p_T the teacher's masked softmax and p the current one,
 * both over the legal entries of the stored mask, in the reference's form:
 *   KL_T = (1 / T_a) sum_t sum_{h in S_t} sum_{a legal} p_T(a) (log p_T(a) - log p(a))      (0 when T_a = 0)
 *   loss += lambda KL_T,   dlogits[t, h, a] += (lambda / T_a)(p(a) - p_T(a)) for h in S_t, a legal
 * with lambda = *teacher_coef.  The same definition as KL control's, with the teacher's rows for the prep-time ones.
 *
 * dc_ppo_loss_fwd_bwd_teacher: the arguments of dc_ppo_loss_fwd_bwd_kl, with old_log_probs and kl_out nullable (NULL:
 *   no KL penalty), plus
 *   teacher_log_probs [N, DC_KL_ROW_FLOATS]  the teacher's rows, as dc_selected_logp_rows writes them
 *   teacher_coef       one fp64 device value, lambda >= 0 (kept off the hparams block, read on every launch)
 *   teacher_stats [DC_TEACHER_STATS_SLOTS] fp32 out: 0 KL_T, 1..5 the per-head KL (sum over the head's action rows of its
 *                      row's KL to the teacher, over their count; 0 for a head without any), 6 lambda KL_T
 *   The loss adds lambda KL_T into out[0] (after beta KL when old_log_probs is given).  With lambda = 0 the loss, dlogits,
 *   dvalue, stats and kl_out are those of _kl (old_log_probs given) or _masked / _joint (NULL) bit for bit; teacher_stats
 *   still reports the KL.
 * Algorithmic bytes: those of the entry point it extends + 260 per token (the teacher's rows).  Checked before any CUDA
 * call: the arguments of _kl and non-null teacher_log_probs, teacher_coef and teacher_stats -> DC_EINVAL.
 */
#define DC_TEACHER_STATS_SLOTS 7
int dc_ppo_loss_fwd_bwd_teacher(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                const uint8_t *const masks[DC_NUM_HEADS], const uint8_t *const actions[DC_NUM_HEADS],
                                const float *old_logp, const float *old_log_probs, const float *teacher_log_probs,
                                const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                                const double *teacher_coef, int joint, float *const dlogits[DC_NUM_HEADS],
                                const int64_t ld_dlogits[DC_NUM_HEADS], float *dvalue, int64_t ld_dvalue, float *out,
                                float *stats, float *kl_out, float *teacher_stats, int32_t *n_actions, void *workspace,
                                dc_stream_t stream);

/* ---- behaviour cloning: the log-likelihood of a demonstrator's actions (supervised pretraining) ---------------------
 * No counterpart in the reference.  With S_t and T_a as for KL control (the counting tokens, their heads with an action
 * row, and the number of counting tokens with S_t not empty), a_{t,h} the action of row (t, h) and p the masked softmax
 * over the legal entries of the stored mask:
 *   NLL = (1 / T_a) sum_t sum_{h in S_t} -log p(a_{t,h})                                      (0 when T_a = 0)
 *   loss = NLL + the entropy term + the value term of dc_ppo_loss_fwd_bwd_masked (clipped or not, value normalisation)
 *   dlogits[t, h, j] = (1 / T_a)(p(j) - [j == a_{t,h}]) + the entropy gradient, for h in S_t and j legal
 * There is no surrogate: old_logp is not an argument and the advantages are read only by the statistics pass, for
 * out[14] / out[15].
 *
 * dc_ppo_loss_fwd_bwd_bc: the arguments of dc_ppo_loss_fwd_bwd_masked without old_logp (valid may be NULL), plus
 *   bc_stats [DC_BC_STATS_SLOTS] fp32 out: 0 NLL, 1..5 the per-head NLL (sum over the head's action rows of -log p(a), over
 *            their count; 0 for a head without any), 6 the token accuracy (the share of the T_a tokens where every head of
 *            S_t has its action as the arg-max of its masked logits, the lowest index on ties), 7..11 the per-head
 *            accuracy (over the head's action rows).
 *   out: 1 is the NLL and 0 adds it; 9..13 are each head's share of the NLL (sum over its rows / T_a).
 *   stats: the approximate KL and clip-fraction slots are 0; the explained variance is that of _masked.
 * Algorithmic bytes: those of dc_ppo_loss_fwd_bwd_masked less the 20 per token of old_logp and the 4 of the advantage in
 * the loss pass.  Checked before any CUDA call: the arguments of _masked, non-null hparams and bc_stats -> DC_EINVAL.
 */
#define DC_BC_STATS_SLOTS 12
int dc_ppo_loss_fwd_bwd_bc(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                           const uint8_t *const masks[DC_NUM_HEADS], const uint8_t *const actions[DC_NUM_HEADS],
                           const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                           const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                           float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS], float *dvalue,
                           int64_t ld_dvalue, float *out, float *stats, float *bc_stats, int32_t *n_actions,
                           void *workspace, dc_stream_t stream);

/* ---- dual-clip PPO: a floor under the surrogate of negative-advantage rows (Ye et al. 2020) -------------------------
 * No counterpart in the reference.  With A_t the token's normalised advantage (as every loss entry point normalises it),
 * r the ratio (per head, or the joint ratio of the token) and s = min(r A_t, clip(r, 1 - eps, 1 + eps) A_t) the clipped
 * surrogate, each row's term becomes
 *   term = s                  if A_t >= 0
 *   term = max(s, c A_t)      if A_t <  0,        c = *dual_clip > 1
 * so the term of a row with A_t < 0 stays bounded as r grows.  The gradient is the autograd of
 * torch.where(A < 0, torch.maximum(s, c A), s): a row where the cap binds (s < c A, that is r > c) gets no surrogate
 * gradient, a tie splits it in half.  Per-head and joint means, the entropy and value terms, the KL penalty and the teacher
 * term are those of dc_ppo_loss_fwd_bwd_teacher.
 *
 * dc_ppo_loss_fwd_bwd_dual_clip: the arguments of dc_ppo_loss_fwd_bwd_teacher, with old_log_probs and kl_out nullable (NULL:
 *   no KL penalty) and teacher_log_probs, teacher_coef and teacher_stats nullable together (NULL: no teacher term), plus
 *   dual_clip          one fp64 device value, c > 1 (kept off the hparams block, read on every launch)
 *   dual_clip_stats [DC_DUAL_CLIP_STATS_SLOTS] fp32 out: 1..5 per head the share of its action rows where the cap binds
 *                      (0 for a head without any, and under the joint ratio), 0 their mean over the heads with action
 *                      rows, 6 the share of the T_a tokens where the joint ratio's cap binds (0 with per-head ratios).
 *   With a c no ratio reaches, the loss, dlogits, dvalue, stats, kl_out and teacher_stats are those of the entry point the
 *   call would otherwise be (_masked / _dev, _joint, _kl or _teacher) bit for bit.
 * Algorithmic bytes: those of the entry point it extends; the cap adds no traffic.  Checked before any CUDA call: the
 * arguments of _masked, non-null hparams, dual_clip and dual_clip_stats, and the teacher's three pointers all given or all
 * NULL -> DC_EINVAL.
 */
#define DC_DUAL_CLIP_STATS_SLOTS 7
int dc_ppo_loss_fwd_bwd_dual_clip(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                  const uint8_t *const masks[DC_NUM_HEADS], const uint8_t *const actions[DC_NUM_HEADS],
                                  const float *old_logp, const float *old_log_probs, const float *teacher_log_probs,
                                  const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                  const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                                  const double *teacher_coef, const double *dual_clip, int joint,
                                  float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                                  float *dvalue, int64_t ld_dvalue, float *out, float *stats, float *kl_out,
                                  float *teacher_stats, float *dual_clip_stats, int32_t *n_actions, void *workspace,
                                  dc_stream_t stream);

/* ---- value normalisation (PopArt, van Hasselt et al. 2016) --------------------------------------------------------
 * No counterpart in the reference, whose critic learns raw returns (optimizer.py:660).
 *   dc_value_norm_stats    out[3] fp64 (device) = count, sum x, sum x^2 over the x[i] [N] with valid[i] != 0 (valid NULL:
 *                          all N), in float64.  Deterministic: one CTA, a fixed-order two-stage reduction without
 *                          atomics, so two calls give the same bits.  N = 0 writes zeros.
 *   dc_value_denorm        out[i] = fp32(mu + sigma * v[i * ld_v]) for i < N, computed in float64 (out contiguous [N]):
 *                          the raw-scale values of a normalised head, e.g. from the value column (pitch 128) of the packed
 *                          head GEMM.  sigma > 0.
 *   dc_value_head_rescale  in place on the value head's weight w [n] and bias b [1] (fp32), computed in float64 and rounded
 *                          once: w = w sigma_old / sigma_new, b = (sigma_old b + mu_old - mu_new) / sigma_new, so that
 *                          sigma v + mu is unchanged when the statistics move from (mu_old, sigma_old) to (mu_new,
 *                          sigma_new).  Both sigmas > 0.
 * Checked before any CUDA call: N >= 0 / n >= 1, ld_v >= 1, non-null pointers where there is work, finite statistics with
 * positive sigmas -> DC_EINVAL.
 */
int dc_value_norm_stats(const float *x, const uint8_t *valid, int64_t N, double *out, dc_stream_t stream);
int dc_value_denorm(const float *v, int64_t ld_v, int64_t N, double mu, double sigma, float *out, dc_stream_t stream);
int dc_value_head_rescale(float *w, int64_t n, float *b, double mu_old, double sigma_old, double mu_new, double sigma_new,
                          dc_stream_t stream);

/* Log-prob of the taken action per head, [N,5] dense (0 where the head took no action):
 * the no-grad half of experiences_from_rollout (optimizer.py:387-390). */
int dc_selected_logp(const float *const logits[DC_NUM_HEADS],
                     const uint8_t *const masks[DC_NUM_HEADS],
                     const uint8_t *const actions[DC_NUM_HEADS], int64_t N, float *logp_out,
                     dc_stream_t stream);

/* ---- gradient finish: count-divide, grad-norm metrics, clip, Adam ------------------------
 * Replaces distributed.py:57 (grad /= has_grad_count), optimizer.py:674-681 (mean_gradient_norm
 * x2, clip_grad_norm_(0.5), NaN guard, Adam.step) on ONE flat fp32 buffer holding all params.
 *   flat_grad  [total + n_seg]  gradients, followed by n_seg has-grad counts (after the
 *                               all-reduce: number of ranks that had a gradient, distributed.py:36-37)
 *   seg_lo/hi  [n_seg] int64    parameter p covers flat elements seg_lo[p] .. seg_hi[p]-1 (tensors may be padded apart)
 *   seg_head   [n_seg]   int32  -1 = always has a gradient; h>=0 = has one only if head h took
 *                               an action this batch (optimizer.py:627-630: skipped heads leave
 *                               .grad = None, so Adam and the norm mean skip those tensors)
 *   steps      [n_seg]   int32  per-parameter Adam step counters (in/out)
 *   loss_out   the `out` vector of dc_ppo_loss_fwd_bwd (NaN guard, optimizer.py:667,678)
 *   metrics [4] fp32 out: 0 mean grad norm unclipped, 1 clipped, 2 total norm, 3 nan flag (1 =
 *                               NaN seen, parameters left untouched -- the caller raises ValueError)
 * dc_grad_flags writes the local has-grad flags (1/0) into flat_grad[total ..] before the all-reduce.
 */
int dc_grad_flags(float *flat_grad, int64_t total, const int32_t *seg_head, int n_seg,
                  const int32_t *n_actions, dc_stream_t stream);
int dc_grad_finish(float *flat_param, float *flat_grad, float *exp_avg, float *exp_avg_sq,
                   int32_t *steps, const int64_t *seg_lo, const int64_t *seg_hi, const int32_t *seg_head, int n_seg,
                   int64_t total, double lr, double beta1, double beta2, double adam_eps,
                   double max_norm, const float *loss_out, float *metrics, void *workspace,
                   dc_stream_t stream);
/* Same, with lr and max_norm read from hparams[DC_HP_LR] / hparams[DC_HP_MAX_GRAD_NORM] (device, see above). */
int dc_grad_finish_dev(float *flat_param, float *flat_grad, float *exp_avg, float *exp_avg_sq,
                       int32_t *steps, const int64_t *seg_lo, const int64_t *seg_hi, const int32_t *seg_head, int n_seg,
                       int64_t total, const double *hparams, double beta1, double beta2, double adam_eps,
                       const float *loss_out, float *metrics, void *workspace, dc_stream_t stream);
#define DC_FINISH_WORKSPACE_BYTES 1024
/* dc_grad_finish_dev with the KL early stop.  flat_grad holds two more floats after the n_seg flags: the all-reduced
 * (sum_t KL_t, T_a) that dc_ppo_loss_fwd_bwd_kl wrote (kl_out) on every rank.  KL = sum / T_a (0 when T_a = 0).  When
 * hparams[DC_HP_KL_STOP] > 0 and KL exceeds it, the step is skipped: parameters, moments and step counters are left
 * untouched, as on the NaN path, but it is not an error.  Every rank reads the same all-reduced numbers, so every rank
 * makes the same decision.  metrics [DC_FINISH_KL_METRICS]: 0..3 as dc_grad_finish, 4 KL, 5 skipped (1) or not (0). */
#define DC_FINISH_KL_METRICS 6
int dc_grad_finish_kl(float *flat_param, float *flat_grad, float *exp_avg, float *exp_avg_sq,
                      int32_t *steps, const int64_t *seg_lo, const int64_t *seg_hi, const int32_t *seg_head, int n_seg,
                      int64_t total, const double *hparams, double beta1, double beta2, double adam_eps,
                      const float *loss_out, float *metrics, void *workspace, dc_stream_t stream);

/* ---- actor side: hierarchical action selection for a batch of A agents in one launch ----------------
 * (policy.py:23-33 MaskedCategorical, :169-178 masked_softmax, :190-216 sample_action/select_actions; caller agent.py:578-674)
 * Heads in DC order (enum 4, x 9, y 9, target_unit 40, ability 3).  logits[h]: A rows with pitch ld[h] floats;
 * masks[h]: [A, n_h] bytes (0/1); u: [A,5] uniforms in [0,1) supplied by the caller (torch.multinomial's RNG stream cannot
 * be reproduced, so the contract is the index function: inverse CDF over the masked probabilities, fp32, sequential
 * in index order -- oracle/ref_policy.py:sample_index, up to fp32 rounding near a cumulative boundary).  chosen[A,5]:
 * enum first, then x,y (enum 1) / target_unit (2) / ability (3); -1 for heads that were not sampled.  logp[A,5] (nullable): log-probability of each chosen entry. */
int dc_select_actions(const float *const logits[DC_NUM_HEADS], const int64_t ld[DC_NUM_HEADS],
                      const uint8_t *const masks[DC_NUM_HEADS], const float *u, int64_t A, int32_t *chosen,
                      float *logp, dc_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DOTACLIENT_B200_H */
