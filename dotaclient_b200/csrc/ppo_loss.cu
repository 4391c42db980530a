// Fused PPO loss + gradient over the five action heads and the value head.
//
// Replaces, for one stacked batch of N tokens (optimizer.py line numbers, TimZaman/dotaclient):
//   :587-589  advantage normalisation (mean, unbiased std, +eps) over ALL tokens incl. padding
//   :621-646  per head: actions_step, masked log-softmax (policy.py:169-178: no max-subtraction,
//             normalised over the mask), selected log-prob, ratio, clipped surrogate, entropy
//   :649-665  policy loss = mean over the 5 heads (skipped heads count as 0), entropy loss,
//             value loss over ALL tokens, total
//   :672      loss.backward() down to d loss / d logits and d loss / d value
//
// Two launches.  (1) ppo_stats_kernel: per-head action-row counts and sum / sum-of-squares of
// the raw advantage (float64) -- the counts are needed as divisors by every gradient -- and the first counting token.
// (2) ppo_loss_kernel: one thread per token; a 128-token tile of every head's logits / masks /
// actions is staged through shared memory with coalesced 16-byte loads (rows are 12..160 bytes,
// so per-thread row reads from global would waste most of every sector), the tile is overwritten
// in place with d loss / d logits and written back with coalesced 16-byte stores.
//
// The second launch also accumulates the PPO diagnostics (approximate KL and clip fraction per head, explained variance)
// from the values it already holds in registers, and optionally clips the value loss PPO2-style against old values.
// The `_dev` entry point reads its hyper-parameters from a device block (DC_HPARAM_SLOTS), so a captured CUDA graph of
// the step picks up new values on every replay; the scalar-argument entry points run the same kernel body.
//
// The `_masked` entry point takes a per-token `valid` byte: a token with valid = 0 (the zero padding of a rollout's last
// chunk) is left out of every count, sum and divisor -- advantage mean / std, action counts, policy / entropy means, the
// value loss and its 1/N, the diagnostics -- and receives exactly zero gradient.  The statistics pass counts the valid
// tokens into the workspace (n_valid); with valid == NULL every token counts and the arithmetic is the unmasked one.
//
// The `_joint` entry point (kJoint) clips the ratio of the whole hierarchical action instead of each head's:
// log r_t = sum over the heads with an action row at t of (logp_new - old_logp), one clipped surrogate per token, averaged
// over the T_a counting tokens with at least one action row (counted by the statistics pass).  One thread makes two sweeps
// over its token's heads in the shared-memory tile: (1) log-sum-exp, selected log-prob, entropy, per-head diagnostics and
// the joint log-ratio; (2) every head's dlogits row from the joint ratio's gradient.  Entropy and value terms are per head,
// as in the default objective.
//
// Value normalisation (PopArt): when hparams[DC_HP_VALUE_NORM_STD] = sigma > 0 the value head's output is in normalised
// units, and every raw value target r (and, for the clipped value loss, every raw old value) is read as
// fp32((r - mu) / sigma), computed in float64.  The value loss, dvalue and the explained-variance sums then run in
// normalised units.  No extra bytes; slot 7 = 0 runs the plain arithmetic.
//
// Algorithmic HBM bytes per token: logits 260 + masks 65 + actions 65 + old 20 + adv/ret/value 12
// read, dlogits 260 + dvalue 4 written = 686 (+ 69 for the statistics pass, + 4 for the old value when the value loss
// is clipped, + 1 in each pass for `valid` when given).  The joint ratio reads and writes the same bytes.
//
// KL control (`dc_ppo_loss_fwd_bwd_kl`, kKl): the loss also reads every head's full masked log-prob row of the prep-time
// policy ([N, 65], written by `dc_selected_logp_rows`, 0 at illegal entries) and adds beta * KL, with
//   KL = (1 / T_a) sum_t sum_{h in S_t} sum_{a legal} p_old(a) (log p_old(a) - log p(a)),
// and its gradient (beta / T_a)(p(a) - p_old(a)) to the legal entries of every dlogits row in S_t.  Both come out of the
// loop that already writes that row from p and log p, so the only new work is one exp per legal entry.  beta = 0 skips
// the gradient term and the loss term, so the results are those of the instantiation without kKl, bit for bit.  The
// statistics pass counts T_a (as for the joint ratio), and the last CTA writes (sum_t KL_t, T_a) to `kl_out`.
// The old rows are staged through shared memory as one contiguous [128, 65] tile (33,280 bytes, 16-byte loads; a pitch
// of 65 floats keeps per-thread row reads conflict-free).  Read per thread from global instead, a warp's 32 rows would
// sit 260 bytes apart, every load instruction would touch 32 sectors and the whole tile would have to stay in L1 across
// the five heads.  Staging takes the CTA from 53.5 KB to 86 KB of dynamic shared memory: ptxas gives the loss kernel
// about 160 registers, which already limits it to 3 CTAs per SM, and 86 KB + the static rows still allow 2.  The extra
// HBM traffic is 260 B / token read (686 + 260 = 946 B / token for the loss pass).
//
// Kickstarting (`dc_ppo_loss_fwd_bwd_teacher`, kTeacher, with or without kKl): the loss also reads a frozen teacher's
// rows ([N, 65], as dc_selected_logp_rows writes them) and adds lambda * KL_T with
//   KL_T = (1 / T_a) sum_t sum_{h in S_t} sum_{a legal} p_T(a) (log p_T(a) - log p(a)),
// and (lambda / T_a)(p(a) - p_T(a)) to the legal entries of every dlogits row in S_t, in the same loop as the KL term:
// one more exp per legal entry.  lambda = *teacher_coef (a device double next to the hparams block, not a slot of it);
// lambda = 0 skips both terms, so the results are those of the instantiation without kTeacher, bit for bit.  The teacher
// rows are staged like the old rows, one more [128, 65] tile (33,280 bytes) after them.  ptxas (sm_90a, no spills, with
// __launch_bounds__(128, 2)): teacher alone 214 registers per-head / 196 joint, 86.8 KB dynamic + 8.9 / 9.9 KB static
// shared memory, 2 CTAs per SM like the KL tile; teacher and KL 194 / 197 registers, 120 KB dynamic + 11.5 / 12.5 KB
// static, 1 CTA per SM.  Both are staged, for the reason the old rows are: read per thread from global, a warp's rows sit
// 260 bytes apart and are touched in five head slices.  Measured on an H100 80GB HBM3 (700 W) at 131,072 tokens with a
// valid mask (tools/teacher_bench.py, medians of 200 calls): _masked 206 us, _kl 320 us, teacher alone 295 us, teacher and
// KL 441 us, so the 1-CTA combined instantiation costs 121 us more than _kl, about 1 % of the C2 step.  Algorithmic bytes:
// + 260 / token read for the teacher's rows (946 B / token with one row set, 1,206 B with both, + valid and old value).
//
// Behaviour cloning (`dc_ppo_loss_fwd_bwd_bc`, kBc, per-head path): every rollout is a demonstration and the surrogate is
// replaced by the negative log-likelihood of its actions,
//   NLL = (1 / T_a) sum_t sum_{h in S_t} -lp[a],   and (1 / T_a)(p(j) - [j == a]) on the legal entries of every row in S_t,
// in the loop that already writes the row: no extra row reads and no extra exp (KL(onehot(a) || p) is -log p(a), so this is
// the kTeacher gradient with the teacher's row replaced by the action).  A row of S_t also stages its -lp[a] and whether the
// arg-max of its masked logits (the lowest index on ties) is a; the token stages whether every row of S_t is right.  Those
// 11 staging rows are summed in float64 after the others, in the same fixed order, into bc_stats.  The loss pass reads no
// old_logp and no advantage (the statistics pass still sums the advantages for out[14] / out[15]) and computes no
// approximate KL or clip fraction (their slots stay 0); the entropy and value terms and the explained variance are the
// per-head path's.  ptxas (sm_90a, __launch_bounds__(128, 2)): 255 registers, no spills, 0 bytes stack frame, 53.5 KB dynamic
// + 12.0 KB static shared memory, 2 CTAs per SM (at 3 CTAs per SM, ptxas's 168 registers spill 32 bytes).  Algorithmic
// bytes: 686 - 24 = 662 per token for the loss pass (+ 1 valid, + 4 old value).
//
// Dual clip (`dc_ppo_loss_fwd_bwd_dual_clip`, kDual, either ratio mode, with or without kKl and kTeacher; Ye et al. 2020):
// for a row with a negative normalised advantage A the clipped surrogate s = min(r A, clip(r) A) is floored at c A,
//   term = max(s, c A) if A < 0, s otherwise,   c = *dual_clip > 1 (a device double next to the hparams block),
// in head_token for each head's ratio and in the joint-ratio block for the token's.  The gradient is torch.where /
// torch.maximum's: d term / d s = 1 above the floor, 1/2 on a tie, 0 below it, so a row where the floor binds (s < c A,
// i.e. r > c) gets no surrogate gradient and keeps its entropy, KL and teacher terms.  With g_s = 1 the arithmetic is the
// instantiation without kDual's (x * 1 is exact), so a c no ratio reaches gives its results bit for bit.  A bound row stages
// a 1 in one more row per head (per-head ratios) or one row (joint), summed in float64 after the other staging rows, in the
// same fixed order, into dual_clip_stats.  No extra bytes.  ptxas (sm_90a, __launch_bounds__(128, 2) for kDual, no spills, no
// stack frame), registers and static shared memory per head / joint:
//   alone           207 / 196 registers,  53.5 KB dynamic +  8.9 /  7.8 KB static, 2 CTAs per SM
//   with kKl        193 / 197 registers,  86.8 KB dynamic + 11.5 / 10.4 KB static, 2 CTAs per SM
//   with kTeacher   193 / 197 registers,  86.8 KB dynamic + 11.5 / 10.4 KB static, 2 CTAs per SM
//   with both       195 / 198 registers, 120.1 KB dynamic + 14.1 / 13.0 KB static, 1 CTA per SM
// The per-head instantiation alone runs at 2 CTAs per SM where _masked runs at 3 (ptxas's default 168 registers, with a
// 48-byte spill): at 3 CTAs per SM the kDual code would spill too.
#include "dc_common.cuh"

namespace {

constexpr int kHeads = DC_NUM_HEADS;
constexpr int kTile = 128;  // tokens per CTA == threads per CTA
__host__ __device__ constexpr int head_n(int h) { return h == 0 ? 4 : h == 1 ? 9 : h == 2 ? 9 : h == 3 ? 40 : 3; }
// odd row pitch in shared memory -> conflict-free per-thread row access
__host__ __device__ constexpr int head_pitch(int h) { return h == 0 ? 5 : h == 1 ? 9 : h == 2 ? 9 : h == 3 ? 41 : 3; }
__host__ __device__ constexpr int logit_off(int h) {  // float offset of head h's tile in smem
    int o = 0;
    for (int i = 0; i < h; ++i) o += head_pitch(i) * kTile;
    return o;
}
__host__ __device__ constexpr int byte_off(int h) {
    int o = 0;
    for (int i = 0; i < h; ++i) o += head_n(i) * kTile;
    return o;
}
constexpr int kLogitFloats = logit_off(kHeads);      // 67 * 128
constexpr int kOldFloats = 5 * kTile;
constexpr int kByteTile = byte_off(kHeads);          // 65 * 128
constexpr size_t kSmemBytes = (size_t)(kLogitFloats + kOldFloats) * 4 + 2 * (size_t)kByteTile;
// KL control: the prep-time log-prob rows, [N, 65] in head order, staged contiguously after the byte tiles
constexpr int kRowFloats = DC_KL_ROW_FLOATS;
__host__ __device__ constexpr int row_col(int h) { return byte_off(h) / kTile; }   // first column of head h in a row
static_assert(kRowFloats == byte_off(kHeads) / kTile, "a log-prob row holds every head's entries");
static_assert(kSmemBytes % 16 == 0, "the old-row tile is 16-byte aligned");
constexpr size_t kSmemBytesKl = kSmemBytes + (size_t)kTile * kRowFloats * 4;
// the teacher's rows: one more tile of the same layout, after the old rows when both are staged (teacher alone: kSmemBytesKl)
constexpr size_t kSmemBytesKlTeacher = kSmemBytesKl + (size_t)kTile * kRowFloats * 4;
static_assert(DC_TEACHER_STATS_SLOTS >= 2 + DC_NUM_HEADS, "teacher_stats too small");

struct HeadPtrs {
    const float *logits[kHeads];
    const uint8_t *masks[kHeads];
    const uint8_t *actions[kHeads];
    float *dlogits[kHeads];
    long long ld_l[kHeads];     // row pitch (floats) of logits[h]; == n_h when contiguous.  A pitch of 128 lets the four
    long long ld_d[kHeads];     // small heads + value live as column ranges of ONE packed [N,128] GEMM output / gradient
    long long ld_v, ld_dv;      // pitches of value / dvalue
};

// PPO diagnostics accumulated per token: k3 KL and clipped rows per head, then sums of (ret - v), (ret - v)^2, ret, ret^2
constexpr int kStats = 2 * kHeads + 4;
constexpr int kStKl = 0, kStClip = kHeads, kStD = 2 * kHeads, kStD2 = kStD + 1, kStR = kStD + 2, kStR2 = kStD + 3;
constexpr int kTokD = 2 * kHeads, kTokR = kTokD + 1, kTokRows = kTokR + 1;   // rows of the per-token staging
// joint ratio only: two more staging rows and sums after the above (k3 KL and clip flag of the joint ratio)
constexpr int kTokJoint = kTokRows, kJointStats = 2;
// KL control only: one staging row and sum per head of the exact KL of that head's row (after the joint rows, if any)
constexpr int kKlStats = kHeads;
// teacher only: the same per head for the KL to the teacher's row (after the KL control rows, if any)
constexpr int kTeachStats = kHeads;
// behaviour cloning only: per head the NLL of its action row, the token's all-heads-right flag, per head the arg-max flag
// (the order of bc_stats)
constexpr int kBcStats = 2 * kHeads + 1;
// dual clip only: per head (per-head ratios) or once (the joint ratio) the flag of a row whose cap binds, after the above
constexpr int kDualStats = kHeads;
static_assert(DC_DUAL_CLIP_STATS_SLOTS == 2 + kHeads, "dual_clip_stats: the mean, per head, the joint ratio's");
static_assert(DC_BC_STATS_SLOTS == 2 + 2 * kHeads, "bc_stats: the NLL, per head, the token accuracy, per head");
static_assert(2 * kHeads + 3 < DC_PPO_STATS_SLOTS, "stats output too small");
static_assert(DC_STAT_KL_PENALTY < DC_PPO_STATS_SLOTS, "stats output too small");

// Workspace layout (DC_PPO_WORKSPACE_BYTES, zeroed per call)
struct Workspace {
    double pol[kHeads];   // sum over action rows of min(surr1, surr2); joint ratio: pol[0] sums over the T_a tokens
    double ent[kHeads];   // sum over masked entries of -p*logp
    double vl;            // sum (ret - v)^2, or of the clipped value loss term
    double adv_sum, adv_sq;
    double st[kStats];    // diagnostics (kSt* above)
    int cnt[kHeads];
    unsigned long long n_valid;   // tokens that count (all N when no valid mask is given)
    unsigned ticket_stats, ticket_loss;
    float adv_mean, adv_std;
    unsigned long long n_joint;      // joint ratio: T_a, the tokens that count with at least one action row
    double st_joint[kJointStats];    // joint ratio: sums over the T_a tokens of its k3 KL and of its clip flag
    unsigned long long first_rev;    // N - (index of the first token that counts); 0 when no token counts
    double st_kl[kKlStats];          // KL control: per head, the sum over its action rows of the exact KL of the row
    double st_teach[kTeachStats];    // teacher: per head, the sum over its action rows of the KL to the teacher's row
    double st_bc[kBcStats];          // behaviour cloning: the sums of its staging rows (kBcStats above)
    double st_dual[kDualStats];      // dual clip: per head (joint ratio: [0]) the rows whose cap binds
};
static_assert(sizeof(Workspace) <= DC_PPO_WORKSPACE_BYTES, "workspace too small");

// Cooperative copy of `count` rows of N floats (contiguous in global) into smem rows of pitch P.
template <int N, int P>
__device__ __forceinline__ void stage_rows_f32(float *dst, const float *__restrict__ base, long long ld, int64_t t0, int count) {
    const int total = count * N;
    if (ld != N) {                                   // strided rows (column range of a wider matrix)
        for (int idx = threadIdx.x; idx < total; idx += kTile) dst[(idx / N) * P + (idx % N)] = base[(t0 + idx / N) * ld + (idx % N)];
        return;
    }
    const float *src = base + t0 * N;
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const int nvec = total >> 2;
        for (int i = threadIdx.x; i < nvec; i += kTile) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(src) + i);
            const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int idx = i * 4 + q;
                dst[(idx / N) * P + (idx % N)] = e[q];
            }
        }
        for (int idx = (nvec << 2) + threadIdx.x; idx < total; idx += kTile) dst[(idx / N) * P + (idx % N)] = src[idx];
    } else {
        for (int idx = threadIdx.x; idx < total; idx += kTile) dst[(idx / N) * P + (idx % N)] = src[idx];
    }
}

template <int N, int P>
__device__ __forceinline__ void unstage_rows_f32(float *__restrict__ base, long long ld, int64_t t0, const float *src, int count) {
    const int total = count * N;
    if (ld != N) {
        for (int idx = threadIdx.x; idx < total; idx += kTile) base[(t0 + idx / N) * ld + (idx % N)] = src[(idx / N) * P + (idx % N)];
        return;
    }
    float *dst = base + t0 * N;
    if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        const int nvec = total >> 2;
        for (int i = threadIdx.x; i < nvec; i += kTile) {
            float e[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int idx = i * 4 + q;
                e[q] = src[(idx / N) * P + (idx % N)];
            }
            reinterpret_cast<float4 *>(dst)[i] = make_float4(e[0], e[1], e[2], e[3]);
        }
        for (int idx = (nvec << 2) + threadIdx.x; idx < total; idx += kTile) dst[idx] = src[(idx / N) * P + (idx % N)];
    } else {
        for (int idx = threadIdx.x; idx < total; idx += kTile) dst[idx] = src[(idx / N) * P + (idx % N)];
    }
}

__device__ __forceinline__ void stage_bytes(uint8_t *dst, const uint8_t *__restrict__ src, int total) {
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const int nvec = total >> 4;
        for (int i = threadIdx.x; i < nvec; i += kTile)
            reinterpret_cast<uint4 *>(dst)[i] = __ldg(reinterpret_cast<const uint4 *>(src) + i);
        for (int idx = (nvec << 4) + threadIdx.x; idx < total; idx += kTile) dst[idx] = src[idx];
    } else {
        for (int idx = threadIdx.x; idx < total; idx += kTile) dst[idx] = src[idx];
    }
}

// (x - mu) / sigma in float64, rounded once to fp32: a raw value target in the units of a normalised value head
__device__ __forceinline__ float vn_normalise(float x, double mu, double sigma) {
    return (float)__ddiv_rn(__dsub_rn((double)x, mu), sigma);
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T *scratch) {
    v = dc_warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
    __syncthreads();
    T r = 0;
    for (int w = 0; w < kTile / 32; ++w) r += scratch[w];
    return r;
}

// ---- pass 1: counts + advantage statistics ------------------------------------------------
// kJoint (the joint ratio, and KL control): also counts T_a (tokens that count with an action row in any head) into
// ws->n_joint
template <bool kJoint>
__global__ void __launch_bounds__(kTile) ppo_stats_kernel(HeadPtrs hp, const float *__restrict__ adv,
                                                           const uint8_t *__restrict__ valid, int64_t N,
                                                           Workspace *ws, int32_t *n_actions_out) {
    __shared__ __align__(16) uint8_t s_act[kByteTile];
    __shared__ double s_red[kTile / 32];
    __shared__ bool s_last;
    __shared__ int s_first;
    const int64_t t0 = (int64_t)blockIdx.x * kTile;
    const int count = (int)min((int64_t)kTile, N - t0);
    if (threadIdx.x == 0) s_first = kTile;
#pragma unroll
    for (int h = 0; h < kHeads; ++h) stage_bytes(s_act + byte_off(h), hp.actions[h] + t0 * head_n(h), count * head_n(h));
    __syncthreads();
    // a token that does not count (valid = 0) adds nothing to the sums and the action counts
    const bool live = threadIdx.x < count && (valid == nullptr || valid[t0 + threadIdx.x] != 0);
    if (live) atomicMin(&s_first, (int)threadIdx.x);
    double a = 0.0;
    if (live) a = (double)adv[t0 + threadIdx.x];
    int has[kHeads];
#pragma unroll
    for (int h = 0; h < kHeads; ++h) {
        int any = 0;
        if (live) {
            const uint8_t *row = s_act + byte_off(h) + threadIdx.x * head_n(h);
            for (int j = 0; j < head_n(h); ++j) any |= row[j];
        }
        has[h] = any != 0;
    }
    const double sa = block_sum(a, s_red);
    const double sq = block_sum(a * a, s_red);
    int tot[kHeads];
#pragma unroll
    for (int h = 0; h < kHeads; ++h) tot[h] = __syncthreads_count(has[h]);
    const int n_live = __syncthreads_count(live);
    int n_joint = 0;
    if constexpr (kJoint) n_joint = __syncthreads_count(has[0] | has[1] | has[2] | has[3] | has[4]);
    if (threadIdx.x == 0) {
        atomicAdd(&ws->adv_sum, sa);
        atomicAdd(&ws->adv_sq, sq);
        atomicAdd(&ws->n_valid, (unsigned long long)n_live);
        if (kJoint && n_joint) atomicAdd(&ws->n_joint, (unsigned long long)n_joint);
        if (s_first < kTile) atomicMax(&ws->first_rev, (unsigned long long)(N - (t0 + s_first)));
#pragma unroll
        for (int h = 0; h < kHeads; ++h)
            if (tot[h]) atomicAdd(&ws->cnt[h], tot[h]);
        __threadfence();
        s_last = atomicAdd(&ws->ticket_stats, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last && threadIdx.x == 0) {
        __threadfence();
        // over the tokens that count: N without a valid mask (the same double), N_v with one
        const double n = (double)*((volatile unsigned long long *)&ws->n_valid);
        const double sum = *((volatile double *)&ws->adv_sum), sq2 = *((volatile double *)&ws->adv_sq);
        const double mean = sum / n;
        // torch.std: unbiased (N-1); NaN for N == 1 (and for N_v = 0 or 1) like torch.
        const double var = (sq2 - n * mean * mean) / (n - 1.0);
        ws->adv_mean = (float)mean;
        ws->adv_std = (float)sqrt(var > 0.0 ? var : (var == var ? 0.0 : var));
        for (int h = 0; h < kHeads; ++h) n_actions_out[h] = *((volatile int *)&ws->cnt[h]);
    }
}

// ---- pass 2: loss + gradient --------------------------------------------------------------
// Dual clip of one surrogate s = min(r A, clip(r) A): for A < 0, s <- max(s, c A), with g_s = d max / d s by the autograd
// of torch.maximum (1 above the cap, 1/2 on a tie, 0 below it; NaN stays NaN as torch.maximum keeps it), and *bound = 1
// where the cap binds (s < c A).  A >= 0 leaves s and g_s = 1 alone.
__device__ __forceinline__ void dual_clip_term(float &s, float &g_s, float adv_n, float c, float *bound) {
    if (adv_n < 0.f) {
        const float cap = c * adv_n;
        g_s = s > cap ? 1.f : (s == cap ? 0.5f : 0.f);
        if (s < cap) {
            *bound = 1.f;
            s = cap;
        }
    }
}

// kKl, loss: `orow` is the token's prep-time log-prob row of head H; the exact KL of the row goes to *kl_row_out (when
// the head has an action row here) and, with kl_scale = beta / T_a > 0, its gradient joins the dlogits row.
// kKl, select (logp_out given): the full masked log-prob row overwrites the logits row in the tile, 0 at illegal entries.
// kTeach, loss: `trow` is the teacher's log-prob row of head H, used as kKl uses `orow` (t_scale = lambda / T_a).
// kBc (behaviour cloning, a loss): no surrogate.  A row with an action a (a row of S_t) writes -lp[a] to *nll_out and its
// arg-max flag to *acc_out, sets bit H of *bc_in (and of *bc_miss when the arg-max is not a), and adds
// bc_scale (p - [j == a]) to its legal entries, bc_scale = 1 / T_a.
// kDual (dual clip, a loss): for adv_n < 0 the row's term is max(s, dual_c adv_n), s the clipped surrogate; a row where the
// cap binds (s < dual_c adv_n) writes 1 to *dual_out and gets no surrogate gradient.
template <int H, bool kGrad, bool kKl = false, bool kTeach = false, bool kBc = false, bool kDual = false>
__device__ __forceinline__ void head_token(float *lrow, const uint8_t *mrow, const uint8_t *arow, float old_lp,
                                           float adv_n, int n_h, float e_clip, float entropy_coef, float &pol_acc,
                                           float &ent_acc, float *kl_out, float *clip_out, float *logp_out,
                                           const float *orow = nullptr, float kl_scale = 0.f, float *kl_row_out = nullptr,
                                           const float *trow = nullptr, float t_scale = 0.f, float *t_row_out = nullptr,
                                           float bc_scale = 0.f, float *nll_out = nullptr, float *acc_out = nullptr,
                                           int *bc_in = nullptr, int *bc_miss = nullptr, float dual_c = 0.f,
                                           float *dual_out = nullptr) {
    constexpr int N = head_n(H);
    float l[N], e[N];
    int mask_any = 0, a_idx = -1;
    float se = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        l[j] = lrow[j];
        const int m = mrow[j];
        mask_any |= m;
        e[j] = m ? __expf(l[j]) : 0.f;   // masked_exp[~mask] = 0 (policy.py:172-174)
        se += e[j];
        if (arow[j]) a_idx = j;
    }
    if (logp_out) {  // no-grad selected log-prob (optimizer.py:387-390)
        float lp = 0.f;
        if (a_idx >= 0) {
            float la = l[0];
#pragma unroll
            for (int j = 1; j < N; ++j) la = (j == a_idx) ? l[j] : la;
            lp = la - logf(se);
        }
        *logp_out = lp;
        if (kKl) {   // the same expression as the selected entry, so row[a] == *logp_out bit for bit
#pragma unroll
            for (int j = 0; j < N; ++j) lrow[j] = mrow[j] ? l[j] - logf(se) : 0.f;
        }
        return;
    }
    // A head nobody used this batch is skipped entirely (optimizer.py:627-630); a row with an
    // empty mask and no action contributes exactly zero (its NaN is erased by the index_put backward).
    if (n_h == 0 || (!mask_any && a_idx < 0)) {
        if (kGrad) {
#pragma unroll
            for (int j = 0; j < N; ++j) lrow[j] = 0.f;
        }
        return;
    }
    const float lse = logf(se);          // policy.py:175-177
    const float inv_se = 1.0f / se;
    float ent_row = 0.f;
    float p[N], lp[N];
#pragma unroll
    for (int j = 0; j < N; ++j) {
        lp[j] = l[j] - lse;
        p[j] = e[j] * inv_se;            // exp(log_prob) over the mask, 0 outside
        if (mrow[j]) ent_row -= p[j] * lp[j];
    }
    ent_acc += ent_row;                   // optimizer.py:644-646 (divided by n_actions at the end)
    float g_lp = 0.f;                     // d loss / d logp[a]
    if (kBc && a_idx >= 0) {
        float lpa = lp[0];
        int best = -1;                    // arg-max of the masked logits, the lowest index on ties
        float lbest = 0.f;
#pragma unroll
        for (int j = 0; j < N; ++j) {
            lpa = (j == a_idx) ? lp[j] : lpa;
            if (mrow[j] && (best < 0 || l[j] > lbest)) {
                best = j;
                lbest = l[j];
            }
        }
        *nll_out = -lpa;
        *acc_out = best == a_idx ? 1.f : 0.f;
        *bc_in |= 1 << H;
        if (best != a_idx) *bc_miss |= 1 << H;
    }
    if (!kBc && a_idx >= 0) {
        float lpa = lp[0];
#pragma unroll
        for (int j = 1; j < N; ++j) lpa = (j == a_idx) ? lp[j] : lpa;
        const float log_r = lpa - old_lp;
        const float ratio = __expf(log_r);                             // optimizer.py:638
        // k3 estimator of KL(old || new); expm1f keeps it accurate for small |log r|, where r - 1 from __expf
        // would carry an error as large as the value itself
        *kl_out = expm1f(log_r) - log_r;
        *clip_out = fabsf(ratio - 1.0f) > e_clip ? 1.f : 0.f;
        const float lo = 1.0f - e_clip, hi = 1.0f + e_clip;
        const float s1 = ratio * adv_n;                                // :639
        const float s2 = fminf(fmaxf(ratio, lo), hi) * adv_n;          // :640
        float surr = fminf(s1, s2), g_s = 1.f;
        if (kDual) dual_clip_term(surr, g_s, adv_n, dual_c, dual_out);  // max(surr, c A) for A < 0
        pol_acc += surr;                                               // :641 (negated, averaged at the end)
        // autograd of torch.min(a, b): ties split the gradient in half; clamp passes it inside [lo, hi].
        const float g1 = s1 < s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
        const float g2 = s2 < s1 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
        const float in_range = (ratio >= lo && ratio <= hi) ? 1.f : 0.f;
        g_lp = -(1.0f / kHeads) / (float)n_h * adv_n * (g1 + g2 * in_range) * ratio;
        if (kDual) g_lp *= g_s;
    }
    if (kGrad) {
        const float ce = entropy_coef > 0.f ? entropy_coef / (float)n_h : 0.f;   // optimizer.py:652-656
        float kl_row = 0.f, t_row = 0.f;
#pragma unroll
        for (int j = 0; j < N; ++j) {
            float g = -g_lp * p[j];                       // through logsumexp (masked entries only: p = 0 outside)
            if (j == a_idx) g += g_lp;
            if (mrow[j]) g += ce * p[j] * (lp[j] + ent_row);   // d(-coef * entropy)/d logit
            if (kKl && a_idx >= 0 && mrow[j]) {          // KL(p_old || p) of a row in S_t, and beta / T_a (p - p_old)
                const float lo = orow[j], po = __expf(lo);
                kl_row += po * (lo - lp[j]);
                if (kl_scale > 0.f) g += kl_scale * (p[j] - po);
            }
            if (kTeach && a_idx >= 0 && mrow[j]) {       // KL(p_T || p), and lambda / T_a (p - p_T)
                const float lt = trow[j], pt = __expf(lt);
                t_row += pt * (lt - lp[j]);
                if (t_scale > 0.f) g += t_scale * (p[j] - pt);
            }
            if (kBc && a_idx >= 0 && mrow[j]) g += bc_scale * (j == a_idx ? p[j] - 1.0f : p[j]);   // -log p(a) / T_a
            lrow[j] = g;
        }
        if (kKl && a_idx >= 0) *kl_row_out = kl_row;
        if (kTeach && a_idx >= 0) *t_row_out = t_row;
    }
}

// Joint ratio, sweep 1 over head H of one token: masked log-softmax, entropy and the per-head diagnostics as head_token,
// and the head's term lp[a] - old_lp of the joint log-ratio.  Sets bit H of in_s when the head has an action row here.
template <int H>
__device__ __forceinline__ void joint_head_fwd(const float *lrow, const uint8_t *mrow, const uint8_t *arow, float old_lp,
                                               int n_h, float e_clip, float &ent_acc, float *kl_out, float *clip_out,
                                               float &log_r, int &in_s) {
    constexpr int N = head_n(H);
    float l[N], e[N];
    int mask_any = 0, a_idx = -1;
    float se = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        l[j] = lrow[j];
        const int m = mrow[j];
        mask_any |= m;
        e[j] = m ? __expf(l[j]) : 0.f;
        se += e[j];
        if (arow[j]) a_idx = j;
    }
    if (n_h == 0 || (!mask_any && a_idx < 0)) return;     // skipped as in head_token
    const float lse = logf(se);
    const float inv_se = 1.0f / se;
    float ent_row = 0.f, lpa = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const float lp = l[j] - lse;
        if (mrow[j]) ent_row -= (e[j] * inv_se) * lp;
        if (j == a_idx) lpa = lp;
    }
    ent_acc += ent_row;
    if (a_idx >= 0) {
        const float lr = lpa - old_lp;
        *kl_out = expm1f(lr) - lr;
        *clip_out = fabsf(__expf(lr) - 1.0f) > e_clip ? 1.f : 0.f;
        log_r += lr;                      // head order 0..4, fp32
        in_s |= 1 << H;
    }
}

// Joint ratio, sweep 2 over head H: the dlogits row, with g_lp = d loss / d lp[a] of the joint surrogate (the same for
// every head with an action row) and the head's entropy term, recomputed from the tile exactly as sweep 1 computed it.
// kKl / kTeach: the head's exact KL to the old / teacher row and its gradient, as in head_token.
template <int H, bool kKl = false, bool kTeach = false>
__device__ __forceinline__ void joint_head_bwd(float *lrow, const uint8_t *mrow, const uint8_t *arow, int n_h, float g_lp,
                                               float entropy_coef, const float *orow = nullptr, float kl_scale = 0.f,
                                               float *kl_row_out = nullptr, const float *trow = nullptr,
                                               float t_scale = 0.f, float *t_row_out = nullptr) {
    constexpr int N = head_n(H);
    float l[N], e[N];
    int mask_any = 0, a_idx = -1;
    float se = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        l[j] = lrow[j];
        const int m = mrow[j];
        mask_any |= m;
        e[j] = m ? __expf(l[j]) : 0.f;
        se += e[j];
        if (arow[j]) a_idx = j;
    }
    if (n_h == 0 || (!mask_any && a_idx < 0)) {
#pragma unroll
        for (int j = 0; j < N; ++j) lrow[j] = 0.f;
        return;
    }
    const float lse = logf(se);
    const float inv_se = 1.0f / se;
    float ent_row = 0.f;
    float p[N], lp[N];
#pragma unroll
    for (int j = 0; j < N; ++j) {
        lp[j] = l[j] - lse;
        p[j] = e[j] * inv_se;
        if (mrow[j]) ent_row -= p[j] * lp[j];
    }
    if (a_idx < 0) g_lp = 0.f;
    const float ce = entropy_coef > 0.f ? entropy_coef / (float)n_h : 0.f;
    float kl_row = 0.f, t_row = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        float g = -g_lp * p[j];
        if (j == a_idx) g += g_lp;
        if (mrow[j]) g += ce * p[j] * (lp[j] + ent_row);
        if (kKl && a_idx >= 0 && mrow[j]) {
            const float lo = orow[j], po = __expf(lo);
            kl_row += po * (lo - lp[j]);
            if (kl_scale > 0.f) g += kl_scale * (p[j] - po);
        }
        if (kTeach && a_idx >= 0 && mrow[j]) {
            const float lt = trow[j], pt = __expf(lt);
            t_row += pt * (lt - lp[j]);
            if (t_scale > 0.f) g += t_scale * (p[j] - pt);
        }
        lrow[j] = g;
    }
    if (kKl && a_idx >= 0) *kl_row_out = kl_row;
    if (kTeach && a_idx >= 0) *t_row_out = t_row;
}

// kSelectOnly && kKl: the selected log-probs and, written through hp.dlogits (column ranges of the [N, 65] rows), every
// head's masked log-prob row.  !kSelectOnly && kKl: the loss with the KL penalty (old_rows, kl_out).  kTeacher (a loss):
// the teacher term (teacher_rows, *teacher_coef, teacher_stats), with or without kKl.
// kBc (a loss, per-head path, neither kKl nor kTeacher): behaviour cloning, the NLL of the actions in place of the surrogate
// (bc_stats); old_logp and the advantages are not read.
// kDual (a loss, either ratio mode, with or without kKl and kTeacher): dual clip, the floor under negative-advantage
// surrogates (*dual_clip, dual_clip_stats).
// kTeacher, kBc and kDual ask for 2 CTAs per SM, which lets ptxas use more than the ~168 registers it picks otherwise and
// spill nothing; the other instantiations keep ptxas's default (minBlocks 0 is "not given"), so their code is unchanged.
template <bool kSelectOnly, bool kJoint, bool kKl = false, bool kTeacher = false, bool kBc = false, bool kDual = false>
__global__ void __launch_bounds__(kTile, (kTeacher || kBc || kDual) ? 2 : 0) ppo_loss_kernel(HeadPtrs hp, const float *__restrict__ old_logp,
                                                          const float *__restrict__ adv_raw,
                                                          const float *__restrict__ ret,
                                                          const float *__restrict__ value, int64_t N, float e_clip,
                                                          float entropy_coef, float vf_coef,
                                                          const float *__restrict__ old_value,
                                                          const uint8_t *__restrict__ valid,
                                                          const double *__restrict__ hparams,
                                                          float *__restrict__ dvalue, float *__restrict__ out,
                                                          float *__restrict__ stats, Workspace *ws,
                                                          float *__restrict__ logp_out,
                                                          const float *__restrict__ old_rows, float *__restrict__ kl_out,
                                                          const float *__restrict__ teacher_rows,
                                                          const double *__restrict__ teacher_coef,
                                                          float *__restrict__ teacher_stats,
                                                          float *__restrict__ bc_stats,
                                                          const double *__restrict__ dual_clip,
                                                          float *__restrict__ dual_clip_stats) {
    static_assert(!(kSelectOnly && kJoint), "the joint ratio is a loss");
    static_assert(!kDual || !(kSelectOnly || kBc), "dual clip caps the PPO surrogate");
    static_assert(!(kSelectOnly && kTeacher), "the teacher term is a loss");
    static_assert(!kBc || !(kSelectOnly || kJoint || kKl || kTeacher), "behaviour cloning is a per-head loss of its own");
    constexpr bool kKlLoss = kKl && !kSelectOnly;
    constexpr int kTokKl = kTokRows + (kJoint ? kJointStats : 0);
    constexpr int kTokTeach = kTokKl + (kKlLoss ? kKlStats : 0);
    constexpr int kTokBc = kTokTeach + (kTeacher ? kTeachStats : 0);
    constexpr int kTokDual = kTokBc + (kBc ? kBcStats : 0);
    constexpr int kRows = kTokDual + (kDual ? (kJoint ? 1 : kDualStats) : 0);
    constexpr int kSumKl = kStats + (kJoint ? kJointStats : 0);
    constexpr int kSumTeach = kSumKl + (kKlLoss ? kKlStats : 0);
    constexpr int kSumBc = kSumTeach + (kTeacher ? kTeachStats : 0);
    constexpr int kSumDual = kSumBc + (kBc ? kBcStats : 0);
    constexpr int kSums = kSumDual + (kDual ? (kJoint ? 1 : kDualStats) : 0);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *s_logits = reinterpret_cast<float *>(smem_raw);
    float *s_old = s_logits + kLogitFloats;
    uint8_t *s_mask = reinterpret_cast<uint8_t *>(s_old + kOldFloats);
    uint8_t *s_act = s_mask + kByteTile;
    float *s_orows = reinterpret_cast<float *>(smem_raw + kSmemBytes);    // kKlLoss: [kTile][65] prep-time log-prob rows
    float *s_trows = s_orows + (kKlLoss ? kTile * kRowFloats : 0);          // kTeacher: [kTile][65] teacher log-prob rows
    __shared__ float s_red[kTile / 32];
    // per-token diagnostics (rows kStKl.., kStClip.., then ret - v and ret, then the joint ratio's), staged here rather
    // than held in registers across the head loop, and their block sums
    __shared__ float s_tok[kRows][kTile];
    __shared__ double s_st[kSums];
    __shared__ bool s_last;

    // hyper-parameters from the device block when given, rounded to the types of the scalar arguments
    float value_clip = 0.f;
    double vn_mu = 0.0, vn_sigma = 0.0;     // value normalisation: sigma > 0 turns it on
    float kl_coef = 0.f;                    // KL control: beta
    if (!kSelectOnly && hparams) {
        e_clip = (float)hparams[DC_HP_E_CLIP];
        entropy_coef = (float)hparams[DC_HP_ENTROPY_COEF];
        vf_coef = (float)hparams[DC_HP_VF_COEF];
        value_clip = (float)hparams[DC_HP_VALUE_CLIP];
        vn_mu = hparams[DC_HP_VALUE_NORM_MEAN];
        vn_sigma = hparams[DC_HP_VALUE_NORM_STD];
        if (kKlLoss) kl_coef = (float)hparams[DC_HP_KL_COEF];
    }
    const float t_coef = kTeacher ? (float)*teacher_coef : 0.f;     // teacher: lambda
    const float dual_c = kDual ? (float)*dual_clip : 0.f;            // dual clip: c
    const bool vnorm = vn_sigma > 0.0;
    const bool clip_value = old_value != nullptr && value_clip > 0.f;

    const int64_t t0 = (int64_t)blockIdx.x * kTile;
    const int count = (int)min((int64_t)kTile, N - t0);
    stage_rows_f32<4, 5>(s_logits + logit_off(0), hp.logits[0], hp.ld_l[0], t0, count);
    stage_rows_f32<9, 9>(s_logits + logit_off(1), hp.logits[1], hp.ld_l[1], t0, count);
    stage_rows_f32<9, 9>(s_logits + logit_off(2), hp.logits[2], hp.ld_l[2], t0, count);
    stage_rows_f32<40, 41>(s_logits + logit_off(3), hp.logits[3], hp.ld_l[3], t0, count);
    stage_rows_f32<3, 3>(s_logits + logit_off(4), hp.logits[4], hp.ld_l[4], t0, count);
    if (!kSelectOnly && !kBc) stage_rows_f32<5, 5>(s_old, old_logp, 5, t0, count);
#pragma unroll
    for (int h = 0; h < kHeads; ++h) {
        stage_bytes(s_mask + byte_off(h), hp.masks[h] + t0 * head_n(h), count * head_n(h));
        stage_bytes(s_act + byte_off(h), hp.actions[h] + t0 * head_n(h), count * head_n(h));
    }
    if (kKlLoss)      // contiguous rows: a byte copy of the tile with 16-byte loads
        stage_bytes(reinterpret_cast<uint8_t *>(s_orows), reinterpret_cast<const uint8_t *>(old_rows + t0 * kRowFloats),
                    count * kRowFloats * 4);
    if (kTeacher)
        stage_bytes(reinterpret_cast<uint8_t *>(s_trows), reinterpret_cast<const uint8_t *>(teacher_rows + t0 * kRowFloats),
                    count * kRowFloats * 4);
    __syncthreads();

    const int t = threadIdx.x;
    const bool live = t < count;
    float pol[kHeads] = {0, 0, 0, 0, 0}, ent[kHeads] = {0, 0, 0, 0, 0};
    float vl = 0.f;
    if (!kSelectOnly) {
#pragma unroll
        for (int i = 0; i < kRows; ++i) s_tok[i][t] = 0.f;        // rows without an action (and dead threads) count 0
    }
    int cnt[kHeads] = {0, 0, 0, 0, 0};
    float adv_n = 0.f;
    // a token that does not count (valid = 0): every contribution below is skipped and its gradients are zero
    const bool use = live && (valid == nullptr || valid[t0 + t] != 0);
    if (!kSelectOnly) {
#pragma unroll
        for (int h = 0; h < kHeads; ++h) cnt[h] = ws->cnt[h];
        if (use && !kBc) {
            // (advantage - mean) / (std + eps), fp32 like optimizer.py:588
            adv_n = __fdiv_rn(__fsub_rn(adv_raw[t0 + t], ws->adv_mean), __fadd_rn(ws->adv_std, 1.1920928955078125e-07f));
        }
    }
    // KL control: beta / T_a, the weight of (p - p_old) in the dlogits rows of S_t; 0 (no gradient term) when beta = 0
    float kl_scale = 0.f;
    if (kKlLoss && kl_coef > 0.f) {
        const unsigned long long n_a = ws->n_joint;
        if (n_a) kl_scale = kl_coef / (float)n_a;
    }
    // KL control: this token's entry in the staging row of head 0's KL (head H's is H rows further).  Without kKl those
    // rows do not exist and nothing is staged there.
    float *const s_kl_tok = kKlLoss ? &s_tok[0][0] + kTokKl * kTile + t : nullptr;
    // teacher: lambda / T_a (0 when lambda = 0), and this token's entry in the staging row of head 0's teacher KL
    float t_scale = 0.f;
    if (kTeacher && t_coef > 0.f) {
        const unsigned long long n_a = ws->n_joint;
        if (n_a) t_scale = t_coef / (float)n_a;
    }
    float *const s_t_tok = kTeacher ? &s_tok[0][0] + kTokTeach * kTile + t : nullptr;
    // behaviour cloning: 1 / T_a, and this token's entry in the staging row of head 0's NLL (the rows of kBcStats follow)
    float bc_scale = 0.f;
    if (kBc) {
        const unsigned long long n_a = ws->n_joint;
        if (n_a) bc_scale = 1.0f / (float)n_a;
    }
    float *const s_bc_tok = kBc ? &s_tok[0][0] + kTokBc * kTile + t : nullptr;
    // dual clip: this token's entry in the staging row of head 0's bound flag (joint ratio: the token's only one)
    float *const s_dual_tok = kDual ? &s_tok[0][0] + kTokDual * kTile + t : nullptr;
    int bc_in = 0, bc_miss = 0;       // behaviour cloning: the heads of S_t, and those whose arg-max is not the action
    if (live) {
        float lp_sel[kHeads];
        if constexpr (kJoint) {
            float log_r = 0.f;
            int in_s = 0;
#define DC_JHEAD(H)                                                                                                 \
            joint_head_fwd<H>(s_logits + logit_off(H) + t * head_pitch(H), s_mask + byte_off(H) + t * head_n(H),    \
                              s_act + byte_off(H) + t * head_n(H), s_old[t * 5 + H], use ? cnt[H] : 0, e_clip,       \
                              ent[H], &s_tok[kStKl + H][t], &s_tok[kStClip + H][t], log_r, in_s);
            DC_JHEAD(0) DC_JHEAD(1) DC_JHEAD(2) DC_JHEAD(3) DC_JHEAD(4)
#undef DC_JHEAD
            float g_lp = 0.f;                 // d loss / d lp[a], the same for every head in S_t
            if (in_s) {                       // S_t not empty (so the token counts and T_a >= 1)
                const float ratio = __expf(log_r);
                s_tok[kTokJoint][t] = expm1f(log_r) - log_r;
                s_tok[kTokJoint + 1][t] = fabsf(ratio - 1.0f) > e_clip ? 1.f : 0.f;
                const float lo = 1.0f - e_clip, hi = 1.0f + e_clip;
                const float s1 = ratio * adv_n;
                const float s2 = fminf(fmaxf(ratio, lo), hi) * adv_n;
                float surr = fminf(s1, s2), g_s = 1.f;
                if (kDual) dual_clip_term(surr, g_s, adv_n, dual_c, s_dual_tok);   // as head_token caps each head's
                pol[0] += surr;
                // the same autograd rules as head_token: ties of torch.min split, clamp passes inside [lo, hi]
                const float g1 = s1 < s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
                const float g2 = s2 < s1 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
                const float in_range = (ratio >= lo && ratio <= hi) ? 1.f : 0.f;
                g_lp = -1.0f / (float)ws->n_joint * adv_n * (g1 + g2 * in_range) * ratio;
                if (kDual) g_lp *= g_s;
            }
            // sweep 2 re-reads the tile: without this the compiler keeps every head's sweep-1 values live instead
            asm volatile("" ::: "memory");
#define DC_JHEAD(H)                                                                                                 \
            joint_head_bwd<H, kKlLoss, kTeacher>(s_logits + logit_off(H) + t * head_pitch(H),                          \
                                       s_mask + byte_off(H) + t * head_n(H),                                            \
                                       s_act + byte_off(H) + t * head_n(H), use ? cnt[H] : 0, g_lp, entropy_coef,       \
                                       s_orows + t * kRowFloats + row_col(H), kl_scale,                                 \
                                       kKlLoss ? s_kl_tok + (H) * kTile : nullptr,                                      \
                                       s_trows + t * kRowFloats + row_col(H), t_scale,                                  \
                                       kTeacher ? s_t_tok + (H) * kTile : nullptr);
            DC_JHEAD(0) DC_JHEAD(1) DC_JHEAD(2) DC_JHEAD(3) DC_JHEAD(4)
#undef DC_JHEAD
        } else {
#define DC_HEAD(H)                                                                                              \
        head_token<H, true, kKl, kTeacher, kBc, kDual>(s_logits + logit_off(H) + t * head_pitch(H),              \
                                 s_mask + byte_off(H) + t * head_n(H),                                               \
                                 s_act + byte_off(H) + t * head_n(H),                                                \
                                 (kSelectOnly || kBc) ? 0.f : s_old[t * 5 + H], adv_n,                               \
                                 use ? cnt[H] : 0, e_clip, entropy_coef, pol[H], ent[H], &s_tok[kStKl + H][t],       \
                                 &s_tok[kStClip + H][t], kSelectOnly ? &lp_sel[H] : nullptr,                         \
                                 s_orows + t * kRowFloats + row_col(H), kl_scale,                                    \
                                 kKlLoss ? s_kl_tok + (H) * kTile : nullptr,                                         \
                                 s_trows + t * kRowFloats + row_col(H), t_scale,                                     \
                                 kTeacher ? s_t_tok + (H) * kTile : nullptr, bc_scale,                               \
                                 kBc ? s_bc_tok + (H) * kTile : nullptr,                                             \
                                 kBc ? s_bc_tok + (kHeads + 1 + (H)) * kTile : nullptr, &bc_in, &bc_miss, dual_c,    \
                                 kDual ? s_dual_tok + (H) * kTile : nullptr);
        DC_HEAD(0) DC_HEAD(1) DC_HEAD(2) DC_HEAD(3) DC_HEAD(4)
#undef DC_HEAD
            // behaviour cloning: the token is right when every head of S_t is (counted over the T_a tokens)
            if (kBc && bc_in) s_bc_tok[kHeads * kTile] = bc_miss ? 0.f : 1.f;
        }
        if (kSelectOnly) {
#pragma unroll
            for (int h = 0; h < kHeads; ++h) logp_out[(t0 + t) * 5 + h] = lp_sel[h];
        } else if (!use) {              // masked out: zero gradient rows (head_token with a count of 0), zero dvalue
            dvalue[(t0 + t) * hp.ld_dv] = 0.f;
        } else {
            // under value normalisation the head's output v is in normalised units: the raw target (and the raw old value)
            // are brought to them here, in float64 and rounded once; x - 0 and x / 1 are exact, so (0, 1) changes no bit
            const float v = value[(t0 + t) * hp.ld_v], r = vnorm ? vn_normalise(ret[t0 + t], vn_mu, vn_sigma) : ret[t0 + t];
            const float d = r - v;
            float g = v - r;                                                // d value_loss / d v, up to vf_coef / N
            if (clip_value) {
                // PPO2: max((v - R)^2, (v_old + clip(v - v_old, -eps, eps) - R)^2); autograd of torch.maximum (ties split
                // the gradient in half) and of clamp (passes it inside [-eps, eps])
                const float vo = vnorm ? vn_normalise(old_value[t0 + t], vn_mu, vn_sigma) : old_value[t0 + t];
                const float dv = v - vo;
                const float dc = (vo + fminf(fmaxf(dv, -value_clip), value_clip)) - r;
                const float l1 = d * d, l2 = dc * dc;
                vl = fmaxf(l1, l2);
                const float w1 = l1 > l2 ? 1.f : (l1 == l2 ? 0.5f : 0.f);
                const float w2 = l2 > l1 ? 1.f : (l1 == l2 ? 0.5f : 0.f);
                const float in_range = (dv >= -value_clip && dv <= value_clip) ? 1.f : 0.f;
                g = w1 * g + w2 * in_range * dc;
            } else {
                vl = d * d;                                                 // optimizer.py:660
            }
            dvalue[(t0 + t) * hp.ld_dv] = vf_coef > 0.f ? vf_coef * g / (float)ws->n_valid : 0.f;   // N_v, or N unmasked
            // the explained-variance sums run on values shifted by the first counting token's: constant returns then sum
            // to exactly zero variance (unshifted, the rounding of the float64 sums of r^2 leaves a variance of either
            // sign), and near-constant ones keep their digits; r - shift is exact for r within a factor 2 of the shift
            float shift_r = 0.f, shift_d = 0.f;
            if (stats) {
                const int64_t tf = N - (int64_t)ws->first_rev;    // this token counts, so first_rev > 0
                shift_r = vnorm ? vn_normalise(ret[tf], vn_mu, vn_sigma) : ret[tf];
                shift_d = shift_r - value[tf * hp.ld_v];
            }
            s_tok[kTokD][t] = d - shift_d;
            s_tok[kTokR][t] = r - shift_r;
        }
    }
    if (kSelectOnly && !kKl) return;
    __syncthreads();
    unstage_rows_f32<4, 5>(hp.dlogits[0], hp.ld_d[0], t0, s_logits + logit_off(0), count);
    unstage_rows_f32<9, 9>(hp.dlogits[1], hp.ld_d[1], t0, s_logits + logit_off(1), count);
    unstage_rows_f32<9, 9>(hp.dlogits[2], hp.ld_d[2], t0, s_logits + logit_off(2), count);
    unstage_rows_f32<40, 41>(hp.dlogits[3], hp.ld_d[3], t0, s_logits + logit_off(3), count);
    unstage_rows_f32<3, 3>(hp.dlogits[4], hp.ld_d[4], t0, s_logits + logit_off(4), count);
    if constexpr (!kSelectOnly) {   // kKl select: the log-prob rows went out through hp.dlogits; nothing else to do
        float sums[2 * kHeads + 1];
#pragma unroll
        for (int h = 0; h < kHeads; ++h) {
            sums[h] = block_sum(pol[h], s_red);
            sums[kHeads + h] = block_sum(ent[h], s_red);
        }
        sums[2 * kHeads] = block_sum(vl, s_red);
        // the diagnostics (s_tok is complete: block_sum synchronised the block): one warp per sum, in float64.  KL control
        // and the teacher need their sums for kl_out / teacher_stats whether or not the diagnostics are asked for.
        if (stats || kKlLoss || kTeacher || kBc || kDual) {
            const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
            for (int i = warp; i < kSums; i += kTile / 32) {
                const int row = (kDual && i >= kSumDual) ? kTokDual + (i - kSumDual)
                              : (kBc && i >= kSumBc) ? kTokBc + (i - kSumBc)
                              : (kTeacher && i >= kSumTeach) ? kTokTeach + (i - kSumTeach)
                              : (kKlLoss && i >= kSumKl) ? kTokKl + (i - kSumKl)
                              : (kJoint && i >= kStats) ? kTokJoint + (i - kStats) : (i < kStD ? i : (i < kStR ? kTokD : kTokR));
                const bool square = i == kStD2 || i == kStR2;
                double s = 0.0;
                for (int j = lane; j < kTile; j += 32) {
                    const double v = (double)s_tok[row][j];
                    s += square ? v * v : v;
                }
                s = dc_warp_sum(s);
                if (lane == 0) s_st[i] = s;
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
#pragma unroll
            for (int h = 0; h < kHeads; ++h) {
                if (sums[h] != 0.f) atomicAdd(&ws->pol[h], (double)sums[h]);
                if (sums[kHeads + h] != 0.f) atomicAdd(&ws->ent[h], (double)sums[kHeads + h]);
            }
            atomicAdd(&ws->vl, (double)sums[2 * kHeads]);
            if (stats) {
                for (int i = 0; i < kStats; ++i)
                    if (s_st[i] != 0.0) atomicAdd(&ws->st[i], s_st[i]);
                if constexpr (kJoint) {
                    for (int i = 0; i < kJointStats; ++i)
                        if (s_st[kStats + i] != 0.0) atomicAdd(&ws->st_joint[i], s_st[kStats + i]);
                }
            }
            if constexpr (kKlLoss) {
                for (int i = 0; i < kKlStats; ++i)
                    if (s_st[kSumKl + i] != 0.0) atomicAdd(&ws->st_kl[i], s_st[kSumKl + i]);
            }
            if constexpr (kTeacher) {
                for (int i = 0; i < kTeachStats; ++i)
                    if (s_st[kSumTeach + i] != 0.0) atomicAdd(&ws->st_teach[i], s_st[kSumTeach + i]);
            }
            if constexpr (kBc) {
                for (int i = 0; i < kBcStats; ++i)
                    if (s_st[kSumBc + i] != 0.0) atomicAdd(&ws->st_bc[i], s_st[kSumBc + i]);
            }
            if constexpr (kDual) {
                for (int i = 0; i < kSums - kSumDual; ++i)
                    if (s_st[kSumDual + i] != 0.0) atomicAdd(&ws->st_dual[i], s_st[kSumDual + i]);
            }
            __threadfence();
            s_last = atomicAdd(&ws->ticket_loss, 1u) == gridDim.x - 1;
        }
        __syncthreads();
        if (s_last && threadIdx.x == 0) {
            __threadfence();
            volatile Workspace *w = ws;
            float policy = 0.f, entropy = 0.f;
            for (int h = 0; h < kHeads; ++h) {
                const int n = w->cnt[h];
                const float pl = (!kJoint && !kBc && n) ? (float)(-w->pol[h] / (double)n) : 0.f;   // optimizer.py:641 / :628
                const float en = n ? (float)(w->ent[h] / (double)n) : 0.f;      // optimizer.py:646 / :629
                out[9 + h] = pl;
                out[4 + h] = en;
                policy += pl;
                entropy += en;
            }
            if constexpr (kJoint) {                                             // -(1/T_a) sum_t min(r A, clip(r) A); 0 if T_a = 0
                const unsigned long long n_a = w->n_joint;
                policy = n_a ? (float)(-w->pol[0] / (double)n_a) : 0.f;
            } else if constexpr (kBc) {
                // NLL = (1 / T_a) sum_t sum_{h in S_t} -log p(a_h) (0 when T_a = 0); out[9 + h] is head h's share of it
                const unsigned long long n_a = w->n_joint;
                double nll_sum = 0.0;
                for (int h = 0; h < kHeads; ++h) {
                    nll_sum += w->st_bc[h];
                    out[9 + h] = n_a ? (float)(w->st_bc[h] / (double)n_a) : 0.f;
                }
                policy = n_a ? (float)(nll_sum / (double)n_a) : 0.f;
                bc_stats[0] = policy;
                bc_stats[1 + kHeads] = n_a ? (float)(w->st_bc[kHeads] / (double)n_a) : 0.f;
                for (int h = 0; h < kHeads; ++h) {      // over the head's action rows; 0 for a head without any
                    const int n = w->cnt[h];
                    bc_stats[1 + h] = n ? (float)(w->st_bc[h] / (double)n) : 0.f;
                    bc_stats[2 + kHeads + h] = n ? (float)(w->st_bc[kHeads + 1 + h] / (double)n) : 0.f;
                }
            } else {
                policy /= (float)kHeads;                                        // optimizer.py:650
            }
            const float e_loss = entropy_coef > 0.f ? -entropy_coef * entropy : 0.f;
            const double n_tok_d = (double)w->n_valid;                          // N, or N_v under a valid mask
            const float v_loss = vf_coef > 0.f ? vf_coef * (0.5f * (float)(w->vl / n_tok_d)) : 0.f;
            out[0] = policy + e_loss + v_loss;                                  // optimizer.py:665
            out[1] = policy;
            out[2] = e_loss;
            out[3] = v_loss;
            out[14] = w->adv_mean;
            out[15] = w->adv_std;
            if (stats) {
                float kl_sum = 0.f, clip_sum = 0.f;
                int used = 0;
                for (int h = 0; h < kHeads; ++h) {      // a head without action rows reports 0 and is left out of the mean
                    const int n = w->cnt[h];
                    const float kl_h = n ? (float)(w->st[kStKl + h] / (double)n) : 0.f;
                    const float clip_h = n ? (float)(w->st[kStClip + h] / (double)n) : 0.f;
                    stats[DC_STAT_APPROX_KL + 1 + h] = kl_h;
                    stats[DC_STAT_CLIP_FRACTION + 1 + h] = clip_h;
                    kl_sum += kl_h;
                    clip_sum += clip_h;
                    used += n > 0;
                }
                stats[DC_STAT_APPROX_KL] = used ? kl_sum / (float)used : 0.f;
                stats[DC_STAT_CLIP_FRACTION] = used ? clip_sum / (float)used : 0.f;
                // 1 - Var(ret - v) / Var(ret) over the tokens that count (population variances, from the shifted sums);
                // NaN when the returns are constant
                const double n = n_tok_d;
                const double md = w->st[kStD] / n, mr = w->st[kStR] / n;
                const double var_d = w->st[kStD2] / n - md * md, var_r = w->st[kStR2] / n - mr * mr;
                stats[DC_STAT_EXPLAINED_VAR] = var_r > 0.0 ? (float)(1.0 - var_d / var_r) : __int_as_float(0x7fc00000);
                for (int i = DC_STAT_EXPLAINED_VAR + 1; i < DC_PPO_STATS_SLOTS; ++i) stats[i] = 0.f;
                if constexpr (kJoint) {
                    const unsigned long long n_a = w->n_joint;
                    stats[DC_STAT_JOINT_APPROX_KL] = n_a ? (float)(w->st_joint[0] / (double)n_a) : 0.f;
                    stats[DC_STAT_JOINT_CLIP_FRACTION] = n_a ? (float)(w->st_joint[1] / (double)n_a) : 0.f;
                }
            }
            if constexpr (kKlLoss) {
                // KL = (1 / T_a) sum_t KL_t (0 when T_a = 0); the penalty beta KL joins the total loss only when beta > 0, so
                // beta = 0 leaves out[0] as the instantiation without the penalty computes it
                const unsigned long long n_a = w->n_joint;
                double kl_sum = 0.0;
                for (int h = 0; h < kHeads; ++h) kl_sum += w->st_kl[h];
                const float kl = n_a ? (float)(kl_sum / (double)n_a) : 0.f;
                const float penalty = kl_coef > 0.f ? kl_coef * kl : 0.f;
                if (kl_coef > 0.f) out[0] = out[0] + penalty;
                if (stats) {
                    stats[DC_STAT_KL] = kl;
                    for (int h = 0; h < kHeads; ++h) {       // over the head's action rows; 0 for a head without any
                        const int n = w->cnt[h];
                        stats[DC_STAT_KL + 1 + h] = n ? (float)(w->st_kl[h] / (double)n) : 0.f;
                    }
                    stats[DC_STAT_KL_PENALTY] = penalty;
                }
                if (kl_out) {       // this rank's (sum_t KL_t, T_a): summed over the ranks by the gradient all-reduce
                    kl_out[0] = (float)kl_sum;
                    kl_out[1] = (float)n_a;
                }
            }
            if constexpr (kTeacher) {
                // KL_T = (1 / T_a) sum_t sum_{h in S_t} KL(p_T || p) of the row (0 when T_a = 0); lambda KL_T joins the loss
                // only when lambda > 0, so lambda = 0 leaves out[0] as the instantiation without the teacher computes it
                const unsigned long long n_a = w->n_joint;
                double t_sum = 0.0;
                for (int h = 0; h < kHeads; ++h) t_sum += w->st_teach[h];
                const float kl_t = n_a ? (float)(t_sum / (double)n_a) : 0.f;
                const float term = t_coef > 0.f ? t_coef * kl_t : 0.f;
                if (t_coef > 0.f) out[0] = out[0] + term;
                teacher_stats[0] = kl_t;
                for (int h = 0; h < kHeads; ++h) {           // over the head's action rows; 0 for a head without any
                    const int n = w->cnt[h];
                    teacher_stats[1 + h] = n ? (float)(w->st_teach[h] / (double)n) : 0.f;
                }
                teacher_stats[1 + kHeads] = term;
            }
            if constexpr (kDual) {
                // per head: the share of its action rows where the cap binds (0 for a head without any, and under the
                // joint ratio), their mean over the heads with action rows; the joint ratio: the share of the T_a tokens
                float sum = 0.f;
                int used = 0;
                for (int h = 0; h < kHeads; ++h) {
                    const int n = w->cnt[h];
                    const float f = (!kJoint && n) ? (float)(w->st_dual[h] / (double)n) : 0.f;
                    dual_clip_stats[1 + h] = f;
                    sum += f;
                    used += n > 0;
                }
                dual_clip_stats[0] = used ? sum / (float)used : 0.f;
                const unsigned long long n_a = w->n_joint;
                dual_clip_stats[1 + kHeads] = (kJoint && n_a) ? (float)(w->st_dual[0] / (double)n_a) : 0.f;
            }
        }
    }
}

int check_heads(const float *const logits[], const uint8_t *const masks[], const uint8_t *const actions[]) {
    for (int h = 0; h < kHeads; ++h)
        if (!logits[h] || !masks[h] || !actions[h]) return 0;
    return 1;
}

// Both launches of one loss evaluation.  hparams == nullptr: e_clip / entropy_coef / vf_coef are the scalar arguments and
// the value loss is not clipped; otherwise they come from the device block.  stats == nullptr skips the diagnostics.
// joint: the joint-ratio instantiations of both kernels.
int launch_ppo_loss(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                    const uint8_t *const masks[DC_NUM_HEADS], const uint8_t *const actions[DC_NUM_HEADS],
                    const float *old_logp, const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                    const float *old_value, const uint8_t *valid, int64_t N, float e_clip, float entropy_coef, float vf_coef,
                    const double *hparams, float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                    float *dvalue, int64_t ld_dvalue, float *out, float *stats, int32_t *n_actions, void *workspace,
                    dc_stream_t stream, bool joint = false, const float *old_rows = nullptr, float *kl_out = nullptr,
                    const float *teacher_rows = nullptr, const double *teacher_coef = nullptr,
                    float *teacher_stats = nullptr, float *bc_stats = nullptr, const double *dual_clip = nullptr,
                    float *dual_clip_stats = nullptr) {
    DC_REQUIRE(N > 0, DC_EINVAL, "dc_ppo_loss_fwd_bwd: N=%lld", (long long)N);
    // behaviour cloning (bc_stats given) reads no old_logp
    DC_REQUIRE(check_heads(logits, masks, actions) && (old_logp || bc_stats) && adv_raw && ret && value && dvalue && out &&
                   n_actions && workspace && ld_logits && ld_dlogits, DC_EINVAL, "dc_ppo_loss_fwd_bwd: null pointer");
    HeadPtrs hp;
    for (int h = 0; h < kHeads; ++h) {
        DC_REQUIRE(dlogits[h], DC_EINVAL, "dc_ppo_loss_fwd_bwd: null dlogits[%d]", h);
        DC_REQUIRE(ld_logits[h] >= head_n(h) && ld_dlogits[h] >= head_n(h), DC_EINVAL, "dc_ppo_loss_fwd_bwd: row pitch of head %d", h);
        hp.logits[h] = logits[h]; hp.masks[h] = masks[h]; hp.actions[h] = actions[h]; hp.dlogits[h] = dlogits[h];
        hp.ld_l[h] = ld_logits[h]; hp.ld_d[h] = ld_dlogits[h];
    }
    DC_REQUIRE(ld_value >= 1 && ld_dvalue >= 1, DC_EINVAL, "dc_ppo_loss_fwd_bwd: value pitch");
    hp.ld_v = ld_value; hp.ld_dv = ld_dvalue;
    cudaStream_t st = dc_cu_stream(stream);
    Workspace *ws = reinterpret_cast<Workspace *>(workspace);
    DC_CUDA(cudaMemsetAsync(ws, 0, sizeof(Workspace), st));
    const unsigned blocks = (unsigned)((N + kTile - 1) / kTile);
    if (dual_clip_stats) {      // dual clip, either ratio mode, with or without the KL rows and the teacher's
        // the statistics pass of the entry point without the cap: T_a is counted when a term needs it
        if (joint || old_rows || teacher_rows)
            ppo_stats_kernel<true><<<blocks, kTile, 0, st>>>(hp, adv_raw, valid, N, ws, n_actions);
        else
            ppo_stats_kernel<false><<<blocks, kTile, 0, st>>>(hp, adv_raw, valid, N, ws, n_actions);
        DC_LAUNCH_OK();
        auto kern = ppo_loss_kernel<false, false, false, false, false, true>;
        if (teacher_rows)
            kern = old_rows ? (joint ? ppo_loss_kernel<false, true, true, true, false, true>
                                     : ppo_loss_kernel<false, false, true, true, false, true>)
                            : (joint ? ppo_loss_kernel<false, true, false, true, false, true>
                                     : ppo_loss_kernel<false, false, false, true, false, true>);
        else
            kern = old_rows ? (joint ? ppo_loss_kernel<false, true, true, false, false, true>
                                     : ppo_loss_kernel<false, false, true, false, false, true>)
                            : (joint ? ppo_loss_kernel<false, true, false, false, false, true>
                                     : ppo_loss_kernel<false, false, false, false, false, true>);
        const size_t smem = teacher_rows ? (old_rows ? kSmemBytesKlTeacher : kSmemBytesKl)
                                         : (old_rows ? kSmemBytesKl : kSmemBytes);
        DC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<blocks, kTile, smem, st>>>(hp, old_logp, adv_raw, ret, value, N, e_clip, entropy_coef, vf_coef, old_value,
                                          valid, hparams, dvalue, out, stats, ws, nullptr, old_rows, kl_out, teacher_rows,
                                          teacher_coef, teacher_stats, nullptr, dual_clip, dual_clip_stats);
        DC_LAUNCH_OK();
        return DC_OK;
    }
    if (bc_stats) {             // behaviour cloning: the statistics pass counts T_a
        ppo_stats_kernel<true><<<blocks, kTile, 0, st>>>(hp, adv_raw, valid, N, ws, n_actions);
        DC_LAUNCH_OK();
        auto kern = ppo_loss_kernel<false, false, false, false, true>;
        DC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
        kern<<<blocks, kTile, kSmemBytes, st>>>(hp, nullptr, adv_raw, ret, value, N, e_clip, entropy_coef, vf_coef, old_value,
                                                valid, hparams, dvalue, out, stats, ws, nullptr, nullptr, nullptr, nullptr,
                                                nullptr, nullptr, bc_stats, nullptr, nullptr);
        DC_LAUNCH_OK();
        return DC_OK;
    }
    if (teacher_rows) {         // the teacher term, with or without KL control, either ratio mode; T_a as below
        ppo_stats_kernel<true><<<blocks, kTile, 0, st>>>(hp, adv_raw, valid, N, ws, n_actions);
        DC_LAUNCH_OK();
        auto kern = old_rows ? (joint ? ppo_loss_kernel<false, true, true, true> : ppo_loss_kernel<false, false, true, true>)
                             : (joint ? ppo_loss_kernel<false, true, false, true> : ppo_loss_kernel<false, false, false, true>);
        const size_t smem = old_rows ? kSmemBytesKlTeacher : kSmemBytesKl;
        DC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<blocks, kTile, smem, st>>>(hp, old_logp, adv_raw, ret, value, N, e_clip, entropy_coef, vf_coef, old_value,
                                          valid, hparams, dvalue, out, stats, ws, nullptr, old_rows, kl_out, teacher_rows,
                                          teacher_coef, teacher_stats, nullptr, nullptr, nullptr);
        DC_LAUNCH_OK();
        return DC_OK;
    }
    if (old_rows) {             // KL control, either ratio mode; the statistics pass counts T_a
        ppo_stats_kernel<true><<<blocks, kTile, 0, st>>>(hp, adv_raw, valid, N, ws, n_actions);
        DC_LAUNCH_OK();
        auto kern = joint ? ppo_loss_kernel<false, true, true> : ppo_loss_kernel<false, false, true>;
        DC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytesKl));
        kern<<<blocks, kTile, kSmemBytesKl, st>>>(hp, old_logp, adv_raw, ret, value, N, e_clip, entropy_coef, vf_coef, old_value,
                                                  valid, hparams, dvalue, out, stats, ws, nullptr, old_rows, kl_out,
                                                  nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
        DC_LAUNCH_OK();
        return DC_OK;
    }
    if (joint) {
        ppo_stats_kernel<true><<<blocks, kTile, 0, st>>>(hp, adv_raw, valid, N, ws, n_actions);
        DC_LAUNCH_OK();
        DC_CUDA(cudaFuncSetAttribute(ppo_loss_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)kSmemBytes));
        ppo_loss_kernel<false, true><<<blocks, kTile, kSmemBytes, st>>>(hp, old_logp, adv_raw, ret, value, N, e_clip,
                                                                        entropy_coef, vf_coef, old_value, valid, hparams,
                                                                        dvalue, out, stats, ws, nullptr, nullptr, nullptr, nullptr,
                                                                        nullptr, nullptr, nullptr, nullptr, nullptr);
        DC_LAUNCH_OK();
        return DC_OK;
    }
    ppo_stats_kernel<false><<<blocks, kTile, 0, st>>>(hp, adv_raw, valid, N, ws, n_actions);
    DC_LAUNCH_OK();
    // per-device attribute: set on every call (a process-wide "done" flag breaks the second GPU of a process)
    DC_CUDA(cudaFuncSetAttribute(ppo_loss_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
    DC_CUDA(cudaFuncSetAttribute(ppo_loss_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
    ppo_loss_kernel<false, false><<<blocks, kTile, kSmemBytes, st>>>(hp, old_logp, adv_raw, ret, value, N, e_clip,
                                                                     entropy_coef, vf_coef, old_value, valid, hparams,
                                                                     dvalue, out, stats, ws, nullptr, nullptr, nullptr, nullptr,
                                                                        nullptr, nullptr, nullptr, nullptr, nullptr);
    DC_LAUNCH_OK();
    return DC_OK;
}

}  // namespace

extern "C" int dc_ppo_loss_fwd_bwd_strided(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                           const uint8_t *const masks[DC_NUM_HEADS],
                                           const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                                           const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                           int64_t N, float e_clip, float entropy_coef, float vf_coef,
                                           float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                                           float *dvalue, int64_t ld_dvalue, float *out, int32_t *n_actions, void *workspace,
                                           dc_stream_t stream) {
    return launch_ppo_loss(logits, ld_logits, masks, actions, old_logp, adv_raw, ret, value, ld_value, nullptr, nullptr, N,
                           e_clip, entropy_coef, vf_coef, nullptr, dlogits, ld_dlogits, dvalue, ld_dvalue, out, nullptr, n_actions,
                           workspace, stream);
}

extern "C" int dc_ppo_loss_fwd_bwd_dev(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                       const uint8_t *const masks[DC_NUM_HEADS], const uint8_t *const actions[DC_NUM_HEADS],
                                       const float *old_logp, const float *adv_raw, const float *ret, const float *value,
                                       int64_t ld_value, const float *old_value, int64_t N, const double *hparams,
                                       float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                                       float *dvalue, int64_t ld_dvalue, float *out, float *stats, int32_t *n_actions,
                                       void *workspace, dc_stream_t stream) {
    DC_REQUIRE(hparams, DC_EINVAL, "dc_ppo_loss_fwd_bwd_dev: null hyper-parameter block");
    return launch_ppo_loss(logits, ld_logits, masks, actions, old_logp, adv_raw, ret, value, ld_value, old_value, nullptr,
                           N, 0.f, 0.f, 0.f, hparams, dlogits, ld_dlogits, dvalue, ld_dvalue, out, stats, n_actions,
                           workspace, stream);
}

extern "C" int dc_ppo_loss_fwd_bwd_masked(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                          const uint8_t *const masks[DC_NUM_HEADS],
                                          const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                                          const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                          const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                                          float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                                          float *dvalue, int64_t ld_dvalue, float *out, float *stats, int32_t *n_actions,
                                          void *workspace, dc_stream_t stream) {
    DC_REQUIRE(hparams, DC_EINVAL, "dc_ppo_loss_fwd_bwd_masked: null hyper-parameter block");
    return launch_ppo_loss(logits, ld_logits, masks, actions, old_logp, adv_raw, ret, value, ld_value, old_value, valid,
                           N, 0.f, 0.f, 0.f, hparams, dlogits, ld_dlogits, dvalue, ld_dvalue, out, stats, n_actions,
                           workspace, stream);
}

extern "C" int dc_ppo_loss_fwd_bwd_joint(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                         const uint8_t *const masks[DC_NUM_HEADS],
                                         const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                                         const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                         const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                                         float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                                         float *dvalue, int64_t ld_dvalue, float *out, float *stats, int32_t *n_actions,
                                         void *workspace, dc_stream_t stream) {
    DC_REQUIRE(hparams, DC_EINVAL, "dc_ppo_loss_fwd_bwd_joint: null hyper-parameter block");
    return launch_ppo_loss(logits, ld_logits, masks, actions, old_logp, adv_raw, ret, value, ld_value, old_value, valid,
                           N, 0.f, 0.f, 0.f, hparams, dlogits, ld_dlogits, dvalue, ld_dvalue, out, stats, n_actions,
                           workspace, stream, true);
}

extern "C" int dc_ppo_loss_fwd_bwd(const float *const logits[DC_NUM_HEADS], const uint8_t *const masks[DC_NUM_HEADS],
                                   const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                                   const float *adv_raw, const float *ret, const float *value, int64_t N,
                                   float e_clip, float entropy_coef, float vf_coef,
                                   float *const dlogits[DC_NUM_HEADS], float *dvalue, float *out,
                                   int32_t *n_actions, void *workspace, dc_stream_t stream) {
    const int64_t ld[DC_NUM_HEADS] = {4, 9, 9, 40, 3};
    return dc_ppo_loss_fwd_bwd_strided(logits, ld, masks, actions, old_logp, adv_raw, ret, value, 1, N, e_clip, entropy_coef,
                                       vf_coef, dlogits, ld, dvalue, 1, out, n_actions, workspace, stream);
}

extern "C" int dc_selected_logp(const float *const logits[DC_NUM_HEADS], const uint8_t *const masks[DC_NUM_HEADS],
                                const uint8_t *const actions[DC_NUM_HEADS], int64_t N, float *logp_out,
                                dc_stream_t stream) {
    DC_REQUIRE(N > 0, DC_EINVAL, "dc_selected_logp: N=%lld", (long long)N);
    DC_REQUIRE(check_heads(logits, masks, actions) && logp_out, DC_EINVAL, "dc_selected_logp: null pointer");
    HeadPtrs hp;
    for (int h = 0; h < kHeads; ++h) {
        hp.logits[h] = logits[h]; hp.masks[h] = masks[h]; hp.actions[h] = actions[h]; hp.dlogits[h] = nullptr;
        hp.ld_l[h] = head_n(h); hp.ld_d[h] = head_n(h);
    }
    hp.ld_v = 1; hp.ld_dv = 1;
    // per-device attribute: set on every call (a process-wide "done" flag breaks the second GPU of a process)
    DC_CUDA(cudaFuncSetAttribute(ppo_loss_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
    const unsigned blocks = (unsigned)((N + kTile - 1) / kTile);
    ppo_loss_kernel<true, false><<<blocks, kTile, kSmemBytes, dc_cu_stream(stream)>>>(
        hp, nullptr, nullptr, nullptr, nullptr, N, 0.f, 0.f, 0.f, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
        nullptr, logp_out, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_selected_logp_rows(const float *const logits[DC_NUM_HEADS], const uint8_t *const masks[DC_NUM_HEADS],
                                     const uint8_t *const actions[DC_NUM_HEADS], int64_t N, float *logp_out,
                                     float *logp_rows, dc_stream_t stream) {
    DC_REQUIRE(N > 0, DC_EINVAL, "dc_selected_logp_rows: N=%lld", (long long)N);
    DC_REQUIRE(check_heads(logits, masks, actions) && logp_out && logp_rows, DC_EINVAL,
               "dc_selected_logp_rows: null pointer");
    HeadPtrs hp;
    for (int h = 0; h < kHeads; ++h) {      // head h's entries are columns row_col(h).. of the [N, 65] rows
        hp.logits[h] = logits[h]; hp.masks[h] = masks[h]; hp.actions[h] = actions[h];
        hp.dlogits[h] = logp_rows + row_col(h);
        hp.ld_l[h] = head_n(h); hp.ld_d[h] = kRowFloats;
    }
    hp.ld_v = 1; hp.ld_dv = 1;
    DC_CUDA(cudaFuncSetAttribute(ppo_loss_kernel<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)kSmemBytes));
    const unsigned blocks = (unsigned)((N + kTile - 1) / kTile);
    ppo_loss_kernel<true, false, true><<<blocks, kTile, kSmemBytes, dc_cu_stream(stream)>>>(
        hp, nullptr, nullptr, nullptr, nullptr, N, 0.f, 0.f, 0.f, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
        nullptr, logp_out, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_ppo_loss_fwd_bwd_kl(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                      const uint8_t *const masks[DC_NUM_HEADS], const uint8_t *const actions[DC_NUM_HEADS],
                                      const float *old_logp, const float *old_log_probs, const float *adv_raw,
                                      const float *ret, const float *value, int64_t ld_value, const float *old_value,
                                      const uint8_t *valid, int64_t N, const double *hparams, int joint,
                                      float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                                      float *dvalue, int64_t ld_dvalue, float *out, float *stats, float *kl_out,
                                      int32_t *n_actions, void *workspace, dc_stream_t stream) {
    DC_REQUIRE(hparams, DC_EINVAL, "dc_ppo_loss_fwd_bwd_kl: null hyper-parameter block");
    DC_REQUIRE(old_log_probs, DC_EINVAL, "dc_ppo_loss_fwd_bwd_kl: null old_log_probs");
    return launch_ppo_loss(logits, ld_logits, masks, actions, old_logp, adv_raw, ret, value, ld_value, old_value, valid,
                           N, 0.f, 0.f, 0.f, hparams, dlogits, ld_dlogits, dvalue, ld_dvalue, out, stats, n_actions,
                           workspace, stream, joint != 0, old_log_probs, kl_out);
}

extern "C" int dc_ppo_loss_fwd_bwd_teacher(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                           const uint8_t *const masks[DC_NUM_HEADS],
                                           const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                                           const float *old_log_probs, const float *teacher_log_probs,
                                           const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                           const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                                           const double *teacher_coef, int joint, float *const dlogits[DC_NUM_HEADS],
                                           const int64_t ld_dlogits[DC_NUM_HEADS], float *dvalue, int64_t ld_dvalue,
                                           float *out, float *stats, float *kl_out, float *teacher_stats,
                                           int32_t *n_actions, void *workspace, dc_stream_t stream) {
    DC_REQUIRE(hparams, DC_EINVAL, "dc_ppo_loss_fwd_bwd_teacher: null hyper-parameter block");
    DC_REQUIRE(teacher_log_probs && teacher_coef && teacher_stats, DC_EINVAL,
               "dc_ppo_loss_fwd_bwd_teacher: null teacher_log_probs, teacher_coef or teacher_stats");
    return launch_ppo_loss(logits, ld_logits, masks, actions, old_logp, adv_raw, ret, value, ld_value, old_value, valid,
                           N, 0.f, 0.f, 0.f, hparams, dlogits, ld_dlogits, dvalue, ld_dvalue, out, stats, n_actions,
                           workspace, stream, joint != 0, old_log_probs, kl_out, teacher_log_probs, teacher_coef,
                           teacher_stats);
}

extern "C" int dc_ppo_loss_fwd_bwd_bc(const float *const logits[DC_NUM_HEADS], const int64_t ld_logits[DC_NUM_HEADS],
                                      const uint8_t *const masks[DC_NUM_HEADS], const uint8_t *const actions[DC_NUM_HEADS],
                                      const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                      const float *old_value, const uint8_t *valid, int64_t N, const double *hparams,
                                      float *const dlogits[DC_NUM_HEADS], const int64_t ld_dlogits[DC_NUM_HEADS],
                                      float *dvalue, int64_t ld_dvalue, float *out, float *stats, float *bc_stats,
                                      int32_t *n_actions, void *workspace, dc_stream_t stream) {
    DC_REQUIRE(hparams, DC_EINVAL, "dc_ppo_loss_fwd_bwd_bc: null hyper-parameter block");
    DC_REQUIRE(bc_stats, DC_EINVAL, "dc_ppo_loss_fwd_bwd_bc: null bc_stats");
    return launch_ppo_loss(logits, ld_logits, masks, actions, nullptr, adv_raw, ret, value, ld_value, old_value, valid, N,
                           0.f, 0.f, 0.f, hparams, dlogits, ld_dlogits, dvalue, ld_dvalue, out, stats, n_actions, workspace,
                           stream, false, nullptr, nullptr, nullptr, nullptr, nullptr, bc_stats);
}

extern "C" int dc_ppo_loss_fwd_bwd_dual_clip(const float *const logits[DC_NUM_HEADS],
                                             const int64_t ld_logits[DC_NUM_HEADS],
                                             const uint8_t *const masks[DC_NUM_HEADS],
                                             const uint8_t *const actions[DC_NUM_HEADS], const float *old_logp,
                                             const float *old_log_probs, const float *teacher_log_probs,
                                             const float *adv_raw, const float *ret, const float *value, int64_t ld_value,
                                             const float *old_value, const uint8_t *valid, int64_t N,
                                             const double *hparams, const double *teacher_coef, const double *dual_clip,
                                             int joint, float *const dlogits[DC_NUM_HEADS],
                                             const int64_t ld_dlogits[DC_NUM_HEADS], float *dvalue, int64_t ld_dvalue,
                                             float *out, float *stats, float *kl_out, float *teacher_stats,
                                             float *dual_clip_stats, int32_t *n_actions, void *workspace,
                                             dc_stream_t stream) {
    DC_REQUIRE(hparams, DC_EINVAL, "dc_ppo_loss_fwd_bwd_dual_clip: null hyper-parameter block");
    DC_REQUIRE(dual_clip && dual_clip_stats, DC_EINVAL, "dc_ppo_loss_fwd_bwd_dual_clip: null dual_clip or dual_clip_stats");
    // the teacher term: its rows, coefficient and statistics together, or none of them
    DC_REQUIRE((teacher_log_probs != nullptr) == (teacher_coef != nullptr) &&
                   (teacher_log_probs != nullptr) == (teacher_stats != nullptr),
               DC_EINVAL, "dc_ppo_loss_fwd_bwd_dual_clip: teacher_log_probs, teacher_coef and teacher_stats go together");
    return launch_ppo_loss(logits, ld_logits, masks, actions, old_logp, adv_raw, ret, value, ld_value, old_value, valid,
                           N, 0.f, 0.f, 0.f, hparams, dlogits, ld_dlogits, dvalue, ld_dvalue, out, stats, n_actions,
                           workspace, stream, joint != 0, old_log_probs, kl_out, teacher_log_probs, teacher_coef,
                           teacher_stats, nullptr, dual_clip, dual_clip_stats);
}
