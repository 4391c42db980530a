// The value loss of K value heads (DotaOptimizer(value_heads=...)), one pass over the tokens.
//
// Per counting token t and head k, with v = value[t * ld_value + k] (the K value columns of the packed head output) and
// r = ret[t * K + k]:
//   l_k,t = (r - v)^2, or with the PPO2 clip against old_value[t * K + k] the ppo_loss.cu term and gradient
//   dvalue[t * ld_dvalue + k] = vf_coef * d l_k,t / d v / 2 / N_v     (0 on tokens that do not count)
//   value loss = vf_coef * 0.5 * sum_k mean_t l_k,t                   -> out[3], and added to out[0]
// which is ppo_loss.cu's value term for each head (same fp32 expressions, same divisor), so one head gives today's value
// loss.  The PPO kernel runs before this one with its value term off (vf_coef = 0 and no clip in its hparams block), so
// it leaves out[0] without a value loss and zero in the first value column of the gradient.
//
// Statistics (head_stats, float64 sums rounded once): the value loss of every head, its explained variance
// 1 - Var(r_k - v_k) / Var(r_k), and the explained variance of sum_k v_k against sum_k r_k (the sums in float64, rounded
// once) into stats[DC_STAT_EXPLAINED_VAR].  Like ppo_loss.cu the variance sums run on values shifted by the first
// counting token's, so constant targets give exactly zero variance (explained variance NaN).
//
// Three launches on the stream: a memset of the workspace header, a count of the tokens that count (N_v and the first
// of them; one byte per token under a valid mask, one thread without), then the loss.  The loss kernel keeps 5 float64
// sums per head and 4 for the totals in registers, reduces them per block in a fixed order into the workspace, and the last block to finish
// adds the block partials in block order: the results are bitwise reproducible.
//
// Algorithmic HBM bytes per token: value 4K + ret 4K (+ old value 4K with the clip) + valid 1 read, dvalue 4K written:
// 12K + 1 B, 16K + 1 with the clip -- 121 B at K = 10 (161 B clipped).
#include "dc_common.cuh"

namespace {

constexpr int kMax = DC_VALUE_HEADS_MAX;
constexpr int kThreads = 256;
constexpr int kMaxBlocks = 256;
// per head: value-loss sum, shifted (r - v) sum and square sum, shifted r sum and square sum; then the same four of the
// totals
constexpr int kSumVl = 0, kSumD = kMax, kSumD2 = 2 * kMax, kSumR = 3 * kMax, kSumR2 = 4 * kMax, kSumTot = 5 * kMax;
constexpr int kSums = 5 * kMax + 4;

struct Workspace {
    unsigned long long n_valid;     // N_v
    unsigned long long first_rev;   // N - (first counting token)
    unsigned int ticket;
    unsigned int pad[11];
    double part[kMaxBlocks][kSums];
};
static_assert(sizeof(Workspace) <= DC_VALUE_HEADS_WORKSPACE_BYTES, "DC_VALUE_HEADS_WORKSPACE_BYTES is too small");

__global__ void __launch_bounds__(kThreads) value_heads_count_kernel(const uint8_t *__restrict__ valid, int64_t N,
                                                                      Workspace *ws) {
    if (!valid) {                   // every token counts, the first is token 0
        if (blockIdx.x == 0 && threadIdx.x == 0) ws->n_valid = ws->first_rev = (unsigned long long)N;
        return;
    }
    unsigned long long n = 0, first = 0;
    for (int64_t t = blockIdx.x * (int64_t)kThreads + threadIdx.x; t < N; t += (int64_t)gridDim.x * kThreads) {
        if (valid[t]) {
            ++n;
            first = max(first, (unsigned long long)(N - t));
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        n += __shfl_xor_sync(0xffffffffu, n, o);
        first = max(first, __shfl_xor_sync(0xffffffffu, first, o));
    }
    if ((threadIdx.x & 31) == 0 && n) {
        atomicAdd(&ws->n_valid, n);
        atomicMax(&ws->first_rev, first);
    }
}

__device__ __forceinline__ double explained_variance(double n, double s_d, double s_d2, double s_r, double s_r2) {
    const double md = s_d / n, mr = s_r / n;
    const double var_d = s_d2 / n - md * md, var_r = s_r2 / n - mr * mr;
    return var_r > 0.0 ? 1.0 - var_d / var_r : (double)__int_as_float(0x7fc00000);
}

__global__ void __launch_bounds__(kThreads) value_heads_loss_kernel(
    const float *__restrict__ value, int64_t ld_v, const float *__restrict__ ret, const float *__restrict__ old_value,
    const uint8_t *__restrict__ valid, int64_t N, int K, const double *__restrict__ hparams, float *__restrict__ dvalue,
    int64_t ld_dv, float *__restrict__ out, float *__restrict__ stats, float *__restrict__ head_stats, Workspace *ws) {
    __shared__ double s_part[kThreads / 32][kSums];
    __shared__ bool s_last;
    const float vf_coef = (float)hparams[DC_HP_VF_COEF];
    const float value_clip = (float)hparams[DC_HP_VALUE_CLIP];
    const bool clip_value = old_value != nullptr && value_clip > 0.f;
    const unsigned long long n_valid = *((volatile unsigned long long *)&ws->n_valid);
    const float div_v = (float)n_valid;
    // the shifts: the first counting token's targets and residuals, per head and of the totals
    float sh_r[kMax], sh_d[kMax], sh_rt = 0.f, sh_dt = 0.f;
    {
        const int64_t tf = n_valid ? N - (int64_t)ws->first_rev : 0;
        double vt = 0.0, rt = 0.0;
#pragma unroll
        for (int k = 0; k < kMax; ++k) {
            sh_r[k] = sh_d[k] = 0.f;
            if (k < K && n_valid) {
                const float v = value[tf * ld_v + k], r = ret[tf * K + k];
                sh_r[k] = r;
                sh_d[k] = r - v;
                vt += (double)v;
                rt += (double)r;
            }
        }
        sh_rt = (float)rt;
        sh_dt = sh_rt - (float)vt;
    }
    double acc[kSums];
#pragma unroll
    for (int i = 0; i < kSums; ++i) acc[i] = 0.0;
    for (int64_t t = blockIdx.x * (int64_t)kThreads + threadIdx.x; t < N; t += (int64_t)gridDim.x * kThreads) {
        if (valid && !valid[t]) {
#pragma unroll
            for (int k = 0; k < kMax; ++k)
                if (k < K) dvalue[t * ld_dv + k] = 0.f;
            continue;
        }
        double vt = 0.0, rt = 0.0;
#pragma unroll
        for (int k = 0; k < kMax; ++k) {
            if (k < K) {
                const float v = value[t * ld_v + k], r = ret[t * K + k];
                const float d = r - v;
                float g = v - r, vl;
                if (clip_value) {       // ppo_loss.cu's PPO2 term and its autograd gradient
                    const float vo = old_value[t * K + k];
                    const float dv = v - vo;
                    const float dc = (vo + fminf(fmaxf(dv, -value_clip), value_clip)) - r;
                    const float l1 = d * d, l2 = dc * dc;
                    vl = fmaxf(l1, l2);
                    const float w1 = l1 > l2 ? 1.f : (l1 == l2 ? 0.5f : 0.f);
                    const float w2 = l2 > l1 ? 1.f : (l1 == l2 ? 0.5f : 0.f);
                    const float in_range = (dv >= -value_clip && dv <= value_clip) ? 1.f : 0.f;
                    g = w1 * g + w2 * in_range * dc;
                } else {
                    vl = d * d;
                }
                dvalue[t * ld_dv + k] = vf_coef > 0.f ? vf_coef * g / div_v : 0.f;
                const double ds = (double)(d - sh_d[k]), rs = (double)(r - sh_r[k]);
                acc[kSumVl + k] += (double)vl;
                acc[kSumD + k] += ds;
                acc[kSumD2 + k] += ds * ds;
                acc[kSumR + k] += rs;
                acc[kSumR2 + k] += rs * rs;
                vt += (double)v;
                rt += (double)r;
            }
        }
        const float rf = (float)rt;
        const double ds = (double)((rf - (float)vt) - sh_dt), rs = (double)(rf - sh_rt);
        acc[kSumTot + 0] += ds;
        acc[kSumTot + 1] += ds * ds;
        acc[kSumTot + 2] += rs;
        acc[kSumTot + 3] += rs * rs;
    }
    // block partials in a fixed order: warp sums, then the warps in order
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < kSums; ++i) {
        const double s = dc_warp_sum(acc[i]);
        if (lane == 0) s_part[warp][i] = s;
    }
    __syncthreads();
    if (threadIdx.x < kSums) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) s += s_part[w][threadIdx.x];
        ws->part[blockIdx.x][threadIdx.x] = s;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&ws->ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    __shared__ double s_tot[kSums];
    if (threadIdx.x < kSums) {
        double s = 0.0;
        for (unsigned b = 0; b < gridDim.x; ++b) s += ((volatile double *)ws->part[b])[threadIdx.x];
        s_tot[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const double n = (double)n_valid;
    double vl_all = 0.0;
    for (int k = 0; k < K; ++k) {
        vl_all += s_tot[kSumVl + k];
        head_stats[k] = vf_coef > 0.f ? vf_coef * (0.5f * (float)(s_tot[kSumVl + k] / n)) : 0.f;
        head_stats[kMax + k] = (float)explained_variance(n, s_tot[kSumD + k], s_tot[kSumD2 + k], s_tot[kSumR + k],
                                                         s_tot[kSumR2 + k]);
    }
    for (int k = K; k < kMax; ++k) head_stats[k] = head_stats[kMax + k] = 0.f;
    const float v_loss = vf_coef > 0.f ? vf_coef * (0.5f * (float)(vl_all / n)) : 0.f;
    out[3] = v_loss;
    out[0] = out[0] + v_loss;
    if (stats)
        stats[DC_STAT_EXPLAINED_VAR] = (float)explained_variance(n, s_tot[kSumTot], s_tot[kSumTot + 1],
                                                                 s_tot[kSumTot + 2], s_tot[kSumTot + 3]);
}

}  // namespace

extern "C" int dc_value_heads_loss(const float *value, int64_t ld_value, const float *ret, const float *old_value,
                                   const uint8_t *valid, int64_t N, int K, const double *hparams, float *dvalue,
                                   int64_t ld_dvalue, float *out, float *stats, float *head_stats, void *workspace,
                                   dc_stream_t stream) {
    DC_REQUIRE(N > 0, DC_EINVAL, "dc_value_heads_loss: N=%lld", (long long)N);
    DC_REQUIRE(K >= 1 && K <= DC_VALUE_HEADS_MAX, DC_EINVAL, "dc_value_heads_loss: K=%d value heads (1 .. %d)", K,
               DC_VALUE_HEADS_MAX);
    DC_REQUIRE(ld_value >= K && ld_dvalue >= K, DC_EINVAL, "dc_value_heads_loss: pitches %lld / %lld below K=%d",
               (long long)ld_value, (long long)ld_dvalue, K);
    DC_REQUIRE(value && ret && hparams && dvalue && out && head_stats && workspace, DC_EINVAL,
               "dc_value_heads_loss: null pointer");
    const cudaStream_t st = dc_cu_stream(stream);
    Workspace *ws = static_cast<Workspace *>(workspace);
    DC_CUDA(cudaMemsetAsync(ws, 0, offsetof(Workspace, part), st));
    const int64_t want = (N + kThreads - 1) / kThreads;
    const int blocks = (int)(want < kMaxBlocks ? want : kMaxBlocks);
    value_heads_count_kernel<<<valid ? blocks : 1, kThreads, 0, st>>>(valid, N, ws);
    DC_LAUNCH_OK();
    value_heads_loss_kernel<<<blocks, kThreads, 0, st>>>(value, ld_value, ret, old_value, valid, N, K, hparams, dvalue,
                                                          ld_dvalue, out, stats, head_stats, ws);
    DC_LAUNCH_OK();
    return DC_OK;
}
