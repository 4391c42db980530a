// Gradient finish on one flat fp32 buffer: count-divide, grad-norm metrics, global-norm clip, Adam.
//
// Replaces (TimZaman/dotaclient):
//   distributed.py:36-57   per-parameter has-grad count + grad /= count (after ONE flat all-reduce
//                          instead of the reference's 68 gloo collectives)
//   optimizer.py:674-676   mean_gradient_norm (unclipped / clipped), clip_grad_norm_(params, 0.5)
//   optimizer.py:667,678   NaN guards (device flag; parameters are left untouched when it trips)
//   optimizer.py:681       torch.optim.Adam.step (betas .9/.999, eps 1e-8, no weight decay; per-parameter
//                          step counters: a parameter without a gradient is skipped entirely)
//
// Three small launches over <= 11 MB: (A) divide + per-parameter sum of squares (float64 atomics),
// (B) clip coefficient + Adam in one elementwise sweep, (C) step counters + metrics.
// dc_grad_finish_dev reads lr and the clip norm from the device hyper-parameter block (DC_HPARAM_SLOTS) in (B).
// HBM-bound elementwise work: 4 B read + 4 B written per element in A, 16 B read + 12 B written in B.
// dc_grad_finish_kl also reads the all-reduced (sum_t KL_t, T_a) behind the flags in (B): above hparams[DC_HP_KL_STOP] the
// step is skipped like the NaN path (no parameter, moment or counter changes), and (C) reports the KL and the skip.
#include "dc_common.cuh"

namespace {

constexpr int kMaxSeg = 96;
constexpr int kThreads = 256;

struct FinishWs {
    double sumsq[kMaxSeg];
    float clip_coef;
    int nan_flag;
    float mean_norm, total_norm;
    float kl;             // dc_grad_finish_kl: the all-ranks KL
    int kl_skip;          // dc_grad_finish_kl: 1 when the KL exceeded the limit and the step was skipped
};
static_assert(sizeof(FinishWs) <= DC_FINISH_WORKSPACE_BYTES, "finish workspace too small");

__global__ void grad_flags_kernel(float *flat_grad, int64_t total, const int32_t *seg_head, int n_seg,
                                  const int32_t *n_actions) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_seg) return;
    const int h = seg_head[p];
    flat_grad[total + p] = (h < 0 || n_actions[h] > 0) ? 1.0f : 0.0f;
}

__global__ void __launch_bounds__(kThreads) grad_sumsq_kernel(float *__restrict__ g, const int64_t *__restrict__ seg_lo,
                                                              const int64_t *__restrict__ seg_hi, int n_seg, int64_t total,
                                                              FinishWs *ws) {
    __shared__ double s_red[kThreads / 32];
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    for (int p = 0; p < n_seg; ++p) {
        const float count = g[total + p];
        if (!(count > 0.f)) continue;                    // nobody has a gradient: skip (distributed.py:40-42)
        const int64_t lo = seg_lo[p], hi = seg_hi[p];
        double acc = 0.0;
        for (int64_t i = lo + (int64_t)blockIdx.x * kThreads + threadIdx.x; i < hi; i += stride) {
            float v = g[i];
            if (count != 1.f) { v = __fdiv_rn(v, count); g[i] = v; }   // grad_data /= has_grad_count
            acc += (double)v * (double)v;
        }
        acc = dc_warp_sum(acc);
        __syncthreads();
        if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            double r = 0.0;
            for (int w = 0; w < kThreads / 32; ++w) r += s_red[w];
            if (r != 0.0) atomicAdd(&ws->sumsq[p], r);
        }
    }
}

__device__ __forceinline__ void finish_scalars(const float *g_tail, int n_seg, const FinishWs *ws, const float *loss_out,
                                               float max_norm, float &coef, int &nan_flag, float &mean_norm,
                                               float &total_norm) {
    double tot = 0.0, mean = 0.0;
    int n_has = 0;
    for (int p = 0; p < n_seg; ++p) {
        if (g_tail[p] > 0.f) {
            const double s = ws->sumsq[p];
            tot += s;
            mean += (double)(float)sqrt(s);     // per-tensor fp32 norms, then their mean (optimizer.py:691-695)
            ++n_has;
        }
    }
    total_norm = (float)sqrt(tot);
    mean_norm = n_has ? (float)(mean / n_has) : 0.f;
    const float c = max_norm / (total_norm + 1e-6f);     // torch.nn.utils.clip_grad_norm_
    coef = c < 1.0f ? c : 1.0f;
    nan_flag = (loss_out && isnan(loss_out[0])) || isnan(mean_norm);
}

__global__ void __launch_bounds__(kThreads) adam_kernel(float *__restrict__ param, float *__restrict__ g,
                                                        float *__restrict__ m, float *__restrict__ v,
                                                        const int32_t *__restrict__ steps,
                                                        const int64_t *__restrict__ seg_lo,
                                                        const int64_t *__restrict__ seg_hi, int n_seg, int64_t total,
                                                        double lr, double beta1_d, double beta2_d, double eps_d,
                                                        float max_norm, const double *__restrict__ hparams,
                                                        const float *__restrict__ loss_out, FinishWs *ws,
                                                        const float *__restrict__ kl) {
    __shared__ float s_coef;
    __shared__ int s_nan;
    if (hparams) {                                       // the device block overrides the scalar arguments
        lr = hparams[DC_HP_LR];
        max_norm = (float)hparams[DC_HP_MAX_GRAD_NORM];
    }
    if (threadIdx.x == 0) {
        float coef, mn, tn;
        int nf;
        finish_scalars(g + total, n_seg, ws, loss_out, max_norm, coef, nf, mn, tn);
        s_coef = coef;
        s_nan = nf;
        if (kl) {    // KL early stop: kl = (sum_t KL_t, T_a) summed over the ranks; a limit <= 0 (or no block) is none
            const double n_a = (double)kl[1], k = n_a > 0.0 ? (double)kl[0] / n_a : 0.0;
            const double limit = hparams ? hparams[DC_HP_KL_STOP] : 0.0;
            const int skip = limit > 0.0 && k > limit;
            s_nan |= skip;
            if (blockIdx.x == 0) { ws->kl = (float)k; ws->kl_skip = skip; }
        }
        if (blockIdx.x == 0) { ws->clip_coef = coef; ws->nan_flag = nf; ws->mean_norm = mn; ws->total_norm = tn; }
    }
    __syncthreads();
    if (s_nan) return;                                   // ValueError path (or a KL skip): leave parameters untouched
    const float coef = s_coef;
    // 1 - beta rounded from float64, as torch receives it (a Python float): 1 - (float)0.999 in fp32 would be 1.3e-5
    // off 0.001 and move the first updates of a fresh state by ~6e-6 relative
    const float beta2 = (float)beta2_d, eps = (float)eps_d;
    const float one_m_beta1 = (float)(1.0 - beta1_d), one_m_beta2 = (float)(1.0 - beta2_d);
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    // per-tensor scalars once per block (thread p -> tensor p): the float64 pow() calls are ~100 instructions each and were
    // being repeated by every thread for every tensor (0.10 ms for a 1 MB parameter set)
    __shared__ float s_bc2[kMaxSeg], s_step[kMaxSeg];
    for (int p = threadIdx.x; p < n_seg; p += kThreads) {
        // torch computes the bias corrections as Python floats (float64) and folds them into fp32 scalars.
        const int step = steps[p] + 1;
        const double bc1 = 1.0 - pow(beta1_d, (double)step);
        s_bc2[p] = (float)sqrt(1.0 - pow(beta2_d, (double)step));
        s_step[p] = (float)(lr / bc1);
    }
    __syncthreads();
    for (int p = 0; p < n_seg; ++p) {
        if (!(g[total + p] > 0.f)) continue;             // .grad is None -> Adam skips the tensor
        const float bc2_sqrt = s_bc2[p], step_size = s_step[p];
        const int64_t lo = seg_lo[p], hi = seg_hi[p];
        for (int64_t i = lo + (int64_t)blockIdx.x * kThreads + threadIdx.x; i < hi; i += stride) {
            const float gi = g[i] * coef;
            g[i] = gi;                                   // clipped gradient stays visible in .grad
            const float mi = m[i] + (gi - m[i]) * one_m_beta1;             // exp_avg.lerp_(grad, 1-beta1)
            const float vi = v[i] * beta2 + one_m_beta2 * gi * gi;         // mul_(beta2).addcmul_(g, g, 1-beta2)
            m[i] = mi;
            v[i] = vi;
            const float denom = sqrtf(vi) / bc2_sqrt + eps;
            param[i] = param[i] - step_size * (mi / denom);                // addcdiv_(exp_avg, denom, -step_size)
        }
    }
}

__global__ void finish_tail_kernel(int32_t *steps, const float *g_tail, int n_seg, const FinishWs *ws, float *metrics,
                                   bool kl) {
    const int p = threadIdx.x;
    const int nan_flag = ws->nan_flag;
    const int skip = kl ? ws->kl_skip : 0;
    if (p < n_seg && !nan_flag && !skip && g_tail[p] > 0.f) steps[p] += 1;
    if (p == 0) {
        metrics[0] = ws->mean_norm;                      // grad_norm 'unclipped'
        metrics[1] = ws->mean_norm * ws->clip_coef;      // grad_norm 'clipped'
        metrics[2] = ws->total_norm;
        metrics[3] = nan_flag ? 1.0f : 0.0f;
        if (kl) {
            metrics[4] = ws->kl;
            metrics[5] = skip ? 1.0f : 0.0f;
        }
    }
}

int launch_finish(float *flat_param, float *flat_grad, float *exp_avg, float *exp_avg_sq, int32_t *steps,
                  const int64_t *seg_lo, const int64_t *seg_hi, int n_seg, int64_t total, double lr, double beta1, double beta2,
                  double adam_eps, double max_norm, const double *hparams, const float *loss_out, float *metrics,
                  void *workspace, dc_stream_t stream, bool kl = false) {
    DC_REQUIRE(flat_param && flat_grad && exp_avg && exp_avg_sq && steps && seg_lo && seg_hi && metrics && workspace,
               DC_EINVAL, "dc_grad_finish: null pointer");
    DC_REQUIRE(n_seg > 0 && n_seg <= kMaxSeg && total > 0, DC_EINVAL, "dc_grad_finish: n_seg=%d total=%lld", n_seg,
               (long long)total);
    cudaStream_t st = dc_cu_stream(stream);
    FinishWs *ws = reinterpret_cast<FinishWs *>(workspace);
    DC_CUDA(cudaMemsetAsync(ws, 0, sizeof(FinishWs), st));
    const int blocks = 2 * dc_sm_count();
    grad_sumsq_kernel<<<blocks, kThreads, 0, st>>>(flat_grad, seg_lo, seg_hi, n_seg, total, ws);
    DC_LAUNCH_OK();
    adam_kernel<<<blocks, kThreads, 0, st>>>(flat_param, flat_grad, exp_avg, exp_avg_sq, steps, seg_lo, seg_hi, n_seg, total,
                                             lr, beta1, beta2, adam_eps, (float)max_norm, hparams, loss_out, ws,
                                             kl ? flat_grad + total + n_seg : nullptr);
    DC_LAUNCH_OK();
    finish_tail_kernel<<<1, kMaxSeg, 0, st>>>(steps, flat_grad + total, n_seg, ws, metrics, kl);
    DC_LAUNCH_OK();
    return DC_OK;
}

}  // namespace

extern "C" int dc_grad_flags(float *flat_grad, int64_t total, const int32_t *seg_head, int n_seg,
                             const int32_t *n_actions, dc_stream_t stream) {
    DC_REQUIRE(flat_grad && seg_head && n_actions && n_seg > 0 && n_seg <= kMaxSeg && total > 0, DC_EINVAL,
               "dc_grad_flags: bad arguments (n_seg=%d)", n_seg);
    grad_flags_kernel<<<1, 128, 0, dc_cu_stream(stream)>>>(flat_grad, total, seg_head, n_seg, n_actions);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_grad_finish(float *flat_param, float *flat_grad, float *exp_avg, float *exp_avg_sq, int32_t *steps,
                              const int64_t *seg_lo, const int64_t *seg_hi, const int32_t *seg_head, int n_seg, int64_t total,
                              double lr,
                              double beta1, double beta2, double adam_eps, double max_norm, const float *loss_out,
                              float *metrics, void *workspace, dc_stream_t stream) {
    (void)seg_head;
    return launch_finish(flat_param, flat_grad, exp_avg, exp_avg_sq, steps, seg_lo, seg_hi, n_seg, total, lr, beta1, beta2,
                         adam_eps, max_norm, nullptr, loss_out, metrics, workspace, stream);
}

extern "C" int dc_grad_finish_dev(float *flat_param, float *flat_grad, float *exp_avg, float *exp_avg_sq, int32_t *steps,
                                  const int64_t *seg_lo, const int64_t *seg_hi, const int32_t *seg_head, int n_seg,
                                  int64_t total, const double *hparams, double beta1, double beta2, double adam_eps,
                                  const float *loss_out, float *metrics, void *workspace, dc_stream_t stream) {
    (void)seg_head;
    DC_REQUIRE(hparams, DC_EINVAL, "dc_grad_finish_dev: null hyper-parameter block");
    return launch_finish(flat_param, flat_grad, exp_avg, exp_avg_sq, steps, seg_lo, seg_hi, n_seg, total, 0.0, beta1, beta2,
                         adam_eps, 0.0, hparams, loss_out, metrics, workspace, stream);
}

extern "C" int dc_grad_finish_kl(float *flat_param, float *flat_grad, float *exp_avg, float *exp_avg_sq, int32_t *steps,
                                 const int64_t *seg_lo, const int64_t *seg_hi, const int32_t *seg_head, int n_seg,
                                 int64_t total, const double *hparams, double beta1, double beta2, double adam_eps,
                                 const float *loss_out, float *metrics, void *workspace, dc_stream_t stream) {
    (void)seg_head;
    DC_REQUIRE(hparams, DC_EINVAL, "dc_grad_finish_kl: null hyper-parameter block");
    return launch_finish(flat_param, flat_grad, exp_avg, exp_avg_sq, steps, seg_lo, seg_hi, n_seg, total, 0.0, beta1, beta2,
                         adam_eps, 0.0, hparams, loss_out, metrics, workspace, stream, true);
}
