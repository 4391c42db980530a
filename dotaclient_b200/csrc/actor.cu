// Actor-side action selection for a batch of agents in ONE launch (policy.py:23-33,169-216; caller agent.py:578-674).
//
// The reference picks an action per agent per observation with ~30 tiny torch ops: masked log-softmax of the `enum`
// head, torch.multinomial over its masked probabilities, then the same for the one or two sub-heads the chosen enum
// implies (1 -> x and y, 2 -> target_unit, 3 -> ability; 0 = no-op).  For an in-process pool of agents that is
// launch-latency work; here one thread handles one agent end to end.
//
// torch.multinomial's RNG stream cannot be reproduced on a GPU, so what is held to the oracle is the INDEX
// FUNCTION (oracle/ref_policy.py:sample_index): inverse CDF over the masked probabilities for a caller-supplied uniform
// u in [0,1) -- fp32, sequential accumulation in index order, first valid index whose cumulative mass exceeds
// u * total, falling back to the last valid index.  The log-probability of the chosen entry comes back too (it is what
// the optimizer later recomputes as old_logp, optimizer.py:386-398).  expf and this sequential normaliser round
// differently from torch's exp and sum, which can move a cumulative boundary by a few ulp: a u that close to a boundary
// may take the adjacent legal index, so the two agree only outside that band.
#include "dc_common.cuh"

namespace {

constexpr int kHeads = DC_NUM_HEADS;
__host__ __device__ constexpr int head_n(int h) { return h == 0 ? 4 : h == 1 ? 9 : h == 2 ? 9 : h == 3 ? 40 : 3; }

struct ActorPtrs {
    const float *logits[kHeads];
    int64_t ld[kHeads];
    const uint8_t *masks[kHeads];
};

// masked log-softmax without max-subtraction (policy.py:169-178) + inverse-CDF draw; returns -1 when no entry is valid
__device__ __forceinline__ int draw(const float *__restrict__ l, const uint8_t *__restrict__ m, int n, float u, float *logp) {
    float s = 0.f;
    for (int i = 0; i < n; ++i)
        if (m[i]) s += expf(l[i]);
    const float log_s = logf(s);
    float total = 0.f;
    for (int i = 0; i < n; ++i)
        if (m[i]) total += expf(l[i] - log_s);
    const float target = u * total;
    float acc = 0.f;
    int last = -1;
    for (int i = 0; i < n; ++i) {
        if (!m[i]) continue;
        last = i;
        acc += expf(l[i] - log_s);
        if (acc > target) break;
    }
    *logp = last >= 0 ? l[last] - log_s : 0.f;
    return last;
}

__global__ void __launch_bounds__(128) select_actions_kernel(ActorPtrs p, const float *__restrict__ u, int64_t A,
                                                             int32_t *__restrict__ chosen, float *__restrict__ logp) {
    const int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A) return;
    int pick[kHeads];
    float lp[kHeads];
#pragma unroll
    for (int h = 0; h < kHeads; ++h) { pick[h] = -1; lp[h] = 0.f; }
    pick[0] = draw(p.logits[0] + a * p.ld[0], p.masks[0] + a * head_n(0), head_n(0), u[a * kHeads + 0], &lp[0]);
    // policy.py:203-214: the enum decides which sub-heads are sampled
#pragma unroll
    for (int h = 1; h < kHeads; ++h) {
        const bool used = (pick[0] == 1 && (h == 1 || h == 2)) || (pick[0] == 2 && h == 3) || (pick[0] == 3 && h == 4);
        if (used) pick[h] = draw(p.logits[h] + a * p.ld[h], p.masks[h] + a * head_n(h), head_n(h), u[a * kHeads + h], &lp[h]);
    }
#pragma unroll
    for (int h = 0; h < kHeads; ++h) {
        chosen[a * kHeads + h] = pick[h];
        if (logp) logp[a * kHeads + h] = lp[h];
    }
}

}  // namespace

extern "C" int dc_select_actions(const float *const logits[DC_NUM_HEADS], const int64_t ld[DC_NUM_HEADS],
                                 const uint8_t *const masks[DC_NUM_HEADS], const float *u, int64_t A, int32_t *chosen,
                                 float *logp, dc_stream_t stream) {
    DC_REQUIRE(A > 0 && u && chosen, DC_EINVAL, "dc_select_actions: bad arguments (A=%lld)", (long long)A);
    ActorPtrs p;
    for (int h = 0; h < kHeads; ++h) {
        DC_REQUIRE(logits[h] && masks[h] && ld[h] >= head_n(h), DC_EINVAL, "dc_select_actions: head %d: null pointer or short row pitch", h);
        p.logits[h] = logits[h];
        p.ld[h] = ld[h];
        p.masks[h] = masks[h];
    }
    select_actions_kernel<<<(unsigned)((A + 127) / 128), 128, 0, dc_cu_stream(stream)>>>(p, u, A, chosen, logp);
    DC_LAUNCH_OK();
    return DC_OK;
}
