// The state refresh between PPO epochs (DotaOptimizer(recompute_states=True)): after a no-grad rollout-major forward over a
// time block [t0, t0 + T) of every rollout, copy each layer's recomputed recurrent state at the chunk starts that fall in the
// block into the training batch, in place, and accumulate how far the states moved.
//
//   dc_refresh_states   one warp per (destination d, layer l): reads state-buffer row (step[d] - t0) * R + rollout[d] of
//                       layer l ([T + 1, R, H], and the LSTM's c buffer), writes it over the batch's copy -- h0[l, slot]
//                       for slot < B, or the H-wide slice l of reset-table row slot - B ([K, B, L*H]) -- and writes the
//                       float64 sums (sum (new - old)^2, sum old^2) of its H (or 2H) floats to partial[d * L + l].  Then
//                       one CTA adds the partials, in index order per thread and a fixed tree over the CTA, to acc[2].
//                       No atomics: two calls on the same data give the same bits.
//
// Accesses are 16 bytes (H is a multiple of 32, so a lane moves H / 128 float4 per array).  Algorithmic HBM bytes per
// state float replaced: 4 read from the state buffer, 4 read and 4 written in the batch = 12 B, plus 16 B of partials per
// (destination, layer) and the 24 B of its (step, rollout, slot) index.
#include "dc_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kReduceThreads = 1024;

struct LayerPtrs {
    const float *h[DC_REFRESH_MAX_LAYERS];
    const float *c[DC_REFRESH_MAX_LAYERS];
};

__device__ __forceinline__ void move_row(const float4 *__restrict__ src, float4 *__restrict__ dst, int n4, int lane,
                                         double &d2, double &o2) {
    for (int i = lane; i < n4; i += 32) {
        const float4 n = src[i], o = dst[i];
        dst[i] = n;
        const double dx = (double)n.x - (double)o.x, dy = (double)n.y - (double)o.y;
        const double dz = (double)n.z - (double)o.z, dw = (double)n.w - (double)o.w;
        d2 = __dadd_rn(d2, __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)),
                                      __dadd_rn(__dmul_rn(dz, dz), __dmul_rn(dw, dw))));
        o2 = __dadd_rn(o2, __dadd_rn(__dadd_rn(__dmul_rn((double)o.x, (double)o.x), __dmul_rn((double)o.y, (double)o.y)),
                                      __dadd_rn(__dmul_rn((double)o.z, (double)o.z), __dmul_rn((double)o.w, (double)o.w))));
    }
}

__global__ void __launch_bounds__(kThreads) refresh_states_kernel(
    const __grid_constant__ LayerPtrs bufs, int n_layers, int H, int64_t R, int64_t t0, const int64_t *__restrict__ step,
    const int64_t *__restrict__ rollout, const int64_t *__restrict__ slot, int64_t n, int64_t B, float *__restrict__ h0,
    float *__restrict__ c0, float *__restrict__ reset_h, float *__restrict__ reset_c, double2 *__restrict__ partial) {
    const int64_t w = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n * n_layers) return;                                  // warp-uniform
    const int64_t d = w / n_layers;
    const int l = (int)(w - d * n_layers);
    const int64_t src_row = (step[d] - t0) * R + rollout[d];
    const int64_t s = slot[d];
    const int64_t dst_off = s < B ? ((int64_t)l * B + s) * H : ((s - B) * n_layers + l) * (int64_t)H;
    const int n4 = H >> 2;
    double d2 = 0.0, o2 = 0.0;
    move_row(reinterpret_cast<const float4 *>(bufs.h[l] + src_row * H),
             reinterpret_cast<float4 *>((s < B ? h0 : reset_h) + dst_off), n4, lane, d2, o2);
    if (bufs.c[l] != nullptr)
        move_row(reinterpret_cast<const float4 *>(bufs.c[l] + src_row * H),
                 reinterpret_cast<float4 *>((s < B ? c0 : reset_c) + dst_off), n4, lane, d2, o2);
    d2 = dc_warp_sum(d2);
    o2 = dc_warp_sum(o2);
    if (lane == 0) partial[w] = make_double2(d2, o2);
}

__global__ void __launch_bounds__(kReduceThreads) refresh_drift_reduce_kernel(const double2 *__restrict__ partial,
                                                                               int64_t n, double *__restrict__ acc) {
    __shared__ double s_red[2][kReduceThreads / 32];
    double a = 0.0, b = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += kReduceThreads) {     // stage 1: a fixed strided slice per thread
        a = __dadd_rn(a, partial[i].x);
        b = __dadd_rn(b, partial[i].y);
    }
    a = dc_warp_sum(a);                                              // stage 2: a fixed tree over the CTA
    b = dc_warp_sum(b);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        s_red[0][warp] = a;
        s_red[1][warp] = b;
    }
    __syncthreads();
    if (warp == 0) {
        a = dc_warp_sum(s_red[0][lane]);
        b = dc_warp_sum(s_red[1][lane]);
        if (lane == 0) {
            acc[0] = __dadd_rn(acc[0], a);
            acc[1] = __dadd_rn(acc[1], b);
        }
    }
}
static_assert(kReduceThreads / 32 == 32, "the second stage reduces one value per warp in one warp");

bool aligned16(const void *p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

}  // namespace

extern "C" int dc_refresh_states(int n_layers, int H, const float *const *h_bufs, const float *const *c_bufs, int64_t R,
                                 int64_t t0, const int64_t *step, const int64_t *rollout, const int64_t *slot, int64_t n,
                                 int64_t B, int64_t K, float *h0, float *c0, float *reset_h, float *reset_c,
                                 double *partial, double *acc, dc_stream_t stream) {
    DC_REQUIRE(n_layers >= 1 && n_layers <= DC_REFRESH_MAX_LAYERS, DC_EINVAL,
               "dc_refresh_states: n_layers=%d outside [1, %d]", n_layers, DC_REFRESH_MAX_LAYERS);
    DC_REQUIRE(H >= 32 && H % 32 == 0, DC_EINVAL, "dc_refresh_states: H=%d must be a positive multiple of 32", H);
    DC_REQUIRE(R >= 1 && B >= 1 && K >= 0 && n >= 0 && t0 >= 0, DC_EINVAL,
               "dc_refresh_states: R=%lld B=%lld K=%lld n=%lld t0=%lld", (long long)R, (long long)B, (long long)K,
               (long long)n, (long long)t0);
    DC_REQUIRE(acc, DC_EINVAL, "dc_refresh_states: null acc");
    if (n == 0) return DC_OK;
    DC_REQUIRE(h_bufs && step && rollout && slot && h0 && partial, DC_EINVAL, "dc_refresh_states: null pointer");
    DC_REQUIRE((c_bufs == nullptr) == (c0 == nullptr), DC_EINVAL,
               "dc_refresh_states: c_bufs and c0 must both be given (LSTM) or both be null (GRU)");
    DC_REQUIRE(K == 0 || (reset_h && (c0 == nullptr) == (reset_c == nullptr)), DC_EINVAL,
               "dc_refresh_states: K=%lld needs reset_h (and reset_c exactly for the LSTM)", (long long)K);
    DC_REQUIRE(n <= INT64_MAX / n_layers && n * n_layers <= (int64_t)INT32_MAX * (kThreads / 32), DC_EINVAL,
               "dc_refresh_states: n=%lld destinations is too many", (long long)n);
    LayerPtrs p;
    for (int l = 0; l < DC_REFRESH_MAX_LAYERS; ++l) {
        p.h[l] = l < n_layers ? h_bufs[l] : nullptr;
        p.c[l] = l < n_layers && c_bufs ? c_bufs[l] : nullptr;
    }
    for (int l = 0; l < n_layers; ++l)
        DC_REQUIRE(p.h[l] && aligned16(p.h[l]) && (!c_bufs || (p.c[l] && aligned16(p.c[l]))), DC_EINVAL,
                   "dc_refresh_states: layer %d's state buffer is null or not 16-byte aligned", l);
    DC_REQUIRE(aligned16(partial), DC_EINVAL, "dc_refresh_states: partial must be 16-byte aligned");
    DC_REQUIRE(aligned16(h0) && (!c0 || aligned16(c0)) && (!reset_h || aligned16(reset_h)) &&
                   (!reset_c || aligned16(reset_c)),
               DC_EINVAL, "dc_refresh_states: the batch's state tensors must be 16-byte aligned");
    const int64_t warps = n * n_layers;
    const int64_t blocks = (warps * 32 + kThreads - 1) / kThreads;
    refresh_states_kernel<<<(unsigned)blocks, kThreads, 0, dc_cu_stream(stream)>>>(
        p, n_layers, H, R, t0, step, rollout, slot, n, B, h0, c0, reset_h, reset_c, reinterpret_cast<double2 *>(partial));
    DC_LAUNCH_OK();
    refresh_drift_reduce_kernel<<<1, kReduceThreads, 0, dc_cu_stream(stream)>>>(reinterpret_cast<const double2 *>(partial),
                                                                                warps, acc);
    DC_LAUNCH_OK();
    return DC_OK;
}
