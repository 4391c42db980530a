// Value normalisation (PopArt, van Hasselt et al. 2016): the three small kernels around the critic's running statistics.
//
//   dc_value_norm_stats     count, sum and sum of squares (float64) of the raw value targets that the value loss averages
//                           over: ONE CTA, a fixed-order two-stage reduction (per-thread strided sums, then a fixed tree
//                           over the CTA), no atomics, so two calls on the same data give the same bits.  It runs once per
//                           prepared batch; 4 bytes per token (+1 for the valid mask).
//   dc_value_denorm         out = fp32(mu + sigma * v) in float64 from a strided column (the value column of the packed
//                           head GEMM): what experience prep reads from a normalised head.  8 bytes per token (4 at pitch).
//   dc_value_head_rescale   the POP step on the value head's weight and bias, in place: the unnormalised output
//                           sigma * v + mu is preserved across a change of (mu, sigma).
// Every operation is written with explicit round-to-nearest intrinsics, so no multiply-add is contracted and the results
// are those of numpy's float64 expressions in the same order.
#include <math.h>
#include "dc_common.cuh"

namespace {

constexpr int kStatsThreads = 1024;

__global__ void __launch_bounds__(kStatsThreads) value_norm_stats_kernel(const float *__restrict__ x,
                                                                          const uint8_t *__restrict__ valid, int64_t N,
                                                                          double *__restrict__ out) {
    __shared__ double s_red[3][kStatsThreads / 32];
    double n = 0.0, s1 = 0.0, s2 = 0.0;
    for (int64_t i = threadIdx.x; i < N; i += kStatsThreads) {     // stage 1: a fixed strided slice per thread
        if (valid != nullptr && valid[i] == 0) continue;
        const double v = (double)x[i];
        n = __dadd_rn(n, 1.0);
        s1 = __dadd_rn(s1, v);
        s2 = __dadd_rn(s2, __dmul_rn(v, v));
    }
    n = dc_warp_sum(n);                                              // stage 2: a fixed tree over the CTA
    s1 = dc_warp_sum(s1);
    s2 = dc_warp_sum(s2);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        s_red[0][warp] = n;
        s_red[1][warp] = s1;
        s_red[2][warp] = s2;
    }
    __syncthreads();
    if (warp == 0) {
        n = s_red[0][lane];
        s1 = s_red[1][lane];
        s2 = s_red[2][lane];
        n = dc_warp_sum(n);
        s1 = dc_warp_sum(s1);
        s2 = dc_warp_sum(s2);
        if (lane == 0) {
            out[0] = n;
            out[1] = s1;
            out[2] = s2;
        }
    }
}
static_assert(kStatsThreads / 32 == 32, "the second stage reduces one value per warp in one warp");

__global__ void value_denorm_kernel(const float *__restrict__ v, int64_t ld_v, int64_t N, double mu, double sigma,
                                    float *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) out[i] = (float)__dadd_rn(mu, __dmul_rn(sigma, (double)v[i * ld_v]));
}

__global__ void value_head_rescale_kernel(float *__restrict__ w, int64_t n, float *__restrict__ b, double mu_old,
                                          double sigma_old, double mu_new, double sigma_new) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) w[i] = (float)__ddiv_rn(__dmul_rn((double)w[i], sigma_old), sigma_new);        // W sigma_old / sigma_new
    if (i == 0) {                                               // (sigma_old b + mu_old - mu_new) / sigma_new
        const double num = __dsub_rn(__dadd_rn(__dmul_rn(sigma_old, (double)b[0]), mu_old), mu_new);
        b[0] = (float)__ddiv_rn(num, sigma_new);
    }
}

bool positive_finite(double x) { return x > 0.0 && isfinite(x); }

}  // namespace

extern "C" int dc_value_norm_stats(const float *x, const uint8_t *valid, int64_t N, double *out, dc_stream_t stream) {
    DC_REQUIRE(N >= 0, DC_EINVAL, "dc_value_norm_stats: N=%lld", (long long)N);
    DC_REQUIRE(out && (x || N == 0), DC_EINVAL, "dc_value_norm_stats: null pointer");
    value_norm_stats_kernel<<<1, kStatsThreads, 0, dc_cu_stream(stream)>>>(x, valid, N, out);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_value_denorm(const float *v, int64_t ld_v, int64_t N, double mu, double sigma, float *out,
                               dc_stream_t stream) {
    DC_REQUIRE(N >= 0, DC_EINVAL, "dc_value_denorm: N=%lld", (long long)N);
    DC_REQUIRE(ld_v >= 1, DC_EINVAL, "dc_value_denorm: ld_v=%lld", (long long)ld_v);
    DC_REQUIRE(positive_finite(sigma) && isfinite(mu), DC_EINVAL, "dc_value_denorm: mu=%g sigma=%g", mu, sigma);
    DC_REQUIRE((v && out) || N == 0, DC_EINVAL, "dc_value_denorm: null pointer");
    if (N == 0) return DC_OK;
    const int threads = 256;
    value_denorm_kernel<<<(unsigned)((N + threads - 1) / threads), threads, 0, dc_cu_stream(stream)>>>(v, ld_v, N, mu, sigma,
                                                                                                       out);
    DC_LAUNCH_OK();
    return DC_OK;
}

extern "C" int dc_value_head_rescale(float *w, int64_t n, float *b, double mu_old, double sigma_old, double mu_new,
                                     double sigma_new, dc_stream_t stream) {
    DC_REQUIRE(n >= 1, DC_EINVAL, "dc_value_head_rescale: n=%lld", (long long)n);
    DC_REQUIRE(w && b, DC_EINVAL, "dc_value_head_rescale: null pointer");
    DC_REQUIRE(positive_finite(sigma_old) && positive_finite(sigma_new) && isfinite(mu_old) && isfinite(mu_new), DC_EINVAL,
               "dc_value_head_rescale: statistics (%g, %g) -> (%g, %g)", mu_old, sigma_old, mu_new, sigma_new);
    const int threads = 256;
    value_head_rescale_kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, dc_cu_stream(stream)>>>(
        w, n, b, mu_old, sigma_old, mu_new, sigma_new);
    DC_LAUNCH_OK();
    return DC_OK;
}
