// Entry points of the recurrent core (dc_rnn_seq_fwd / dc_rnn_seq_bwd, and the _reset variants with recurrent-state resets
// inside a sequence) and kernel dispatch.
//
// Replaces the time loop inside nn.GRU / nn.LSTM (policy.py:66,141).  Layout, saved tensors and
// in-place reuse of the gate buffer are described in include/dotaclient_b200.h and DESIGN.md.
#include "rnn_generic.cuh"
#include "rnn_resident.cuh"
#include "rnn_cluster.cuh"
#include "rnn_stepwise.cuh"

// Kernel selection by width (no environment switches, no library fallback):
//   H == 128  rnn_resident.cuh  W_hh resident in registers + shared memory of ONE SM, fp32 FFMA
//   H == 256  rnn_cluster.cuh   W_hh resident in registers + shared memory of an 8-CTA cluster, wgmma 3xTF32
//   H % 128 == 0 (384, 512, ...)  rnn_stepwise.cuh  per step: split-K wgmma 3xTF32 GEMM over all SMs + gate kernel
//   other H   rnn_generic.cuh   W_hh streamed from L2 every step, scalar FMA (correct for any H % 4 == 0)

extern "C" size_t dc_rnn_workspace_bytes(int cell, int B, int H) {
    const int G = cell == DC_CELL_GRU ? 3 : 4;
    if (dc_rnnc::cluster_supported(H)) return dc_rnnc::bwd_workspace_bytes(B > 0 ? B : 1);   // partial-sum exchange (backward)
    if (dc_rnns::stepwise_supported(H)) return dc_rnns::workspace_bytes(cell, B > 0 ? B : 1, H);
    return (size_t)G * H * H * sizeof(float);   // W_hh^T for the resident and generic forward kernels
}

static int check_rnn_args(const char *fn, int cell, int B, int S, int H) {
    DC_REQUIRE(cell == DC_CELL_GRU || cell == DC_CELL_LSTM, DC_EINVAL, "%s: unknown cell %d", fn, cell);
    DC_REQUIRE(B > 0 && S > 0, DC_EINVAL, "%s: B=%d S=%d", fn, B, S);
    DC_REQUIRE(H >= 4 && H % 4 == 0 && H <= 2048, DC_EUNSUPPORTED, "%s: H=%d must be a multiple of 4 in [4, 2048]", fn, H);
    return DC_OK;
}

// Dispatch shared by the plain entry points (kReset = false, rs unused) and the _reset ones.
template <bool kReset>
static int rnn_fwd(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf, float *cbuf, int B, int S, int H,
                   void *workspace, dc_rnn::Reset rs, cudaStream_t st) {
    if (dc_rnn::resident_supported(H)) return dc_rnn::launch_fwd_resident<kReset>(cell, gates, w_hh, b_hh, ybuf, cbuf, B, S, workspace, rs, st);
    if (dc_rnnc::cluster_supported(H)) return dc_rnnc::launch_fwd<kReset>(cell, gates, w_hh, b_hh, ybuf, cbuf, B, S, rs, st);
    if (dc_rnns::stepwise_supported(H)) return dc_rnns::launch_fwd<kReset>(cell, gates, w_hh, b_hh, ybuf, cbuf, B, S, H, workspace, rs, st);
    return dc_rnn::launch_fwd_generic<kReset>(cell, gates, w_hh, b_hh, ybuf, cbuf, B, S, H, workspace, rs, st);
}

template <bool kReset>
static int rnn_bwd(const char *fn, int cell, float *gates, const float *w_hh, const float *ybuf, float *cbuf, const float *dy,
                   const float *dhn, const float *dcn, float *dh0, float *dc0, int B, int S, int H, void *workspace,
                   dc_rnn::Reset rs, cudaStream_t st) {
    if (dc_rnn::resident_supported(H)) return dc_rnn::launch_bwd_resident<kReset>(cell, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, rs, st);
    if (dc_rnnc::cluster_supported(H)) {
        DC_REQUIRE(workspace, DC_EINVAL, "%s: the H = 256 kernels need the workspace (dc_rnn_workspace_bytes)", fn);
        return dc_rnnc::launch_bwd<kReset>(cell, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, reinterpret_cast<float *>(workspace),
                                           B, S, rs, st);
    }
    if (dc_rnns::stepwise_supported(H)) {
        DC_REQUIRE(workspace, DC_EINVAL, "%s: the step-wise kernels need the workspace (dc_rnn_workspace_bytes)", fn);
        return dc_rnns::launch_bwd<kReset>(cell, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, H, workspace, rs, st);
    }
    return dc_rnn::launch_bwd_generic<kReset>(cell, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, H, rs, st);
}

extern "C" int dc_rnn_seq_fwd(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf, float *cbuf,
                              int B, int S, int H, void *workspace, dc_stream_t stream) {
    int rc = check_rnn_args("dc_rnn_seq_fwd", cell, B, S, H);
    if (rc) return rc;
    DC_REQUIRE(gates && w_hh && b_hh && ybuf && cbuf && workspace, DC_EINVAL, "dc_rnn_seq_fwd: null pointer");
    return rnn_fwd<false>(cell, gates, w_hh, b_hh, ybuf, cbuf, B, S, H, workspace, dc_rnn::Reset{}, dc_cu_stream(stream));
}

extern "C" int dc_rnn_seq_bwd(int cell, float *gates, const float *w_hh, const float *ybuf, float *cbuf, const float *dy,
                              const float *dhn, const float *dcn, float *dh0, float *dc0, int B, int S, int H,
                              void *workspace, dc_stream_t stream) {
    int rc = check_rnn_args("dc_rnn_seq_bwd", cell, B, S, H);
    if (rc) return rc;
    DC_REQUIRE(gates && w_hh && ybuf && cbuf && dy, DC_EINVAL, "dc_rnn_seq_bwd: null pointer");
    return rnn_bwd<false>("dc_rnn_seq_bwd", cell, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, H, workspace,
                          dc_rnn::Reset{}, dc_cu_stream(stream));
}

static int check_reset_args(const char *fn, const int32_t *reset_slot, const float *reset_prev, const float *reset_pre, int K,
                            bool need_pre) {
    DC_REQUIRE(reset_slot, DC_EINVAL, "%s: null reset_slot", fn);
    DC_REQUIRE(K >= 0, DC_EINVAL, "%s: K=%d", fn, K);
    DC_REQUIRE(K == 0 || (reset_prev && (reset_pre || !need_pre)), DC_EINVAL, "%s: null reset table with K=%d", fn, K);
    return DC_OK;
}

extern "C" int dc_rnn_seq_fwd_reset(int cell, float *gates, const float *w_hh, const float *b_hh, float *ybuf, float *cbuf,
                                    const int32_t *reset_slot, const float *reset_prev, const float *reset_pre, int K, int B,
                                    int S, int H, void *workspace, dc_stream_t stream) {
    int rc = check_rnn_args("dc_rnn_seq_fwd_reset", cell, B, S, H);
    if (rc) return rc;
    DC_REQUIRE(gates && w_hh && b_hh && ybuf && cbuf && workspace, DC_EINVAL, "dc_rnn_seq_fwd_reset: null pointer");
    rc = check_reset_args("dc_rnn_seq_fwd_reset", reset_slot, reset_prev, reset_pre, K, true);
    if (rc) return rc;
    return rnn_fwd<true>(cell, gates, w_hh, b_hh, ybuf, cbuf, B, S, H, workspace, dc_rnn::Reset{reset_slot, reset_prev, reset_pre},
                         dc_cu_stream(stream));
}

extern "C" int dc_rnn_seq_bwd_reset(int cell, float *gates, const float *w_hh, const float *ybuf, float *cbuf, const float *dy,
                                    const float *dhn, const float *dcn, float *dh0, float *dc0, const int32_t *reset_slot,
                                    const float *reset_prev, int K, int B, int S, int H, void *workspace, dc_stream_t stream) {
    int rc = check_rnn_args("dc_rnn_seq_bwd_reset", cell, B, S, H);
    if (rc) return rc;
    DC_REQUIRE(gates && w_hh && ybuf && cbuf && dy, DC_EINVAL, "dc_rnn_seq_bwd_reset: null pointer");
    rc = check_reset_args("dc_rnn_seq_bwd_reset", reset_slot, reset_prev, nullptr, K, false);
    if (rc) return rc;
    return rnn_bwd<true>("dc_rnn_seq_bwd_reset", cell, gates, w_hh, ybuf, cbuf, dy, dhn, dcn, dh0, dc0, B, S, H, workspace,
                         dc_rnn::Reset{reset_slot, reset_prev, nullptr}, dc_cu_stream(stream));
}
