// What the four recurrence designs share: the GRU / LSTM cell arithmetic of one (sequence, unit) pair and the W_hh
// transpose.  The cell functions define the semantics parity depends on (torch.nn.GRU gate order r, z, n with
// n = tanh(gi_n + r (W_hn h + b_hn)); torch.nn.LSTM gate order i, f, g, o), so every kernel calls them and keeps only its
// own loads, stores and `bias + partial sums` order.
#pragma once
#include "dc_common.cuh"

namespace dc_rnn {

// Recurrent-state resets inside a sequence (dc_rnn_seq_fwd_reset / dc_rnn_seq_bwd_reset).  slot [S, B] int32: k = slot[t*B + b]
// >= 0 replaces the state entering step t of sequence b with row r = k*B + b of the column-local tables
//   prev [K, B, H]      h (GRU) or c (LSTM): the cell's `prev` operand
//   pre  [K, B, G*H]    h W_hh^T + b_hh of the reset h: the cell's `pre` operand (forward only)
// so the mat-vec of the step on the stale state is discarded.  Backward reads `prev` from the table and carries no gradient
// into step t-1 (neither through W_hh nor the direct dh z / dc f path).  Kernels take it as a template flag: the
// instantiations without it are the plain recurrence.
struct Reset {
    const int *slot;
    const float *prev;
    const float *pre;
};

// Forward step.  gi(g): i2h pre-activation of gate g (x W_ih^T + b_ih); pre(g): h2h pre-activation (W_hh h_{t-1} + b_hh);
// prev: h_{t-1} (GRU) or c_{t-1} (LSTM).  gi and pre are callables so that each kernel reads its inputs where the cell
// uses them (keeps register allocation as tight as a hand-inlined cell).  Writes the activated gates to act and what
// backward needs to aux (GRU: W_hn h_{t-1} + b_hn, LSTM: c_t); returns h_t.
// kFuseIG: the LSTM's c_t = f c_{t-1} + i g rounds one of its two products before the add.  The H = 128 kernels have
// always fused f c_{t-1} into the add and the other designs i g; the flag keeps each design's results bit for bit.
template <int G, bool kFuseIG = true, typename GI, typename PRE>
__device__ __forceinline__ float cell_fwd(GI gi, PRE pre, float prev, float (&act)[G], float &aux) {
    if constexpr (G == 3) {
        const float r = dc_sigmoid(gi(0) + pre(0));
        const float z = dc_sigmoid(gi(1) + pre(1));
        const float hn = pre(2);
        const float n = dc_tanh(gi(2) + r * hn);
        act[0] = r; act[1] = z; act[2] = n;
        aux = hn;
        return (1.0f - z) * n + z * prev;
    } else {
        const float ig = dc_sigmoid(gi(0) + pre(0));
        const float fg = dc_sigmoid(gi(1) + pre(1));
        const float gg = dc_tanh(gi(2) + pre(2));
        const float og = dc_sigmoid(gi(3) + pre(3));
        const float c = kFuseIG ? fmaf(ig, gg, fg * prev) : fmaf(fg, prev, ig * gg);
        act[0] = ig; act[1] = fg; act[2] = gg; act[3] = og;
        aux = c;
        return og * dc_tanh(c);
    }
}

// Backward step.  act(g): activated gate g as the forward saved it; aux: the forward's aux of this step; prev: h_{t-1}
// (GRU) or c_{t-1} (LSTM); dh: dL/dh_t; dc (LSTM): in dL/dc_t, out dL/dc_{t-1}.  Writes dgi (wrt the i2h pre-activations)
// and dgh (wrt the h2h pre-activations: the operand of the dh_{t-1} mat-vec; its GRU n entry dghn is what backward leaves
// in cbuf); returns the part of dh_{t-1} that does not go through W_hh.
template <int G, typename ACT>
__device__ __forceinline__ float cell_bwd(ACT act, float aux, float prev, float dh, float &dc, float (&dgi)[G], float (&dgh)[G]) {
    if constexpr (G == 3) {
        const float r = act(0), z = act(1), n = act(2), hn = aux;
        const float dpn = dh * (1.0f - z) * (1.0f - n * n);
        const float dpz = dh * (prev - n) * z * (1.0f - z);
        const float dpr = dpn * hn * r * (1.0f - r);
        const float dghn = dpn * r;
        dgi[0] = dpr; dgi[1] = dpz; dgi[2] = dpn;
        dgh[0] = dpr; dgh[1] = dpz; dgh[2] = dghn;
        return dh * z;
    } else {
        const float ig = act(0), fg = act(1), gg = act(2), og = act(3);
        const float tc = dc_tanh(aux);
        const float dct = dc + dh * og * (1.0f - tc * tc);
        const float dpi = dct * gg * ig * (1.0f - ig);
        const float dpf = dct * prev * fg * (1.0f - fg);
        const float dpg = dct * ig * (1.0f - gg * gg);
        const float dpo = dh * tc * og * (1.0f - og);
        dgi[0] = dpi; dgi[1] = dpf; dgi[2] = dpg; dgi[3] = dpo;
        dgh[0] = dpi; dgh[1] = dpf; dgh[2] = dpg; dgh[3] = dpo;
        dc = dct * fg;
        return 0.f;
    }
}

// out [cols, rows] = in [rows, cols]^T (W_hh^T for the kernels that want output columns contiguous)
__global__ void transpose_kernel(const float *__restrict__ in, float *__restrict__ out, int rows, int cols) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[i][threadIdx.x] = in[(size_t)r * cols + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) out[(size_t)c * rows + r] = tile[threadIdx.x][i];
    }
}

inline int launch_transpose(const float *in, float *out, int rows, int cols, cudaStream_t st) {
    transpose_kernel<<<dim3((cols + 31) / 32, (rows + 31) / 32), dim3(32, 8), 0, st>>>(in, out, rows, cols);
    DC_LAUNCH_OK();
    return DC_OK;
}

}  // namespace dc_rnn
