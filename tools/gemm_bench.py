"""Micro-benchmark of dc_gemm_tf32x3 against cuBLAS fp32 / TF32 on the model's GEMM shapes (CUDA events)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from dotaclient_b200 import _lib, ops  # noqa: E402


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _floor(flops3, bytes_, ms):
    """Fraction of the larger of the tensor floor (3xTF32 flops at the 495 TFLOP/s dense-TF32 data-sheet rate) and the HBM
    floor (algorithmic bytes at 3.35 TB/s) that `ms` reaches, and which of the two bounds it."""
    t_tc, t_hbm = flops3 / 495e12 * 1e3, bytes_ / 3.35e12 * 1e3
    return "%.0f%% of the %s floor" % (100 * max(t_tc, t_hbm) / ms, "tensor" if t_tc >= t_hbm else "HBM")


def main():
    d = torch.device("cuda", 0)
    lib, st = _lib.load(), _lib.stream_ptr()
    shapes = [("unit-embedding (16 units)", 131072 * 16, 128, 128), ("i2h lstm H128", 131072, 512, 128),
              ("pre_rnn", 131072, 128, 896), ("i2h lstm H512 (c4)", 524288 // 4, 2048, 512)]
    for name, M, N, K in shapes:
        a = torch.randn(M, K, device=d)
        b = torch.randn(N, K, device=d) * 0.1
        bias = torch.randn(N, device=d)
        out = torch.empty(M, N, device=d)
        ref = torch.addmm(bias, a, b.t())
        got = ops.gemm_tf32x3(a, b, bias, out=out)
        err = (got - ref).abs().max().item()
        t_ours = timeit(lambda: ops.gemm_tf32x3(a, b, bias, out=out))
        torch.backends.cuda.matmul.allow_tf32 = False
        t_fp32 = timeit(lambda: torch.addmm(bias, a, b.t(), out=out))
        torch.backends.cuda.matmul.allow_tf32 = True
        t_tf32 = timeit(lambda: torch.addmm(bias, a, b.t(), out=out))
        torch.backends.cuda.matmul.allow_tf32 = False
        flops = 2.0 * M * N * K
        bytes_ = 4.0 * (M * K + N * K + M * N)
        print("%-28s M=%8d N=%4d K=%4d | ours %.3f ms (%.1f TF/s eff, %.0f GB/s, %s) | cublas fp32 %.3f ms | cublas tf32 %.3f ms | "
              "max|diff vs fp32| %.2e" % (name, M, N, K, t_ours, flops / t_ours / 1e9, bytes_ / t_ours / 1e6,
                                          _floor(3 * flops, bytes_, t_ours), t_fp32, t_tf32, err))

    # the max-pool epilogue GEMMs of the unit embeddings (dc_gemm_unit_max): 16- and 5-unit groups, [N, 128] outputs
    for n_u in (16, 5):
        N_tok, C = 131072, 128
        basic = torch.randn(N_tok * n_u, C, device=d)
        w = torch.randn(C, C, device=d) * 0.1
        bias = torch.randn(C, device=d)
        xmax = torch.empty(N_tok, 896, device=d)
        am = torch.empty(N_tok, C, dtype=torch.uint8, device=d)
        t = timeit(lambda: _lib.check(lib.dc_gemm_unit_max(basic.data_ptr(), w.data_ptr(), bias.data_ptr(), xmax.data_ptr(), None, 896,
                                                           am.data_ptr(), N_tok, n_u, st), "unit_max"))
        flops = 3 * 2.0 * N_tok * n_u * C * C
        bytes_ = 4.0 * (N_tok * n_u * C + C * C + N_tok * C) + N_tok * C
        print("unit max %2d units           rows=%8d | %.3f ms (%.1f TF/s 3xTF32, %s)" % (n_u, N_tok * n_u, t, flops / t / 1e9,
                                                                                       _floor(flops, bytes_, t)))

    # weight gradients as the C2 step issues them (T = 131072 tokens): plain dW = dY^T X (+ db), and the routed form of the
    # 5- and 16-unit groups (dY generated from the max-pool's arg-max)
    T, C, ld = 131072, 128, 896
    for No, Ni, bias, what in [(128, 128, True, "1-unit group"), (512, 128, True, "i2h dW_ih"), (512, 128, False, "dW_hh"),
                               (128, 896, True, "pre-rnn"), (128, 896, False, "target-unit head att^T s")]:
        dy, x = torch.randn(T, No, device=d), torch.randn(T, Ni, device=d)
        ws = torch.empty(int(lib.dc_gemm_wgrad_workspace_bytes(No, Ni)), dtype=torch.uint8, device=d)
        dw, db = torch.empty(No, Ni, device=d), torch.empty(No, device=d)
        t = timeit(lambda: _lib.check(lib.dc_gemm_wgrad_tf32x3(dy.data_ptr(), No, x.data_ptr(), Ni, T, No, Ni, dw.data_ptr(), Ni,
                                                               db.data_ptr() if bias else None, 0, ws.data_ptr(), st), "wgrad"))
        flops, bytes_ = 3 * 2.0 * T * No * Ni, 4.0 * (T * No + T * Ni + No * Ni)
        print("wgrad %-26s T=%7d No=%4d Ni=%4d | %.3f ms (%.1f TF/s 3xTF32, %s)" % (what, T, No, Ni, t, flops / t / 1e9,
                                                                                 _floor(flops, bytes_, t)))
    xcat = torch.randn(T, ld, device=d)
    ws = torch.empty(int(lib.dc_gemm_wgrad_workspace_bytes(C, C)), dtype=torch.uint8, device=d)
    dw, db = torch.empty(C, C, device=d), torch.empty(C, device=d)
    for n_u in (16, 5):
        R = T * n_u
        basic = torch.randn(R, C, device=d)
        am = torch.randint(0, n_u, (T, C), dtype=torch.uint8, device=d)
        t = timeit(lambda: _lib.check(lib.dc_unit_wgrad_routed(xcat.data_ptr(), None, ld, am.data_ptr(), basic.data_ptr(), T, n_u,
                                                               dw.data_ptr(), db.data_ptr(), ws.data_ptr(), st), "wgrad routed"))
        flops, bytes_ = 3 * 2.0 * R * C * C, 4.0 * (R * C + C * C + T * C) + T * C
        print("wgrad routed %2d units                  rows=%8d | %.3f ms (%.1f TF/s 3xTF32, %s)" % (n_u, R, t, flops / t / 1e9,
                                                                                                  _floor(flops, bytes_, t)))

    # the fused data gradient of the unit-embedding layers (dc_unit_dgrad_fused), with and without the target-unit head
    ws_b = torch.empty(int(lib.dc_unit_basic_bwd_workspace_bytes()), dtype=torch.uint8, device=d)
    w_t, w_b, b_b = torch.randn(C, C, device=d) * 0.1, torch.randn(C, 12, device=d), torch.randn(C, device=d)
    dw_b, db_b = torch.empty(C, 12, device=d), torch.empty(C, device=d)
    dl, att = torch.randn(T, 40, device=d), torch.randn(T, C, device=d)
    for n_u in (16, 5, 1):
        R = T * n_u
        units = torch.randn(R, 12, device=d)
        am = torch.randint(0, n_u, (T, C), dtype=torch.uint8, device=d)
        for head in (False, True):
            t = timeit(lambda: _lib.check(lib.dc_unit_dgrad_fused(
                xcat.data_ptr(), None, ld, am.data_ptr() if n_u > 1 else None, dl.data_ptr() if head else None, 40,
                att.data_ptr() if head else None, w_t.data_ptr(), units.data_ptr(), w_b.data_ptr(), b_b.data_ptr(), T, n_u,
                dw_b.data_ptr(), db_b.data_ptr(), 0, ws_b.data_ptr(), st), "dgrad fused"))
            flops, bytes_ = 3 * 2.0 * R * C * C, T * 5.0 * C + 4.0 * R * 12 + (4.0 * T * (C + n_u) if head else 0)
            print("dgrad fused %2d units %-12s       rows=%8d | %.3f ms (%.1f TF/s 3xTF32, %s)"
                  % (n_u, "with head" if head else "without head", R, t, flops / t / 1e9, _floor(flops, bytes_, t)))


if __name__ == "__main__":
    main()
