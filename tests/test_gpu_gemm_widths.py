"""GPU tests of the wgmma 3xTF32 GEMMs at output widths that are multiples of 32 but not of 128 (the last column tile is
partly filled): the forward / data-gradient GEMM with a ragged N and the weight-gradient GEMM with a ragged No / Ni, against
float64 with the bounds of test_gpu_gemm.py, plus checks that nothing is written outside the output."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = -1234.5


def dev():
    return torch.device("cuda", 0)


@pytest.mark.parametrize("N", [32, 96, 160, 288, 576, 2048 + 32])
@pytest.mark.parametrize("K", [32, 96, 192, 896])
def test_gemm_ragged_n_matches_fp64_and_stays_in_its_columns(N, K):
    """C = relu(A B^T + bias) written into the column-slice view out_big[:M, 128:128+N] of a wider buffer filled with a
    sentinel: the columns of the last, partly filled column tile past N and the rows past M must keep the sentinel."""
    from dotaclient_b200 import ops
    d = dev()
    for M in (1, 127, 129, 5000):
        g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
        a = torch.randn(M, K, generator=g).to(d)
        b = (torch.randn(N, K, generator=g) * 0.3).to(d)
        bias = torch.randn(N, generator=g).to(d)
        out_big = torch.full((M + 1, N + 256), SENTINEL, device=d)
        out = out_big[:M, 128:128 + N]
        ops.gemm_tf32x3(a, b, bias, relu=True, out=out)
        ref = (a.double() @ b.double().t() + bias.double()).clamp_min(0)
        scale = (a.double().abs() @ b.double().abs().t()).max().item()
        err = (out.double() - ref).abs().max().item()
        assert err <= 3e-6 * scale, (M, err, scale)
        assert bool((out_big[:, :128] == SENTINEL).all()), M
        assert bool((out_big[:, 128 + N:] == SENTINEL).all()), M
        assert bool((out_big[M] == SENTINEL).all()), M
        # no bias, no ReLU, contiguous output: the plain layer form
        plain = ops.gemm_tf32x3(a, b)
        err = (plain.double() - a.double() @ b.double().t()).abs().max().item()
        assert err <= 3e-6 * scale, (M, err, scale)


@pytest.mark.parametrize("T,No,Ni", [(1, 32, 96), (777, 96, 160), (4097, 576, 192), (3000, 192, 896), (5000, 128, 96)])
def test_gemm_wgrad_ragged_matches_fp64(T, No, Ni):
    """dW = dY^T X and db = colsum(dY) with No / Ni multiples of 32: float64 bounds, bitwise determinism, and accumulation into
    a row slice of a larger gradient (the GRU's dW_hh[2H:]) that leaves the rows outside the slice untouched."""
    from dotaclient_b200 import ops
    d = dev()
    g = torch.Generator().manual_seed(T + 3 * No + 7 * Ni)
    dy = torch.randn(T, No, generator=g).to(d)                 # contiguous: row stride == No, the last row ends the buffer
    x = torch.randn(T, Ni, generator=g).to(d)
    dw, db = ops.gemm_wgrad_tf32x3(dy, x)
    ref = dy.double().t() @ x.double()
    scale = (dy.double().abs().t() @ x.double().abs()).max().item()
    assert (dw.double() - ref).abs().max().item() <= 3e-6 * scale
    refb = dy.double().sum(0)
    assert (db.double() - refb).abs().max().item() <= 1e-6 * dy.double().abs().sum(0).max().item() + 1e-6
    dw2, db2 = ops.gemm_wgrad_tf32x3(dy, x)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)        # deterministic
    # accumulate into rows [32, 32 + No) of a [No + 64, Ni] gradient, dy a column-slice view (row stride No + 32)
    base = torch.randn(No + 64, Ni, generator=g).to(d)
    acc = base.clone()
    big = torch.randn(T, No + 32, generator=g).to(d)
    dys = big[:, 32:]
    ops.gemm_wgrad_tf32x3(dys, x, want_bias=False, dw_out=acc[32:32 + No], accumulate=True)
    ref2 = base[32:32 + No].double() + dys.double().t() @ x.double()
    assert (acc[32:32 + No].double() - ref2).abs().max().item() <= 3e-6 * max(scale, 1.0) * 4
    assert torch.equal(acc[:32], base[:32]) and torch.equal(acc[32 + No:], base[32 + No:])
