"""GPU test of the wgmma 3xTF32 GEMM (dc_gemm_tf32x3) against a float64 reference.

Tolerance: the 3xTF32 split keeps fp32-level accuracy -- max |err| <= 4e-6 * sqrt(K) * rms(a) * rms(b)-scaled bound below,
i.e. the same order as an fp32 SIMT GEMM and ~1000x tighter than single-pass TF32."""
import pytest
import torch

from test_gpu_rnn_fp64 import tf32_rna

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (1000, 128, 128), (129, 384, 256), (4096, 512, 128), (300, 128, 896),
                                   (1, 128, 128), (20000, 128, 128), (777, 2048, 512)])
@pytest.mark.parametrize("bias,relu", [(False, False), (True, False), (True, True)])
def test_gemm_tf32x3_matches_fp64(M, N, K, bias, relu):
    from dotaclient_b200 import ops
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g)
    b = torch.randn(N, K, generator=g) * 0.3
    bv = torch.randn(N, generator=g) if bias else None
    ref = a.double() @ b.double().t()
    if bias:
        ref = ref + bv.double()
    if relu:
        ref = ref.clamp_min(0)
    d = torch.device("cuda", 0)
    out = ops.gemm_tf32x3(a.to(d), b.to(d), None if bv is None else bv.to(d), relu=relu).cpu().double()
    err = (out - ref).abs().max().item()
    scale = (a.double().abs() @ b.double().abs().t()).max().item()      # sum |a||b| bounds the rounding error
    # measured: ~1.4e-6 * sum|a||b| at K=896 (the tensor core's fp32 accumulation is a little looser than FFMA), ~1e-7
    # at K=128; single-pass TF32 would be ~2e-4.
    assert err <= 3e-6 * scale, (err, scale)
    torch.backends.cuda.matmul.allow_tf32 = True
    tf32 = (a.to(d) @ b.to(d).t()).cpu().double()
    torch.backends.cuda.matmul.allow_tf32 = False
    if bias:
        tf32 = tf32 + bv.double()
    if relu:
        tf32 = tf32.clamp_min(0)
    err_tf32 = (tf32 - ref).abs().max().item()
    if K >= 128 and M >= 128:
        assert err * 20 < err_tf32, (err, err_tf32)       # >= 20x more accurate than single-pass TF32


def test_gemm_tf32x3_strided_views_and_unsupported_shapes():
    from dotaclient_b200 import ops
    d = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(1)
    big = torch.randn(500, 512, generator=g).to(d)
    a = big[:, 128:384]                                   # row stride 512, width 256
    b = torch.randn(128, 256, generator=g).to(d)
    out_big = torch.zeros(500, 256, device=d)
    ops.gemm_tf32x3(a, b, out=out_big[:, 128:])
    ref = (a.double() @ b.double().t())
    scale = (a.double().abs() @ b.double().abs().t()).max().item()
    assert (out_big[:, 128:].double() - ref).abs().max().item() < 3e-6 * scale
    assert float(out_big[:, :128].abs().sum()) == 0.0
    assert not ops.gemm_tf32x3_supported(100, 100, 128) and not ops.gemm_tf32x3_supported(100, 128, 12)
    with pytest.raises(RuntimeError):
        ops.gemm_tf32x3(torch.randn(10, 12, device=d), torch.randn(128, 12, device=d))


@pytest.mark.parametrize("T,No,Ni", [(1, 128, 128), (31, 128, 128), (32, 128, 128), (100, 128, 128), (5000, 128, 128),
                                     (100000, 128, 128), (4097, 512, 128), (3000, 128, 896), (777, 256, 256)])
def test_gemm_wgrad_tf32x3_matches_fp64(T, No, Ni):
    """dW = dY^T X and db = colsum(dY): operands transposed to K-major by the producers, split-K over the SMs, deterministic reduction."""
    from dotaclient_b200 import ops
    g = torch.Generator().manual_seed(T + No + Ni)
    dy = torch.randn(T, No, generator=g)
    x = torch.randn(T, Ni, generator=g)
    d = torch.device("cuda", 0)
    dw, db = ops.gemm_wgrad_tf32x3(dy.to(d), x.to(d))
    ref = dy.double().t() @ x.double()
    scale = (dy.double().abs().t() @ x.double().abs()).max().item()
    assert (dw.cpu().double() - ref).abs().max().item() <= 3e-6 * scale
    refb = dy.double().sum(0)
    assert (db.cpu().double() - refb).abs().max().item() <= 1e-6 * dy.double().abs().sum(0).max().item() + 1e-6
    dw2, db2 = ops.gemm_wgrad_tf32x3(dy.to(d), x.to(d))
    assert torch.equal(dw, dw2) and torch.equal(db, db2)            # deterministic
    # accumulate into an existing gradient, strided views, no bias
    base = torch.randn(No, Ni, generator=g).to(d)
    acc = base.clone()
    big = torch.randn(T, No + 128, generator=g).to(d)
    ops.gemm_wgrad_tf32x3(big[:, 128:], x.to(d), want_bias=False, dw_out=acc, accumulate=True)
    ref2 = base.cpu().double() + big[:, 128:].cpu().double().t() @ x.double()
    assert (acc.cpu().double() - ref2).abs().max().item() <= 3e-6 * max(scale, 1.0) * 4


DENSE_K896_BOUND = (96.0, 2e-6)     # K, FLOOR of max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|


@pytest.mark.parametrize("kind", ["normal", "coherent"])
@pytest.mark.parametrize("M,N", [(131072, 128), (524288, 512)])
def test_gemm_tf32x3_k896_at_benchmark_rows(M, N, kind):
    """The pre-RNN forward (K = 896, the ring kernel gemm_tf32x3_kernel) at c2's and c4's rows, against float64 on a sample
    of rows (tile boundaries included); coherent: A = ReLU(normal), as the encoder's outputs are.  Its accumulation length
    is the model's fixed K, so the error does not grow with M.  Measured on one H100 80GB HBM3 (700 W power limit), the
    ratio max|gpu - f64| / max|torch32 - f64| (torch fp32 on the CPU) and max|gpu - f64| / max|f64|:
        M 131072, N 128   normal 20.0 (6.1e-6)   coherent 27.3 (6.5e-6)
        M 524288, N 512   normal 15.3 (6.2e-6)   coherent 27.7 (8.3e-6)
    K = 96 leaves a margin of 3.5 over the largest ratio.  Single-pass TF32 (operands rounded by tf32_rna, exact sums)
    exceeds the bound 7.0 to 11.8 times."""
    from dotaclient_b200 import ops
    d = torch.device("cuda", 0)
    g = torch.Generator(device=d).manual_seed(M + N + (kind == "coherent"))
    a = torch.randn(M, 896, generator=g, device=d)
    if kind == "coherent":
        a = torch.relu(a)
    b = torch.randn(N, 896, generator=g, device=d) / 896 ** 0.5
    out = ops.gemm_tf32x3(a, b)
    rows = torch.tensor(sorted({0, 1, 127, 128, 255, 256, M // 2, M - 129, M - 128, M - 1}
                               | set(torch.randint(0, M, (54,), generator=torch.Generator().manual_seed(M)).tolist())))
    a_s, b_c = a[rows.to(d)].cpu(), b.cpu()
    f64 = a_s.double() @ b_c.double().t()
    f32 = (a_s @ b_c.t()).double()
    tf = tf32_rna(a_s).double() @ tf32_rna(b_c).double().t()
    err = (out[rows.to(d)].cpu().double() - f64).abs().max().item()
    cal, ref = (f32 - f64).abs().max().item(), f64.abs().max().item()
    lim = DENSE_K896_BOUND[0] * cal + DENSE_K896_BOUND[1] * ref
    print("\nK 896 M %d N %d %s: ratio to fp32 %.1f, max|err|/max|f64| %.2e, tf32 %.1fx the bound"
          % (M, N, kind, err / cal, err / ref, (tf - f64).abs().max().item() / lim))
    assert err <= lim, (err, cal, ref)
    assert (tf - f64).abs().max().item() > lim
