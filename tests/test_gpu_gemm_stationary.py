"""GPU tests of the weight-stationary GEMM (K <= 128) at sizes where every CTA runs several tiles on both consumer
warpgroups: results against float64, the max-pool epilogue's arg-max, and bitwise repeatability."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(50000, 128, 128), (40001, 384, 96), (30000, 160, 64), (9000, 896, 32)])
def test_stationary_gemm_vs_fp64_and_repeatable(M, N, K):
    from dotaclient_b200 import ops
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g)
    b = torch.randn(N, K, generator=g) * 0.3
    bv = torch.randn(N, generator=g)
    d = torch.device("cuda", 0)
    ad, bd, bvd = a.to(d), b.to(d), bv.to(d)
    out1 = ops.gemm_tf32x3(ad, bd, bvd, relu=True)
    out2 = ops.gemm_tf32x3(ad, bd, bvd, relu=True)
    assert torch.equal(out1, out2)
    ref = (a.double() @ b.double().t() + bv.double()).clamp_min(0)
    scale = (a.double().abs() @ b.double().abs().t()).max().item()
    assert (out1.cpu().double() - ref).abs().max().item() <= 3e-6 * scale


@pytest.mark.parametrize("n_units", [5, 16])
def test_unit_max_many_tiles_per_cta(n_units):
    from dotaclient_b200 import _lib
    lib = _lib.load()
    d = torch.device("cuda", 0)
    n_tok, C, ld = 20011, 128, 256
    g = torch.Generator().manual_seed(n_units)
    basic = torch.randn(n_tok * n_units, C, generator=g)
    w = torch.randn(C, C, generator=g) * 0.2
    bias = torch.randn(C, generator=g)
    bd, wd, biasd = basic.to(d), w.to(d), bias.to(d)

    def run():
        xmax = torch.full((n_tok, ld), float("nan"), device=d)
        copy = torch.full((n_tok, ld), float("nan"), device=d)
        am = torch.full((n_tok, C), 255, dtype=torch.uint8, device=d)
        _lib.check(lib.dc_gemm_unit_max(bd.data_ptr(), wd.data_ptr(), biasd.data_ptr(), xmax.data_ptr(), copy.data_ptr(), ld,
                                        am.data_ptr(), n_tok, n_units, _lib.stream_ptr()), "dc_gemm_unit_max")
        torch.cuda.synchronize()
        return xmax, copy, am

    x1, c1, a1 = run()
    x2, c2, a2 = run()
    assert torch.equal(x1[:, :C], x2[:, :C]) and torch.equal(a1, a2) and torch.equal(x1[:, :C], c1[:, :C])
    assert torch.isnan(x1[:, C:]).all()                                   # nothing written past the 128 features
    emb = (basic.double() @ w.double().t()).view(n_tok, n_units, C)
    top2 = emb.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-4 * top2[:, 0].abs().clamp_min(1.0)   # no near-ties: arg-max is well defined
    ref_max, ref_arg = emb.max(dim=1)
    assert ((x1[:, :C].cpu().double() - (ref_max + bias.double())).abs() <= 1e-5 * (1 + ref_max.abs())).all()
    assert torch.equal(a1.cpu().long()[clear], ref_arg[clear])
    assert clear.float().mean() > 0.99
