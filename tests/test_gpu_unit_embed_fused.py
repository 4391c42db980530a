"""GPU tests of the unit encoder's forward without a basic-layer pass of its own: dc_unit_embed_fwd (basic layer generated in
the embedding GEMM's producers) against dc_gemm_unit_max / dc_gemm_tf32x3 on the basic activations it stored, the stored
activations against float64, and the target-unit head (which rebuilds them from the raw unit features) against float64.
Every call is repeated and must give the same bits."""
import pytest
import torch

pytestmark = pytest.mark.gpu

C, F = 128, 12
UNITS = (1, 5, 16, 16, 1, 1)
OFFSETS = (0, 1, 6, 22, 38, 39)


def _weights(seed):
    g = torch.Generator().manual_seed(seed)
    d = torch.device("cuda", 0)
    w_b = (torch.randn(C, F, generator=g) * 0.4).to(d)
    b_b = (torch.randn(C, generator=g) * 0.3).to(d)
    w = (torch.randn(C, C, generator=g) * 0.2).to(d)
    bias = torch.randn(C, generator=g).to(d)
    return g, w_b, b_b, w, bias


def _embed(lib, _lib, units, w_b, b_b, w, bias, n_tok, n_units, store, ld=256):
    d = units.device
    basic = torch.full((n_tok * n_units, C), float("nan"), device=d) if store else None
    xmax = torch.full((n_tok, ld), float("nan"), device=d)
    copy = torch.full((n_tok, ld), float("nan"), device=d) if n_units > 1 else None
    am = torch.full((n_tok, C), 255, dtype=torch.uint8, device=d) if n_units > 1 else None
    _lib.check(lib.dc_unit_embed_fwd(units.data_ptr(), w_b.data_ptr(), b_b.data_ptr(), _lib.ptr(basic), w.data_ptr(), bias.data_ptr(),
                                     xmax.data_ptr(), _lib.ptr(copy), ld, _lib.ptr(am), n_tok, n_units, _lib.stream_ptr()),
               "dc_unit_embed_fwd")
    torch.cuda.synchronize()
    return basic, xmax, copy, am


@pytest.mark.parametrize("n_tok", [1, 7, 20011, 40000])
@pytest.mark.parametrize("n_units", [1, 5, 16])
def test_unit_embed_matches_the_unfused_gemm_bit_for_bit(n_units, n_tok):
    from dotaclient_b200 import _lib
    lib = _lib.load()
    g, w_b, b_b, w, bias = _weights(1000 * n_units + n_tok)
    units = (torch.randn(n_tok * n_units, F, generator=g) * 1.5).to(w.device)
    basic, x1, c1, a1 = _embed(lib, _lib, units, w_b, b_b, w, bias, n_tok, n_units, store=True)
    _, x2, c2, a2 = _embed(lib, _lib, units, w_b, b_b, w, bias, n_tok, n_units, store=True)
    _, x3, c3, a3 = _embed(lib, _lib, units, w_b, b_b, w, bias, n_tok, n_units, store=False)

    # the stored basic layer: float64 relu(units W_b^T + b_b), exact zeros where the ReLU cuts
    assert not torch.isnan(basic).any()
    pre = units.double() @ w_b.double().t() + b_b.double()
    ref = pre.clamp_min(0)
    scale = units.double().abs() @ w_b.double().abs().t() + b_b.double().abs()
    assert ((basic.double() - ref).abs() <= 2e-6 * scale).all()
    assert (basic[pre < -1e-5 * scale] == 0).all()
    assert (basic >= 0).all()

    # the same launch with the stored basic as a plain A operand: the unfused path, bit for bit
    ld = x1.shape[1]
    xr = torch.full((n_tok, ld), float("nan"), device=w.device)
    if n_units > 1:
        cr = torch.full((n_tok, ld), float("nan"), device=w.device)
        ar = torch.full((n_tok, C), 255, dtype=torch.uint8, device=w.device)
        _lib.check(lib.dc_gemm_unit_max(basic.data_ptr(), w.data_ptr(), bias.data_ptr(), xr.data_ptr(), cr.data_ptr(), ld, ar.data_ptr(),
                                        n_tok, n_units, _lib.stream_ptr()), "dc_gemm_unit_max")
    else:
        _lib.check(lib.dc_gemm_tf32x3(basic.data_ptr(), C, w.data_ptr(), C, bias.data_ptr(), xr.data_ptr(), ld, n_tok, C, C, 0,
                                      _lib.stream_ptr()), "dc_gemm_tf32x3")
    torch.cuda.synchronize()
    assert torch.equal(x1[:, :C], xr[:, :C]) and torch.isnan(x1[:, C:]).all()
    for x in (x2, x3):                                  # bitwise repeat, and the basic_out = NULL form
        assert torch.equal(x1[:, :C], x[:, :C])
    if n_units > 1:
        assert torch.equal(c1[:, :C], cr[:, :C]) and torch.equal(a1, ar) and torch.equal(c1[:, :C], x1[:, :C])
        for c, a in ((c2, a2), (c3, a3)):
            assert torch.equal(c1[:, :C], c[:, :C]) and torch.equal(a1, a)
    # and against float64 (max-pool value; the arg-max is pinned by the bitwise comparison above)
    emb = (ref @ w.double().t()).view(n_tok, n_units, C).max(dim=1).values + bias.double()
    tol = 1e-5 * (1 + (scale @ w.double().abs().t()).view(n_tok, n_units, C).max(dim=1).values)
    assert ((x1[:, :C].double() - emb).abs() <= tol).all()


def _head_inputs(seed, N):
    g, w_b, b_b, _, _ = _weights(seed)
    d = w_b.device
    units = [(torch.randn(N * n, F, generator=g) * 1.5).to(d) for n in UNITS]
    q = torch.randn(N, 7 * C, generator=g).to(d)
    q[:, 6 * C + 6:] = float("nan")                     # columns the head never reads
    return g, units, w_b, b_b, q


def _basic64(units, w_b, b_b):
    return [(u.double() @ w_b.double().t() + b_b.double()).clamp_min(0) for u in units]


@pytest.mark.parametrize("N", [1, 3001])
def test_target_unit_head_from_raw_features_vs_fp64(N):
    from dotaclient_b200 import _lib
    lib = _lib.load()
    g, units, w_b, b_b, q = _head_inputs(N, N)
    ptrs = (_lib._c.c_void_p * 6)(*[u.data_ptr() for u in units])
    basics = _basic64(units, w_b, b_b)

    def fwd():
        logits = torch.full((N, 40), float("nan"), device=q.device)
        _lib.check(lib.dc_target_unit_q_fwd(q.data_ptr(), 7 * C, ptrs, w_b.data_ptr(), b_b.data_ptr(), logits.data_ptr(), N,
                                            _lib.stream_ptr()), "dc_target_unit_q_fwd")
        torch.cuda.synchronize()
        return logits

    l1, l2 = fwd(), fwd()
    assert torch.equal(l1, l2)
    q64 = q.double()
    for gi, (n, off) in enumerate(zip(UNITS, OFFSETS)):
        b = basics[gi].view(N, n, C)
        ref = torch.einsum("nuc,nc->nu", b, q64[:, gi * C:(gi + 1) * C]) + q64[:, 6 * C + gi:6 * C + gi + 1]
        scale = torch.einsum("nuc,nc->nu", b, q64[:, gi * C:(gi + 1) * C].abs()) + 1.0
        assert ((l1[:, off:off + n].double() - ref).abs() <= 1e-5 * scale).all(), gi

    dl = torch.randn(N, 40, generator=g).to(q.device)
    dl[::3] = 0.0                                        # tokens that did not use the head
    dl[1::3, :20] = 0.0                                  # ... and partly used rows

    def bwd():
        s = torch.full((N, 7 * C), float("nan"), device=q.device)
        _lib.check(lib.dc_target_unit_q_bwd(dl.data_ptr(), ptrs, w_b.data_ptr(), b_b.data_ptr(), s.data_ptr(), 7 * C, N,
                                            _lib.stream_ptr()), "dc_target_unit_q_bwd")
        torch.cuda.synchronize()
        return s

    s1, s2 = bwd(), bwd()
    assert torch.equal(s1, s2)
    assert (s1[::3] == 0).all()
    dl64 = dl.double()
    ref = torch.zeros(N, 7 * C, dtype=torch.float64, device=q.device)
    scale = torch.zeros_like(ref)
    for gi, (n, off) in enumerate(zip(UNITS, OFFSETS)):
        b = basics[gi].view(N, n, C)
        ref[:, gi * C:(gi + 1) * C] = torch.einsum("nu,nuc->nc", dl64[:, off:off + n], b)
        scale[:, gi * C:(gi + 1) * C] = torch.einsum("nu,nuc->nc", dl64[:, off:off + n].abs(), b)
        ref[:, 6 * C + gi] = dl64[:, off:off + n].sum(1)
        scale[:, 6 * C + gi] = dl64[:, off:off + n].abs().sum(1)
    assert ((s1.double() - ref).abs() <= 2e-6 * (scale + 1.0)).all()
