"""GPU tests of the unit encoder's stored ReLU mask: dc_unit_embed_fwd_mask writes, next to the forward's own results, channel j
of every unit row as bit j / 4 of word j % 4 of the row's 4 words (basic[row, j] > 0), and dc_unit_dgrad_fused_mask takes relu' from those words instead of
recomputing the basic layer.  The stored-mask and the recompute form run the same kernel body and must agree bit for bit;
against float64 at the benchmark's 131,072 tokens for every group shape of the encoder."""
import pytest
import torch

pytestmark = pytest.mark.gpu

C, F = 128, 12
BITS = None


def _unpack(mask):
    """[R, 4] int32 words -> [R, 128] bool (bit i of word w = channel 4i + w)."""
    global BITS
    if BITS is None:
        BITS = torch.arange(32, dtype=torch.int32, device=mask.device)
    return ((mask.unsqueeze(-1) >> BITS) & 1).bool().transpose(1, 2).reshape(mask.shape[0], C)


def _fwd(lib, _lib, units, w_b, b_b, w, bias, n_tok, n_units, basic, mask, ld=256):
    d = units.device
    xmax = torch.full((n_tok, ld), float("nan"), device=d)
    copy = torch.full((n_tok, ld), float("nan"), device=d) if n_units > 1 else None
    am = torch.full((n_tok, C), 255, dtype=torch.uint8, device=d) if n_units > 1 else None
    _lib.check(lib.dc_unit_embed_fwd_mask(units.data_ptr(), w_b.data_ptr(), b_b.data_ptr(), _lib.ptr(basic), _lib.ptr(mask), w.data_ptr(),
                                          bias.data_ptr(), xmax.data_ptr(), _lib.ptr(copy), ld, _lib.ptr(am), n_tok, n_units,
                                          _lib.stream_ptr()), "dc_unit_embed_fwd_mask")
    torch.cuda.synchronize()
    return xmax, copy, am


def _weights(seed):
    g = torch.Generator().manual_seed(seed)
    d = torch.device("cuda", 0)
    w_b = (torch.randn(C, F, generator=g) * 0.4).to(d)
    b_b = (torch.randn(C, generator=g) * 0.3).to(d)
    w = (torch.randn(C, C, generator=g) * 0.2).to(d)
    bias = torch.randn(C, generator=g).to(d)
    return g, w_b, b_b, w, bias


@pytest.mark.parametrize("n_tok", [1, 7, 20011])
@pytest.mark.parametrize("n_units", [1, 5, 16])
def test_stored_mask_is_the_forward_relu(n_units, n_tok):
    """Every bit equals basic > 0 of the activations the same launch stored (partial tiles included: 7 tokens, and 20011 x 5
    rows end inside a 60-row tile), the words past the last row are untouched, and storing the mask changes none of the
    forward's results."""
    from dotaclient_b200 import _lib
    lib = _lib.load()
    g, w_b, b_b, w, bias = _weights(77 * n_units + n_tok)
    R = n_tok * n_units
    units = (torch.randn(R, F, generator=g) * 1.5).to(w.device)
    units[::3, :6] = 0.0                                 # rows whose pre-activation is often exactly b_b: bits on the boundary
    basic = torch.full((R, C), float("nan"), device=w.device)
    mask = torch.full((R + 2, 4), -7, dtype=torch.int32, device=w.device)
    x1, c1, a1 = _fwd(lib, _lib, units, w_b, b_b, w, bias, n_tok, n_units, basic, mask)
    x2, c2, a2 = _fwd(lib, _lib, units, w_b, b_b, w, bias, n_tok, n_units, None, None)
    assert torch.equal(_unpack(mask[:R]), basic > 0)
    assert (mask[R:] == -7).all()
    assert torch.equal(x1[:, :C], x2[:, :C])
    if n_units > 1:
        assert torch.equal(c1[:, :C], c2[:, :C]) and torch.equal(a1, a2)
    mask2 = torch.zeros((R, 4), dtype=torch.int32, device=w.device)
    _fwd(lib, _lib, units, w_b, b_b, w, bias, n_tok, n_units, None, mask2)       # without basic_out: the same words
    assert torch.equal(mask2, mask[:R])


def _grid(g, shape, scale, k):
    """Values on a binary grid, so that the basic layer's pre-activation is exact in fp32 in any summation order and the
    float64 ReLU mask cannot differ from the kernels' by rounding."""
    return torch.round(torch.randn(shape, generator=g, device="cuda") * scale * k) / k


def _inputs(N, n_u, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    units = _grid(g, (N * n_u, F), 1.0, 16)
    w_b, b_b = _grid(g, (C, F), 0.3, 64), _grid(g, (C,), 0.1, 64)
    W = torch.randn(C, C, generator=g, device="cuda") * 0.1
    bias = torch.randn(C, generator=g, device="cuda")
    dx = torch.randn(N, 7 * C, generator=g, device="cuda")           # a pre-rnn gradient row; slots 2 and 5 are read
    am = torch.randint(0, n_u, (N, C), generator=g, device="cuda").to(torch.uint8)
    dl = torch.randn(N, 40, generator=g, device="cuda")
    dl[::2] = 0.0
    att = torch.randn(N, C, generator=g, device="cuda")
    return dict(units=units, w_b=w_b, b_b=b_b, W=W, bias=bias, dx=dx, am=am, dl=dl, att=att)


def _dgrad(lib, _lib, t, N, n_u, mask, routed, dx2, head, accumulate, dwb, dbb, ws, wt):
    dx = t["dx"].data_ptr()
    _lib.check(lib.dc_unit_dgrad_fused_mask(dx + 4 * 256 if routed else None, dx + 4 * 640 if dx2 else None, 896,
                                            t["am"].data_ptr() if (routed and n_u > 1) else None,
                                            t["dl"].data_ptr() + 4 * 3 if head else None, 40, t["att"].data_ptr() if head else None,
                                            wt.data_ptr(), t["units"].data_ptr(), _lib.ptr(mask), t["w_b"].data_ptr(), t["b_b"].data_ptr(),
                                            N, n_u, dwb.data_ptr(), dbb.data_ptr(), accumulate, ws.data_ptr(), _lib.stream_ptr()),
               "dc_unit_dgrad_fused_mask")
    torch.cuda.synchronize()


def _stored_mask(lib, _lib, t, N, n_u):
    mask = torch.empty((N * n_u, 4), dtype=torch.int32, device="cuda")
    _fwd(lib, _lib, t["units"], t["w_b"], t["b_b"], t["W"], t["bias"], N, n_u, None, mask)
    return mask


@pytest.mark.parametrize("N,n_u", [(7, 1), (7, 5), (7, 16), (20011, 1), (20011, 5), (20011, 16)])
def test_stored_mask_and_recompute_give_the_same_bits(N, n_u):
    """dW_b / db_b from the forward's mask and from the mask recomputed in the kernel: the same mask, the same summation."""
    from dotaclient_b200 import _lib
    lib = _lib.load()
    t = _inputs(N, n_u, 5 + N + n_u)
    t["units"] = torch.randn(N * n_u, F, device="cuda") * 1.5                # off the grid: ReLU decided by fp32 rounding
    wt = t["W"].t().contiguous()
    ws = torch.empty(int(lib.dc_unit_basic_bwd_workspace_bytes()), dtype=torch.uint8, device="cuda")
    mask = _stored_mask(lib, _lib, t, N, n_u)
    out = []
    for m in (mask, None):
        dwb, dbb = torch.full((C, F), 7.0, device="cuda"), torch.full((C,), 7.0, device="cuda")
        _dgrad(lib, _lib, t, N, n_u, m, True, n_u == 16, True, 0, dwb, dbb, ws, wt)
        out.append((dwb, dbb))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])

    # the kMask form reads the words: invert word 0 (channels j % 4 == 0) and exactly those rows of dW_b / db_b change
    flipped = mask ^ torch.tensor([-1, 0, 0, 0], dtype=torch.int32, device="cuda")
    dwb, dbb = torch.full((C, F), 7.0, device="cuda"), torch.full((C,), 7.0, device="cuda")
    _dgrad(lib, _lib, t, N, n_u, flipped, True, n_u == 16, True, 0, dwb, dbb, ws, wt)
    keep = torch.arange(C, device="cuda") % 4 != 0
    assert torch.equal(dwb[keep], out[0][0][keep]) and torch.equal(dbb[keep], out[0][1][keep])
    assert (dbb[~keep] != out[0][1][~keep]).any()


# the unit groups of the encoder: (units, routed through the max-pool, second gradient source) -- allied / enemy heroes,
# allied non-heroes, enemy non-heroes (whose maximum also feeds the tower slot), and the towers, which have no forward launch
GROUPS = [(1, True, False), (5, True, False), (16, True, False), (16, True, True), (1, False, False)]


@pytest.mark.parametrize("head", [False, True])
@pytest.mark.parametrize("n_u,routed,dx2", GROUPS)
def test_dgrad_with_stored_mask_vs_fp64_at_benchmark_tokens(n_u, routed, dx2, head):
    """At 131,072 tokens (the benchmark's C2 batch) every CTA runs a hundred tiles or more: dW_b / db_b against the dense
    float64 chain, within 5e-5 of the float64 sum of |terms|.  Routed groups read the forward's mask, the towers recompute it,
    as the encoder does.  A repeated call is bitwise equal, and the accumulate flag gives exactly twice the result."""
    from dotaclient_b200 import _lib
    lib = _lib.load()
    N = 131072
    t = _inputs(N, n_u, 100 * n_u + 10 * routed + dx2 + 2 * head)
    wt = t["W"].t().contiguous()
    ws = torch.empty(int(lib.dc_unit_basic_bwd_workspace_bytes()), dtype=torch.uint8, device="cuda")
    mask = _stored_mask(lib, _lib, t, N, n_u) if routed else None
    dwb, dbb = torch.full((C, F), 7.0, device="cuda"), torch.full((C,), 7.0, device="cuda")
    _dgrad(lib, _lib, t, N, n_u, mask, routed, dx2, head, 0, dwb, dbb, ws, wt)

    ref_w = torch.zeros(C, F, dtype=torch.float64, device="cuda")
    ref_b = torch.zeros(C, dtype=torch.float64, device="cuda")
    abs_w, abs_b = torch.zeros_like(ref_w), torch.zeros_like(ref_b)
    W64, wb64, bb64 = t["W"].double(), t["w_b"].double(), t["b_b"].double()
    step = 8192
    for n0 in range(0, N, step):
        n1 = min(N, n0 + step)
        n = n1 - n0
        u = t["units"][n0 * n_u:n1 * n_u].double()
        basic = torch.relu(u @ wb64.t() + bb64)
        d_emb = torch.zeros(n, n_u, C, dtype=torch.float64, device="cuda")
        if routed:
            d = t["dx"][n0:n1, 2 * C:3 * C].double() + (t["dx"][n0:n1, 5 * C:6 * C].double() if dx2 else 0)
            d_emb.scatter_(1, t["am"][n0:n1].long().unsqueeze(1), d.unsqueeze(1)) if n_u > 1 else d_emb.copy_(d.unsqueeze(1))
        if head:
            d_emb += t["dl"][n0:n1, 3:3 + n_u].double().unsqueeze(-1) * t["att"][n0:n1].double().unsqueeze(1)
        gm = (d_emb.reshape(n * n_u, C) @ W64) * (basic > 0)
        ref_w += gm.t() @ u
        ref_b += gm.sum(0)
        abs_w += gm.abs().t() @ u.abs()
        abs_b += gm.abs().sum(0)
    assert ((dwb.double() - ref_w).abs() <= 5e-5 * abs_w + 1e-6).all()
    assert ((dbb.double() - ref_b).abs() <= 5e-5 * abs_b + 1e-6).all()

    dwb1, dbb1 = dwb.clone(), dbb.clone()
    _dgrad(lib, _lib, t, N, n_u, mask, routed, dx2, head, 0, dwb, dbb, ws, wt)
    assert torch.equal(dwb, dwb1) and torch.equal(dbb, dbb1)
    _dgrad(lib, _lib, t, N, n_u, mask, routed, dx2, head, 1, dwb, dbb, ws, wt)
    assert torch.equal(dwb, 2 * dwb1) and torch.equal(dbb, 2 * dbb1)
