"""GPU tests of the unit-encoder kernel chain and the target-unit head against plain torch on the CPU
(the same ops the oracle's ``RefPolicy.forward`` performs, ``policy.py:99-136,144-153``).

Tolerances: fp32 kernels + 3xTF32 tensor-core GEMMs vs fp32 CPU: forward atol 2e-5 on O(1) activations,
gradients rtol 2e-4 with an absolute floor scaled by the token count (sums over tokens)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

UNITS = (1, 5, 16, 16, 1, 1)


def _reference(env, w_e, b_e, w_b, b_b, units, weights, biases):
    emb = [F.linear(F.relu(F.linear(u, w_b, b_b)), w, b) for u, w, b in zip(units, weights, biases)]
    mx = [e.max(dim=-2)[0] for e in emb]
    mx[5] = mx[3]                                        # policy.py:127
    return torch.cat(emb, dim=-2), torch.cat([F.relu(F.linear(env, w_e, b_e))] + mx, dim=-1)   # policy.py:97,129-136


def _setup(lead, seed):
    g = torch.Generator().manual_seed(seed)
    env = torch.randn(*lead, 3, generator=g)
    w_e = (torch.randn(128, 3, generator=g) * 0.5).requires_grad_(True)
    b_e = (torch.randn(128, generator=g) * 0.1).requires_grad_(True)
    w_b = (torch.randn(128, 12, generator=g) * 0.3).requires_grad_(True)
    b_b = (torch.randn(128, generator=g) * 0.1).requires_grad_(True)
    units = [torch.randn(*lead, n, 12, generator=g) for n in UNITS]
    weights = [(torch.randn(128, 128, generator=g) * 0.1).requires_grad_(True) for _ in UNITS]
    biases = [(torch.randn(128, generator=g) * 0.1).requires_grad_(True) for _ in UNITS]
    return g, env, w_e, b_e, w_b, b_b, units, weights, biases


@pytest.mark.parametrize("lead", [(7,), (3, 5), (1,), (130,), (27,)])
def test_unit_encoder_forward_backward(lead):
    """Pre-rnn row (env encoding + six group maxima, max-pool fused into the embedding GEMM's epilogue -- 125-row tiles for the
    5-unit group, 128 for the 16-unit groups, plain GEMMs for the 1-unit groups) and its gradients, no target-unit head."""
    from dotaclient_b200 import encoder_ops
    g, env, w_e, b_e, w_b, b_b, units, weights, biases = _setup(lead, sum(lead))
    ue_r, xm_r = _reference(env, w_e, b_e, w_b, b_b, units, weights, biases)
    g_xm = torch.randn(xm_r.shape, generator=g)
    (xm_r * g_xm).sum().backward()

    d = torch.device("cuda", 0)
    params = [t.detach().clone().to(d).requires_grad_(True) for t in [w_b, b_b] + weights + biases]
    pe = [t.detach().clone().to(d).requires_grad_(True) for t in (w_e, b_e)]
    link, xm = encoder_ops.unit_encoder(env.to(d), pe[0], pe[1], params[0], params[1], [u.to(d) for u in units], params[2:8],
                                        params[8:14])
    assert xm.shape == xm_r.shape
    torch.testing.assert_close(xm.detach().cpu(), xm_r.detach(), rtol=1e-4, atol=2e-5)
    (xm * g_xm.to(d)).sum().backward()
    n_tok = ue_r.numel() // (40 * 128)
    for mine, ref in zip(params + pe, [w_b, b_b] + weights + biases + [w_e, b_e]):
        expect = ref.grad if ref.grad is not None else torch.zeros_like(ref)      # the enemy-tower layer: no path without the head
        torch.testing.assert_close(mine.grad.cpu(), expect, rtol=2e-4, atol=2e-6 * max(1, n_tok) * 16)


def test_unit_max_tie_breaking_and_grad_routing():
    """Equal maxima: the FIRST unit wins (torch.max semantics on CPU) and receives the whole gradient."""
    from dotaclient_b200 import encoder_ops
    d = torch.device("cuda", 0)
    w_b = torch.zeros(128, 12)
    b_b = torch.ones(128)                                 # basic == 1 for every unit -> all units tie
    units = [torch.randn(4, n, 12) for n in UNITS]
    weights = [torch.eye(128) for _ in UNITS]
    biases = [torch.zeros(128) for _ in UNITS]
    params = [t.to(d).requires_grad_(True) for t in [w_b, b_b] + weights + biases]
    w_e, b_e = torch.zeros(128, 3, device=d, requires_grad=True), torch.full((128,), -1.0, device=d, requires_grad=True)
    link, xcat = encoder_ops.unit_encoder(torch.randn(4, 3, device=d), w_e, b_e, params[0], params[1], [u.to(d) for u in units],
                                          params[2:8], params[8:14])
    xm = xcat[..., 128:]
    assert torch.equal(xm, torch.ones_like(xm))
    assert torch.equal(xcat[..., :128], torch.zeros_like(xcat[..., :128]))      # relu(-1) == 0: a dead env encoder ...
    xcat.sum().backward()
    assert float(w_e.grad.abs().sum()) == 0.0 and float(b_e.grad.abs().sum()) == 0.0   # ... receives no gradient
    # bias gradient of group g == number of tokens routed to it: only unit 0 of each group gets d(max)
    for gidx in range(5):
        expect = 4.0 * (2.0 if gidx == 3 else 1.0)         # enh also receives the enemy-tower slot's gradient
        assert torch.allclose(params[8 + gidx].grad.cpu(), torch.full((128,), expect))
    assert float(params[13].grad.abs().sum()) == 0.0      # eth: no path from the maxima (policy.py:127)
    # the weight gradient of a tied group is carried by unit 0 alone: dW_g = d_emb_g^T basic_g with basic == 1
    assert torch.allclose(params[2 + 2].grad.cpu(), torch.full((128, 128), 4.0))


@pytest.mark.parametrize("lead,use_head", [((7,), True), ((3, 5), True), ((130,), True), ((33,), False), ((257,), True)])
def test_unit_encoder_with_target_unit_head(lead, use_head):
    """The training path: the [N,40,128] unit embedding is never materialised in forward -- the max-pool lives in the
    embedding GEMM's epilogue and the target-unit head runs through q = att [W_g | b_g] on the stored basic activations
    (policy.py:99-136,144-153).  Outputs and every gradient against plain torch autograd on the CPU, which DOES build it."""
    from dotaclient_b200 import encoder_ops
    g, env, w_e, b_e, w_b, b_b, units, weights, biases = _setup(lead, 17 + sum(lead))
    att = torch.randn(*lead, 128, generator=g).requires_grad_(True)
    ue_r, x_r = _reference(env, w_e, b_e, w_b, b_b, units, weights, biases)
    g_x = torch.randn(x_r.shape, generator=g)
    loss_r = (x_r * g_x).sum()
    if use_head:
        tu_r = torch.matmul(att.unsqueeze(-2), ue_r.transpose(-1, -2)).squeeze(-2)
        g_tu = torch.randn(tu_r.shape, generator=g)
        g_tu[..., ::2, :] = 0                              # tokens where the head was not used
        loss_r = loss_r + (tu_r * g_tu).sum()
    loss_r.backward()

    d = torch.device("cuda", 0)
    refs = [w_b, b_b] + weights + biases + [w_e, b_e]
    params = [t.detach().clone().to(d).requires_grad_(True) for t in refs]
    att_d = att.detach().to(d).requires_grad_(True)
    link, x = encoder_ops.unit_encoder(env.to(d), params[14], params[15], params[0], params[1], [u.to(d) for u in units],
                                       params[2:8], params[8:14])
    torch.testing.assert_close(x.detach().cpu(), x_r.detach(), rtol=1e-4, atol=2e-5)
    loss = (x * g_x.to(d)).sum()
    if use_head:
        tu = encoder_ops.target_unit(att_d, link)
        torch.testing.assert_close(tu.detach().cpu(), tu_r.detach(), rtol=1e-4, atol=1e-4)
        loss = loss + (tu * g_tu.to(d)).sum()
    loss.backward()
    n_tok = ue_r.numel() // (40 * 128)
    for mine, ref in zip(params, refs):
        expect = ref.grad if ref.grad is not None else torch.zeros_like(ref)   # e.g. the enemy-tower layer without the head
        torch.testing.assert_close(mine.grad.cpu(), expect, rtol=2e-4, atol=2e-6 * max(1, n_tok) * 16)
    if use_head:
        torch.testing.assert_close(att_d.grad.cpu(), att.grad, rtol=1e-4, atol=1e-4)


def _encoder_check():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "encoder_check.py")
    spec = importlib.util.spec_from_file_location("encoder_check", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("N,n_u,dx2", [(1, 16, False), (7, 5, False), (130, 16, True), (1000, 5, False), (1001, 16, True),
                                       (40000, 5, True), (40000, 5, False), (20011, 16, True), (20011, 16, False)])
def test_routed_wgrad_through_the_c_abi(N, n_u, dx2):
    """dc_unit_wgrad_routed: dW = R^T basic, db = colsum R with the max-pool routing R generated inside the kernel
    (30-row K-chunks of whole tokens for the 5-unit group, ragged last chunk) against the dense fp64 product; at N = 40000 /
    20011 every CTA runs several K-chunks.  The reduction has a fixed order: a repeated call is bitwise equal."""
    from dotaclient_b200 import _lib
    ec = _encoder_check()
    lib, st, dev = _lib.load(), _lib.stream_ptr(), torch.device("cuda", 0)
    inp, (dW_r, db_r, _, _) = ec.dense_reference(N, n_u, 11 + N, dx2, False)
    t = {k: v.to(dev).contiguous() for k, v in inp.items()}
    dW, db = torch.full((128, 128), 7.0, device=dev), torch.full((128,), 7.0, device=dev)
    ws = torch.empty(int(lib.dc_gemm_wgrad_workspace_bytes(128, 128)), dtype=torch.uint8, device=dev)
    dx = t["dx"].data_ptr()
    _lib.check(lib.dc_unit_wgrad_routed(dx + 4 * 256, dx + 4 * 640 if dx2 else None, 896, t["am"].data_ptr(), t["basic"].data_ptr(), N, n_u,
                                        dW.data_ptr(), db.data_ptr(), ws.data_ptr(), st), "dc_unit_wgrad_routed")
    torch.testing.assert_close(dW.cpu().double(), dW_r, rtol=1e-4, atol=2e-5 * max(1.0, float(dW_r.abs().max())))
    torch.testing.assert_close(db.cpu().double(), db_r, rtol=1e-4, atol=2e-5 * max(1.0, float(db_r.abs().max())))
    dW1, db1 = dW.clone(), db.clone()
    _lib.check(lib.dc_unit_wgrad_routed(dx + 4 * 256, dx + 4 * 640 if dx2 else None, 896, t["am"].data_ptr(), t["basic"].data_ptr(), N, n_u,
                                        dW.data_ptr(), db.data_ptr(), ws.data_ptr(), st), "dc_unit_wgrad_routed")
    assert torch.equal(dW, dW1) and torch.equal(db, db1)


@pytest.mark.parametrize("N,n_u,dx2,head,routed", [(1, 1, False, True, True), (7, 5, False, True, True), (130, 16, True, True, True),
                                                   (1000, 5, False, False, True), (1001, 16, False, True, True),
                                                   (300, 1, False, True, False), (26, 5, False, True, True),
                                                   (40000, 1, False, True, True), (40000, 1, False, False, True),
                                                   (40000, 5, True, True, True), (40000, 5, False, False, True),
                                                   (20011, 16, True, True, True), (20011, 16, False, False, True),
                                                   (20011, 16, False, True, False)])
def test_fused_dgrad_through_the_c_abi(N, n_u, dx2, head, routed):
    """dc_unit_dgrad_fused: dW_b, db_b of the shared basic layer from (d_xmax, argmax, dlogits, att) without d(embedding) or
    d_basic in memory -- routing and the rank-1 head term generated in the producers, ReLU mask recomputed in the epilogue --
    against the dense fp64 chain; 125-row tiles for the 5-unit group, tiles split over the two epilogue halves.  From N = 20011
    on there are more tiles than SMs, so each CTA carries its ring phase, its dW_b registers and the re-staged units across
    several tiles.  The reduction has a fixed order: a repeated call is bitwise equal."""
    from dotaclient_b200 import _lib
    ec = _encoder_check()
    lib, st, dev = _lib.load(), _lib.stream_ptr(), torch.device("cuda", 0)
    inp, (_, _, dwb_r, dbb_r) = ec.dense_reference(N, n_u, 5 + N, dx2, head, routed)
    t = {k: v.to(dev).contiguous() for k, v in inp.items()}
    wt = t["W"].t().contiguous()
    dwb, dbb = torch.full((128, 12), 7.0, device=dev), torch.full((128,), 7.0, device=dev)
    ws = torch.empty(int(lib.dc_unit_basic_bwd_workspace_bytes()), dtype=torch.uint8, device=dev)
    dx = t["dx"].data_ptr()
    args = (dx + 4 * 256 if routed else None, dx + 4 * 640 if dx2 else None, 896, t["am"].data_ptr() if (routed and n_u > 1) else None,
            t["dl"].data_ptr() + 4 * 3 if head else None, 40, t["att"].data_ptr() if head else None, wt.data_ptr(),
            t["units"].data_ptr(), t["w_b"].data_ptr(), t["b_b"].data_ptr(), N, n_u, dwb.data_ptr(), dbb.data_ptr())
    _lib.check(lib.dc_unit_dgrad_fused(*args, 0, ws.data_ptr(), st), "dc_unit_dgrad_fused")
    tol = dict(rtol=1e-4, atol=2e-5 * max(1.0, float(dwb_r.abs().max())))
    torch.testing.assert_close(dwb.cpu().double(), dwb_r, **tol)
    torch.testing.assert_close(dbb.cpu().double(), dbb_r, **tol)
    dwb1, dbb1 = dwb.clone(), dbb.clone()
    _lib.check(lib.dc_unit_dgrad_fused(*args, 1, ws.data_ptr(), st), "dc_unit_dgrad_fused")       # accumulate: twice the gradient
    torch.testing.assert_close(dwb.cpu().double(), 2 * dwb_r, **tol)
    _lib.check(lib.dc_unit_dgrad_fused(*args, 0, ws.data_ptr(), st), "dc_unit_dgrad_fused")
    assert torch.equal(dwb, dwb1) and torch.equal(dbb, dbb1)
    # bad arguments are reported, not launched
    assert lib.dc_unit_dgrad_fused(*args[:12], 3, *args[13:], 0, ws.data_ptr(), st) != 0


def _grid(g, shape, k, scale):
    """Integers in [-k, k] / scale: few significant bits, so sums of products of such values are exact in fp32 (and in each
    TF32 half) in any order, and ReLU masks and max-pool arg-maxes cannot differ from a float64 reference by rounding."""
    return torch.randint(-k, k + 1, shape, generator=g).float() / scale


def test_env_encoder_past_one_pass_vs_fp64():
    """dc_env_fwd / dc_env_bwd at N = 140001 rows of the 896-wide pre-rnn row: both grid-stride loops wrap (135168 rows per
    forward pass, 67584 per backward pass on 132 SMs).  Forward exact against float64 (grid inputs) and columns >= 128
    untouched; dW_e, db_e within 4e-6 of the sum of |terms| of float64; a repeated backward is bitwise equal."""
    from dotaclient_b200 import _lib
    lib, st, d = _lib.load(), _lib.stream_ptr(), torch.device("cuda", 0)
    N, ld = 140001, 896
    g = torch.Generator().manual_seed(140001)
    env, w_e, b_e = _grid(g, (N, 3), 48, 16), _grid(g, (128, 3), 32, 64), _grid(g, (128,), 8, 64)
    out_r = F.relu(env.double() @ w_e.double().t() + b_e.double())
    d_out = torch.randn(N, 128, generator=g)
    gm = d_out.double() * (out_r > 0)
    dw_r, db_r = gm.t() @ env.double(), gm.sum(0)
    dw_abs, db_abs = gm.abs().t() @ env.double().abs(), gm.abs().sum(0)

    out = torch.full((N, ld), 7.0, device=d)
    env_d, w_d, b_d = env.to(d), w_e.to(d), b_e.to(d)
    _lib.check(lib.dc_env_fwd(env_d.data_ptr(), w_d.data_ptr(), b_d.data_ptr(), out.data_ptr(), ld, N, st), "dc_env_fwd")
    assert torch.equal(out[:, :128].cpu().double(), out_r)
    assert bool((out[:, 128:] == 7.0).all())
    d_full = torch.zeros(N, ld, device=d)
    d_full[:, :128] = d_out.to(d)
    ws = torch.empty(int(lib.dc_env_bwd_workspace_bytes()), dtype=torch.uint8, device=d)
    results = []
    for _ in range(2):
        dw, db = torch.full((128, 3), 7.0, device=d), torch.full((128,), 7.0, device=d)
        _lib.check(lib.dc_env_bwd(d_full.data_ptr(), out.data_ptr(), ld, env_d.data_ptr(), dw.data_ptr(), db.data_ptr(), N,
                                  ws.data_ptr(), st), "dc_env_bwd")
        results.append((dw.cpu(), db.cpu()))
    (dw, db), (dw2, db2) = results
    assert ((dw.double() - dw_r).abs() <= 4e-6 * dw_abs).all(), float(((dw.double() - dw_r).abs() / dw_abs).max())
    assert ((db.double() - db_r).abs() <= 4e-6 * db_abs).all(), float(((db.double() - db_r).abs() / db_abs).max())
    assert torch.equal(dw, dw2) and torch.equal(db, db2)


def test_unit_encoder_with_target_unit_head_many_tiles_vs_fp64():
    """unit_encoder + target_unit forward and backward at lead (48, 128) = 6144 tokens, 245760 unit rows: the basic-layer
    loop wraps and each CTA of the 16-unit groups' fused data gradient runs about 6 tiles.  Inputs and weights on coarse
    grids make the forward exact, so the pre-rnn row must equal float64 exactly (arg-max ties included: the first unit
    wins on both sides); the target-unit logits and every gradient against float64 autograd."""
    from dotaclient_b200 import encoder_ops
    lead = (48, 128)
    g = torch.Generator().manual_seed(6144)
    env = _grid(g, (*lead, 3), 48, 16)
    w_e, b_e = _grid(g, (128, 3), 32, 64), _grid(g, (128,), 8, 64)
    w_b, b_b = _grid(g, (128, 12), 4, 8), _grid(g, (128,), 16, 32)
    units = [_grid(g, (*lead, n, 12), 4, 4) for n in UNITS]
    weights = [_grid(g, (128, 128), 8, 64) for _ in UNITS]
    biases = [_grid(g, (128,), 8, 64) for _ in UNITS]
    att = torch.randn(*lead, 128, generator=g)
    g_x = torch.randn(*lead, 7 * 128, generator=g)
    g_tu = torch.randn(*lead, 40, generator=g)
    g_tu[..., ::2, :] = 0                                  # tokens where the head was not used

    refs = [t.double().requires_grad_(True) for t in [w_b, b_b] + weights + biases + [w_e, b_e]]
    att_r = att.double().requires_grad_(True)
    ue_r, x_r = _reference(env.double(), refs[14], refs[15], refs[0], refs[1], [u.double() for u in units], refs[2:8],
                           refs[8:14])
    tu_r = torch.matmul(att_r.unsqueeze(-2), ue_r.transpose(-1, -2)).squeeze(-2)
    ((x_r * g_x.double()).sum() + (tu_r * g_tu.double()).sum()).backward()
    del ue_r

    d = torch.device("cuda", 0)
    params = [t.detach().float().to(d).requires_grad_(True) for t in refs]
    att_d = att.to(d).requires_grad_(True)
    link, x = encoder_ops.unit_encoder(env.to(d), params[14], params[15], params[0], params[1], [u.to(d) for u in units],
                                       params[2:8], params[8:14])
    assert torch.equal(x.detach().cpu().double(), x_r.detach())
    tu = encoder_ops.target_unit(att_d, link)
    ((x * g_x.to(d)).sum() + (tu * g_tu.to(d)).sum()).backward()
    tol = lambda ref: dict(rtol=0, atol=2e-5 * float(ref.detach().abs().max()))    # noqa: E731
    torch.testing.assert_close(tu.detach().cpu().double(), tu_r.detach(), **tol(tu_r))
    torch.testing.assert_close(att_d.grad.cpu().double(), att_r.grad, **tol(att_r.grad))
    for i, (mine, ref) in enumerate(zip(params, refs)):
        torch.testing.assert_close(mine.grad.cpu().double(), ref.grad, msg="parameter %d" % i, **tol(ref.grad))
