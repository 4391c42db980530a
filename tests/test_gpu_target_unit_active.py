"""GPU tests of the target-unit head on the active tokens (``Policy._head_outputs(..., active=(mask, action))``): the row list
of ``dc_target_rows``, and the compact branch (attention + head on ``rows[:count]``, every GEMM bounded by the device count)
against the dense branch on the same inputs -- logits bit for bit on the active rows and zero elsewhere, gradients equal up
to fp32 summation order, dW_att / db_att against float64 at the benchmark's 131,072 tokens -- at count 0, and replayed
from one captured graph on batches of different counts."""
import pytest
import torch

pytestmark = pytest.mark.gpu

FLOOR = 5e-5        # max|err| / max|f64| of the token-summed weight gradients (tests/test_gpu_wgrad_length.py)


def _masks(S, B, frac, seed):
    """target_unit (mask, action) rows [S, B, 40] (bool, on the GPU): a share `frac` of the tokens has a mask row with an
    action in it; a few tokens have a mask and no action, a few an action and no mask (both count as active)."""
    g = torch.Generator().manual_seed(seed)
    act = torch.rand(S, B, generator=g) < frac
    valid = torch.rand(S, B, 40, generator=g) < 0.5
    valid[..., 1] = True
    mask = valid & act.unsqueeze(-1)
    action = torch.zeros(S, B, 40, dtype=torch.bool)
    pick = torch.randint(1, 40, (S, B), generator=g)
    action.scatter_(2, pick.unsqueeze(-1), True)
    action &= act.unsqueeze(-1)
    only = torch.rand(S, B, generator=g)
    mask[only < 0.01] = False                              # action without a mask
    action[(only > 0.99) & act] = False                    # mask without an action
    return mask.cuda(), action.cuda()


@pytest.mark.parametrize("N,frac", [(131072, 0.25), (131072, 0.0), (131072, 1.0), (5003, 0.5), (1, 1.0)])
def test_target_rows_order_and_count(N, frac):
    from dotaclient_b200 import encoder_ops
    mask, action = _masks(1, N, frac, 11)
    rows, count, flags = encoder_ops.target_rows(mask, action)
    want = torch.nonzero((mask | action).any(-1).reshape(-1)).reshape(-1).to(torch.int32)
    n = int(count.item())
    assert n == want.numel()
    assert torch.equal(rows[:n], want)
    assert torch.equal(flags.bool(), (mask | action).any(-1).reshape(-1))
    if frac == 1.0:
        assert n == N and torch.equal(rows, torch.arange(N, dtype=torch.int32, device=rows.device))
    if frac == 0.0:
        assert n == 0


def _policy(H, cell, seed=5):
    from dotaclient_b200.policy import Policy
    torch.manual_seed(seed)
    return Policy(hidden_size=H, cell=cell).cuda()


def _obs(S, B, seed):
    from dotaclient_b200.synthetic import OBS_SHAPES
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn((S, B) + shp, generator=g).cuda() for k, shp in OBS_SHAPES.items()}


def _run(pol, obs, active, dl):
    """Forward + backward of the head on detached core outputs -> (logits, dy, {param: grad})."""
    pol.zero_grad(set_to_none=True)
    x, link = pol._encode(obs['env'], [obs[k] for k in pol.INPUT_KEYS[1:]])
    S, B = obs['env'].shape[:2]
    g = torch.Generator().manual_seed(3)
    y = (torch.randn(S, B, pol.hidden_size, generator=g) * 0.5).cuda().requires_grad_(True)
    packed, logits = pol._head_outputs(y, link, active)
    torch.autograd.backward([x, logits], [torch.zeros_like(x), dl])
    grads = {n: (None if p.grad is None else p.grad.clone()) for n, p in pol.named_parameters()}
    return logits.detach(), y.grad.clone(), grads, y.detach()


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("H,cell,S,B,frac", [(128, "lstm", 512, 256, 0.25), (256, "gru", 64, 64, 0.5)])
def test_compact_matches_dense(H, cell, S, B, frac):
    pol = _policy(H, cell)
    obs = _obs(S, B, 1)
    mask, action = _masks(S, B, frac, 2)
    act = (mask | action).any(-1)
    g = torch.Generator().manual_seed(4)
    dl = torch.randn(S, B, 40, generator=g).cuda() * act.unsqueeze(-1)         # the loss gives inactive rows zero dlogits
    l_d, dy_d, g_d, y = _run(pol, obs, None, dl)
    l_c, dy_c, g_c, _ = _run(pol, obs, (mask, action), dl)
    assert torch.equal(l_c[act], l_d[act])
    assert not l_c[~act].any()
    assert _rel(dy_c, dy_d) < 1e-5
    for name in g_d:
        assert (g_c[name] is None) == (g_d[name] is None), name
        if g_d[name] is not None and g_d[name].abs().max() > 0:
            assert _rel(g_c[name], g_d[name]) < 1e-4, name
    # dW_att / db_att against float64: d_att of the compact branch is s_c bm^T, rebuilt here from the dense branch's pieces
    link = pol._encode(obs['env'], [obs[k] for k in pol.INPUT_KEYS[1:]])[1]
    from dotaclient_b200 import encoder_ops
    bm = encoder_ops._head_matrix(link).double()
    idx = torch.nonzero(act.reshape(-1)).reshape(-1)
    s64 = _s_f64(link, dl.reshape(-1, 40), idx)
    d_att = s64 @ bm.t()                                                       # [n_act, 128]
    y64 = y.reshape(-1, H)[idx].double()
    dw64, db64 = d_att.t() @ y64, d_att.sum(0)
    assert _rel(g_c['affine_unit_attention.weight'], dw64) < FLOOR
    assert _rel(g_c['affine_unit_attention.bias'], db64) < FLOOR
    # the head's share of dW_g / db_g, att_c^T s_c over the active tokens (the product UnitEncoder.backward adds), against float64
    w_att, b_att = pol.affine_unit_attention.weight, pol.affine_unit_attention.bias
    rows, count, flags = encoder_ops.target_rows(mask, action)
    lg = encoder_ops.target_unit_rows(y, w_att, b_att, link, rows, count, flags)
    lg.backward(dl)
    _, _, s_c, att_c, cnt = link.pop("pending")
    from dotaclient_b200 import ops
    dw_head, _ = ops.gemm_wgrad_tf32x3(att_c, s_c, want_bias=False, t_dev=cnt)
    att64 = y64 @ w_att.detach().double().t() + b_att.detach().double()
    assert _rel(dw_head, att64.t() @ s64) < FLOOR


def _s_f64(link, dl, idx):
    """s[i] = [sum_u dl[n,u] basic_g[n,u,:] for g] + [sum_u dl[n,u] for g] + zeros, n = idx[i], in float64."""
    from dotaclient_b200.encoder_ops import OFFSETS, UNITS, QW, C
    w_b, b_b = link["w_b"].double(), link["b_b"].double()
    out = torch.zeros(idx.numel(), QW, dtype=torch.float64, device=dl.device)
    for g, (nu, off) in enumerate(zip(UNITS, OFFSETS)):
        u = link["units"][g].reshape(-1, nu, 12)[idx].double()
        basic = torch.relu(u @ w_b.t() + b_b)                                 # [n, nu, 128]
        d = dl[idx, off:off + nu].double()
        out[:, g * C:(g + 1) * C] = torch.einsum("nu,nuc->nc", d, basic)
        out[:, 6 * C + g] = d.sum(1)
    return out


def test_count_zero():
    pol = _policy(128, "lstm")
    S, B = 64, 32
    obs = _obs(S, B, 7)
    mask = torch.zeros(S, B, 40, dtype=torch.bool, device="cuda")
    dl = torch.zeros(S, B, 40, device="cuda")
    l_d, dy_d, g_d, _ = _run(pol, obs, None, dl)
    l_c, dy_c, g_c, _ = _run(pol, obs, (mask, mask), dl)
    assert not l_c.any()
    assert not dy_c.any()
    for name in g_d:
        assert (g_c[name] is None) == (g_d[name] is None), name
    for name in ('affine_unit_attention.weight', 'affine_unit_attention.bias'):
        assert not g_c[name].any(), name
        assert torch.equal(g_c[name], g_d[name]), name


def test_graph_replay_two_counts():
    """One captured forward + backward of the compact branch, replayed on two batches of different active counts: the
    results of eager runs on the same inputs."""
    pol = _policy(128, "lstm")
    S, B = 128, 64
    obs = _obs(S, B, 9)
    x, link = pol._encode(obs['env'], [obs[k] for k in pol.INPUT_KEYS[1:]])
    link = {k: v for k, v in link.items()}
    y = (torch.randn(S, B, 128, generator=torch.Generator().manual_seed(3)) * 0.5).cuda()
    inputs = [_masks(S, B, f, 20 + i) for i, f in enumerate((0.3, 0.7))]
    dls = [torch.randn(S, B, 40).cuda() * (m | a).any(-1, keepdim=True) for m, a in inputs]
    w, b = pol.affine_unit_attention.weight, pol.affine_unit_attention.bias
    from dotaclient_b200 import encoder_ops

    def step(mask, action, dl):
        w.grad = b.grad = None
        yy = y.detach().requires_grad_(True)
        lg = encoder_ops.target_unit_rows(yy, w, b, link, *encoder_ops.target_rows(mask, action))
        lg.backward(dl)
        link.pop("pending", None)
        return lg.detach().clone(), yy.grad.clone(), w.grad.clone(), b.grad.clone()

    eager = [step(m, a, d) for (m, a), d in zip(inputs, dls)]
    sm, sa, sd = (t.clone() for t in (*inputs[0], dls[0]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(sm, sa, sd)                                    # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step(sm, sa, sd)
    for (m, a), d, want in zip(inputs, dls, eager):
        sm.copy_(m), sa.copy_(a), sd.copy_(d)
        graph.replay()
        torch.cuda.synchronize()
        for got, exp in zip(out, want):
            assert torch.equal(got, exp)
