"""GPU tests of sequence packing: the recurrence with state resets (``dc_rnn_seq_fwd_reset`` / ``_bwd_reset`` through
``ops.rnn_sequence(reset=...)``) against a float64 reference that runs every segment on its own, the reset path without
resets against the plain one, and the packed training step (``pack_sequences=True``) against the unpacked masked step."""
import copy
import pickle
import uuid

import numpy as np
import pytest
import torch

from dotaclient_b200.synthetic import make_rollout, split_rollout

pytestmark = pytest.mark.gpu

WEIGHTS = ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0")
# (K, FLOOR) as tests/test_gpu_rnn_fp64.py: max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|
FORWARD_BOUND = (16.0, 1e-6)
STATE_GRAD_BOUND = (32.0, 1e-6)
WEIGHT_GRAD_BOUND = (4.0, 5e-4)


def dev():
    return torch.device("cuda", 0)


# ------------------------------------------------------------------------------------------------ recurrence with resets
def reset_pattern(S, B):
    """reset_slot [S, B] int32 and K: per column, by b % 6, no reset / t = 0 / t = 1 and S-1 / consecutive t = 5, 6 /
    three resets / t = S-1 only."""
    slot = np.full((S, B), -1, dtype=np.int32)
    for b in range(B):
        ts = [[], [0], [1, S - 1], [5, 6], [3, 9, 15], [S - 1]][b % 6]
        for k, t in enumerate(ts):
            slot[t, b] = k
    return slot, 3


def segmented_reference(cell, w, x, h0, c0, slot, h_tab, c_tab, dy, dhn, dcn, dtype):
    """torch's CPU GRU / LSTM in ``dtype``, every segment of every column run on its own from its start state (h0 / c0,
    or the table row of its reset): outputs and the gradients of <y, dy> + <h_n, dhn> (+ <c_n, dcn>)."""
    S, B, H = x.shape
    m = (torch.nn.GRU if cell == "gru" else torch.nn.LSTM)(H, H).to(dtype)
    with torch.no_grad():
        for k in WEIGHTS:
            getattr(m, k).copy_(w[k])
    xr = x.to(dtype, copy=True).requires_grad_(True)
    h0r = h0.to(dtype, copy=True).requires_grad_(True)
    c0r = c0.to(dtype, copy=True).requires_grad_(True) if cell == "lstm" else None
    ys, hns, cns, loss = [], [], [], 0.0
    for b in range(B):
        starts = [0] + [t for t in range(1, S) if slot[t, b] >= 0] + [S]
        col = []
        for t0, t1 in zip(starts, starts[1:]):
            k = int(slot[t0, b])
            if k >= 0:
                h = h_tab[k, b].to(dtype).view(1, 1, H)
                c = c_tab[k, b].to(dtype).view(1, 1, H) if cell == "lstm" else None
            else:
                h = h0r[b].view(1, 1, H)
                c = c0r[b].view(1, 1, H) if cell == "lstm" else None
            if cell == "lstm":
                y, (hn, cn) = m(xr[t0:t1, b:b + 1], (h, c))
            else:
                y, hn = m(xr[t0:t1, b:b + 1], h)
                cn = None
            col.append(y)
        ys.append(torch.cat(col))
        hns.append(hn[0, 0])
        cns.append(None if cn is None else cn[0, 0])
    y = torch.cat(ys, dim=1)
    hn = torch.stack(hns)
    loss = (y * dy.to(dtype)).sum() + (hn * dhn.to(dtype)).sum()
    if cell == "lstm":
        cn = torch.stack(cns)
        loss = loss + (cn * dcn.to(dtype)).sum()
    loss.backward()
    zero = torch.zeros_like(h0r)
    out = {"y": y.detach(), "h_n": hn.detach(), "dx": xr.grad, "dh0": h0r.grad if h0r.grad is not None else zero}
    if cell == "lstm":
        out.update(c_n=cn.detach(), dc0=c0r.grad if c0r.grad is not None else zero)
    out.update({k: getattr(m, k).grad for k in WEIGHTS})
    return out


def bound_check(got, f64, f32, names, bound):
    k, floor = bound
    over = []
    for n in names:
        ref = f64[n]
        err = float((got[n].double().cpu() - ref).abs().max())
        cal = float((f32[n].double() - ref).abs().max())
        if not err <= k * cal + floor * float(ref.abs().max()):
            over.append("%s: max|err| %.3e, torch fp32 %.3e, max|f64| %.3e" % (n, err, cal, float(ref.abs().max())))
    return over


def gpu_run(cell, w, x, h0, c0, dy, dhn, dcn, reset):
    from dotaclient_b200 import ops
    p = [w[k].to(dev()).clone().requires_grad_(True) for k in WEIGHTS]
    xg = x.to(dev()).requires_grad_(True)
    h0g = h0.to(dev()).requires_grad_(True)
    c0g = c0.to(dev()).requires_grad_(True) if cell == "lstm" else None
    if reset is not None:
        reset = tuple(None if t is None else t.to(dev()) for t in reset)
    y, hn, cn = ops.rnn_sequence(xg, *p, h0g, c0g, cell, reset)
    outs, grads = [y, hn], [dy.to(dev()), dhn.to(dev())]
    if cell == "lstm":
        outs.append(cn)
        grads.append(dcn.to(dev()))
    torch.autograd.backward(outs, grads)
    r = {"y": y.detach(), "h_n": hn.detach(), "dx": xg.grad, "dh0": h0g.grad}
    if cell == "lstm":
        r.update(c_n=cn.detach(), dc0=c0g.grad)
    r.update({k: t.grad for k, t in zip(WEIGHTS, p)})
    return {k: v.cpu() for k, v in r.items()}


def make_case(cell, H, S, B, seed):
    torch.manual_seed(seed)
    m = (torch.nn.GRU if cell == "gru" else torch.nn.LSTM)(H, H)
    w = {k: getattr(m, k).detach().clone() for k in WEIGHTS}
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(S, B, H, generator=g)
    h0, c0 = 0.5 * torch.randn(B, H, generator=g), 0.5 * torch.randn(B, H, generator=g)
    slot, K = reset_pattern(S, B)
    h_tab, c_tab = 0.5 * torch.randn(K, B, H, generator=g), 0.5 * torch.randn(K, B, H, generator=g)
    dy, dhn, dcn = torch.randn(S, B, H, generator=g), torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
    return w, x, h0, c0, torch.from_numpy(slot), h_tab, c_tab, dy, dhn, dcn


# H 128 resident, 256 cluster (B 37: a partly filled second cluster), 512 step-wise, 192 and 96 generic
@pytest.mark.parametrize("H", [128, 256, 512, 192, 96])
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_resets_vs_segmented_fp64(cell, H):
    S, B = 24, 37
    w, x, h0, c0, slot, h_tab, c_tab, dy, dhn, dcn = make_case(cell, H, S, B, 11 + H)
    reset = (slot.to(torch.int32), h_tab, c_tab if cell == "lstm" else None)
    got = gpu_run(cell, w, x, h0, c0, dy, dhn, dcn, reset)
    args = (cell, w, x, h0, c0, slot.numpy(), h_tab, c_tab, dy, dhn, dcn)
    f64, f32 = segmented_reference(*args, torch.float64), segmented_reference(*args, torch.float32)
    fwd = ("y", "h_n", "c_n") if cell == "lstm" else ("y", "h_n")
    st = ("dx", "dh0", "dc0") if cell == "lstm" else ("dx", "dh0")
    over = bound_check(got, f64, f32, fwd, FORWARD_BOUND) + bound_check(got, f64, f32, st, STATE_GRAD_BOUND) + \
        bound_check(got, f64, f32, WEIGHTS, WEIGHT_GRAD_BOUND)
    assert not over, over
    # a reset at t = 0 makes h0 / c0 unused: their gradient is exactly zero there
    first = slot[0] >= 0
    assert bool((got["dh0"][first] == 0).all())
    if cell == "lstm":
        assert bool((got["dc0"][first] == 0).all())


@pytest.mark.parametrize("H", [128, 256, 512, 96])
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_reset_path_without_resets_is_bit_identical(cell, H):
    """Every slot at -1: the _reset entry points (and the dW_hh correction, all weights 0) reproduce the plain ones bit
    for bit."""
    S, B = 20, 35
    w, x, h0, c0, _, h_tab, c_tab, dy, dhn, dcn = make_case(cell, H, S, B, 5 + H)
    none = torch.full((S, B), -1, dtype=torch.int32)
    plain = gpu_run(cell, w, x, h0, c0, dy, dhn, dcn, None)
    reset = gpu_run(cell, w, x, h0, c0, dy, dhn, dcn, (none, h_tab, c_tab if cell == "lstm" else None))
    for k in plain:
        assert torch.equal(plain[k], reset[k]), k


# ------------------------------------------------------------------------------------------------ packed training step
def make_optimizer(tmp_path, hidden_size=128, cell="lstm", num_layers=1, seq_len=16, min_seq=1, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="packing", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=min_seq,
                         seq_len=seq_len, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=hidden_size, cell=cell, num_layers=num_layers, **kw)


LENGTHS = (40, 23, 48, 7, 33, 5, 19, 61)          # S = 16: tails 8, 7, -, 7, 1, 5, 3, 13


def ragged_rollouts(pol, seed, vtrace, carried):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, L in enumerate(LENGTHS):
        cut = carried and i % 2 == 0
        r = make_rollout(L + (1 if cut else 0), 100 * seed + i, game_id=i)
        if cut:
            r = split_rollout(r, [L])[0]                                   # non-terminal: the game goes on
        if vtrace:
            r["behaviour_logp"] = -torch.rand(L, 5, generator=g).numpy()
        if carried:
            h = 0.5 * torch.randn(pol.num_layers, 1, pol.hidden_size, generator=g)
            r["initial_hidden"] = (h, 0.5 * torch.randn(h.shape, generator=g)) if pol.cell == "lstm" else h
        out.append(r)
    return out


def _close(a, b, rel, abs_=0.0):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    return float((a - b).abs().max()) <= rel * float(b.abs().max()) + abs_


@pytest.mark.parametrize("H,cell,layers", [(128, "lstm", 1), (256, "gru", 1), (128, "lstm", 2)])
@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
@pytest.mark.parametrize("carried", [False, True])
def test_packed_step_equals_unpacked_masked_step(H, cell, layers, estimator, carried, tmp_path):
    kw = dict(hidden_size=H, cell=cell, num_layers=layers, advantage_estimator=estimator, mask_padding=True)
    unpacked = make_optimizer(tmp_path, **kw)
    packed = make_optimizer(tmp_path, pack_sequences=True, **kw)
    rollouts = ragged_rollouts(unpacked.policy_base, 3, estimator == "vtrace", carried)
    bu = unpacked.batch_from_rollouts(copy.deepcopy(rollouts))
    bp = packed.batch_from_rollouts(copy.deepcopy(rollouts))
    assert bp.batch_size < bu.batch_size and bp.reset_h.shape[0] >= 1
    assert int(bp.valid.sum()) == int(bu.valid.sum()) == sum(LENGTHS)
    for step in range(2):
        lu, eu, gu = unpacked.train(bu)
        lp, ep, gp = packed.train(bp)
        for k in lu:
            assert _close(lp[k], lu[k], 2e-4, 2e-6), (step, k, float(lp[k]), float(lu[k]))
        for k in eu:
            assert _close(ep[k], eu[k], 2e-4, 2e-6), (step, k, float(ep[k]), float(eu[k]))
        for k in gu:
            assert _close(gp[k], gu[k], 2e-3), (step, k, float(gp[k]), float(gu[k]))
        for k, v in unpacked.last_ppo_stats.items():
            assert abs(packed.last_ppo_stats[k] - v) <= 2e-4 * abs(v) + 2e-5, (step, k, packed.last_ppo_stats[k], v)
        fu, fp = unpacked.flat, packed.flat
        for name, lo, hi in zip(fu.names, fu.starts, fu.ends):
            assert _close(fp.grad[lo:hi], fu.grad[lo:hi], 2e-3, 1e-9), (step, "grad", name)
        assert _close(fp.param, fu.param, 0.0, 1e-6), (step, "weights")
        assert _close(packed.exp_avg, unpacked.exp_avg, 2e-3, 1e-12) and torch.equal(packed.adam_steps, unpacked.adam_steps)


def test_packed_minibatch_gather_equals_direct_assembly(tmp_path):
    opt = make_optimizer(tmp_path, hidden_size=128, cell="lstm", num_layers=2, mask_padding=True, pack_sequences=True)
    batch = opt.batch_from_rollouts(ragged_rollouts(opt.policy_base, 4, False, True))
    idx = np.random.default_rng(2).permutation(batch.batch_size)[: batch.batch_size // 2 + 1]
    got = batch.gather(idx)
    index = torch.as_tensor(idx, device=dev())
    want = batch.map(lambda v: v.index_select(1, index))
    for (_, k, a), (_, _, b) in zip(got.tensors(), want.tensors()):
        assert torch.equal(a, b), k
    assert got.graph_key() == want.graph_key()


def test_graph_replayed_packed_step_equals_eager(tmp_path):
    kw = dict(hidden_size=128, cell="gru", num_layers=2, mask_padding=True, pack_sequences=True)
    graphed, eager = make_optimizer(tmp_path, **kw), make_optimizer(tmp_path, **kw)
    eager.use_cuda_graph = False
    rollouts = ragged_rollouts(graphed.policy_base, 5, False, False)
    bg, be = graphed.batch_from_rollouts(copy.deepcopy(rollouts)), eager.batch_from_rollouts(copy.deepcopy(rollouts))
    for step in range(3):                          # eager (first sight), capture + replay, replay
        lg, _, _ = graphed.train(bg)
        le, _, _ = eager.train(be)
        assert all(torch.equal(torch.as_tensor(lg[k]), torch.as_tensor(le[k])) for k in lg), step
        assert torch.equal(graphed.flat.param, eager.flat.param), step
    assert any(not isinstance(v, str) for v in graphed._graphs.values())


def test_run_iteration_reports_packing(tmp_path):
    S = 16
    opt = make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=S, min_seq=6, mask_padding=True,
                         pack_sequences=True)
    for i, L in enumerate(LENGTHS):
        opt.mq.publish_experience(pickle.dumps(make_rollout(L, 900 + i, game_id=i)))
    m = opt.run_iteration(1)
    from dotaclient_b200.optimizer import sequence_count
    pulled = [L for L in LENGTHS][:next(n for n in range(1, len(LENGTHS) + 1)
                                        if sequence_count(LENGTHS[:n], S, pack=True) >= 6)]
    B_packed, B_unpacked = sequence_count(pulled, S, pack=True), sequence_count(pulled, S)
    assert m['packing_saved_fraction'] == pytest.approx(1 - B_packed / B_unpacked)
    assert m['padding_fraction'] == pytest.approx((B_packed * S - sum(pulled)) / (B_packed * S))
    assert np.isfinite(float(m['loss/sum']))
