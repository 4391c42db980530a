"""GPU parity of the stacked recurrent core (``num_layers`` > 1): the chained recurrence kernels against torch's multi-layer
nn.GRU / nn.LSTM, and the whole optimizer (experience prep, train(), CUDA graph, actor pool, checkpoints) against the
stacked CPU oracle (``stacked_oracle.py``).  Checks and tolerances are those of the single-layer tests in
test_gpu_parity.py; every layer runs on the recurrence kernel its width selects."""
import copy
import io
import os
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_parity as P  # noqa: E402
from stacked_oracle import StackedRefPolicy, make_stacked_ref_optimizer  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu


def make_optimizer(hidden_size, cell, seq_len, tmp_path, num_layers=2, checkpoint=False, pretrained_model=None):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="test", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=1,
                         seq_len=seq_len, learning_rate=5e-5, checkpoint=checkpoint, pretrained_model=pretrained_model,
                         mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=hidden_size, cell=cell, num_layers=num_layers)


def make_oracle(hidden_size, cell, seq_len, num_layers=2):
    return make_stacked_ref_optimizer(hidden_size, cell, seq_len, num_layers)


# ------------------------------------------------------------------------------------------------ chained recurrence
# (B, S, H): H = 128 one-SM kernels (B = 37: the last CTA partly filled), H = 256 cluster kernels (B = 33: the last cluster
# partly filled), H = 512 step-wise kernels, H = 96 generic kernels
@pytest.mark.parametrize("L", [2, 3])
@pytest.mark.parametrize("cell", ["gru", "lstm"])
@pytest.mark.parametrize("B,S,H", [(37, 9, 128), (33, 9, 256), (3, 5, 512), (5, 16, 96)])
def test_stacked_rnn_forward_backward_vs_torch(L, cell, B, S, H):
    """ops.rnn_sequence chained over L layers (layer k's input = layer k-1's output view) against nn.GRU / nn.LSTM
    (num_layers=L) on the CPU: output, every layer's h_n / c_n, dx, every layer's dh0 / dc0, every weight and bias
    gradient.  Tolerances of test_rnn_forward_backward_vs_torch."""
    from dotaclient_b200 import ops
    torch.manual_seed(L * 100000 + B * 1000 + S * 10 + H)
    ref = (torch.nn.GRU if cell == "gru" else torch.nn.LSTM)(input_size=H, hidden_size=H, num_layers=L)
    lstm = cell == "lstm"
    x = torch.randn(S, B, H)
    h0 = torch.randn(L, B, H) * 0.5
    c0 = torch.randn(L, B, H) * 0.5
    wy, wh, wc = torch.randn(S, B, H), torch.randn(L, B, H), torch.randn(L, B, H)

    xr = x.clone().requires_grad_(True)
    h0r, c0r = h0.clone().requires_grad_(True), c0.clone().requires_grad_(True)
    if lstm:
        yr, (hn, cn) = ref(xr, (h0r, c0r))
        loss = (yr * wy).sum() + (hn * wh).sum() + (cn * wc).sum()
    else:
        yr, hn = ref(xr, h0r)
        loss = (yr * wy).sum() + (hn * wh).sum()
    loss.backward()

    d = P.dev()
    p = {k: v.detach().clone().to(d).requires_grad_(True) for k, v in ref.named_parameters()}
    xg = x.to(d).requires_grad_(True)
    h0g = h0.to(d).requires_grad_(True)
    c0g = c0.to(d).requires_grad_(True) if lstm else None
    y, hs, cs = xg, [], []
    for k in range(L):
        w = [p["%s_l%d" % (n, k)] for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        y, hk, ck = ops.rnn_sequence(y, *w, h0g[k], c0g[k] if lstm else None, cell)
        hs.append(hk)
        cs.append(ck)
    hng = torch.stack(hs)
    lg = (y * wy.to(d)).sum() + (hng * wh.to(d)).sum()
    if lstm:
        cng = torch.stack(cs)
        lg = lg + (cng * wc.to(d)).sum()
    lg.backward()
    torch.testing.assert_close(y.detach().cpu(), yr.detach(), rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(hng.detach().cpu(), hn.detach(), rtol=1e-4, atol=2e-5)
    if lstm:
        torch.testing.assert_close(cng.detach().cpu(), cn.detach(), rtol=1e-4, atol=2e-5)
    scale = max(1.0, float(S))
    torch.testing.assert_close(xg.grad.cpu(), xr.grad, rtol=2e-4, atol=2e-6 * scale)
    torch.testing.assert_close(h0g.grad.cpu(), h0r.grad, rtol=2e-4, atol=2e-6 * scale)
    if lstm:
        torch.testing.assert_close(c0g.grad.cpu(), c0r.grad, rtol=2e-4, atol=2e-6 * scale)
    for k, v in ref.named_parameters():
        torch.testing.assert_close(p[k].grad.cpu(), v.grad, rtol=5e-4, atol=5e-6 * scale * B, msg=k)


# ------------------------------------------------------------------------------------------------ optimizer
@pytest.mark.parametrize("H,cell,S", [(128, "lstm", 16), (256, "gru", 16), (96, "gru", 16)])
def test_stacked_optimizer_step_vs_oracle(H, cell, S, tmp_path):
    """L = 2: experience prep on ragged rollouts of several chunks (every layer's hidden state at the chunk boundaries, old
    log-probs, advantages, returns) + three train() epochs against the stacked oracle: losses, entropies, grad norms,
    per-tensor gradients and the Adam update -- the checks of test_optimizer_step_vs_oracle."""
    torch.set_num_threads(4)
    mine = make_optimizer(H, cell, S, tmp_path)
    oracle = make_oracle(H, cell, S)
    sd_m, sd_o = mine.policy_base.state_dict(), oracle.policy_base.state_dict()
    assert list(sd_m) == list(sd_o) and len(sd_m) == 38
    for k in sd_m:
        assert torch.equal(sd_m[k].cpu(), sd_o[k]), k
    rollouts = P._rollouts(3, S, seed=H + S)
    assert sum((r["rewards"].shape[0] + S - 1) // S for r in rollouts) > 3          # several chunks per rollout
    xs_m = [s for grp in mine.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in grp]
    xs_o = [s for r in rollouts for s in oracle.experiences_from_rollout(copy.deepcopy(r))]
    for s in xs_m:
        for t in (s.hidden if cell == "lstm" else (s.hidden,)):
            assert t.shape == (2, 1, H)
    P._compare_sequences(xs_m, xs_o, cell)
    for ep in range(3):
        lm, em, gm = mine.train(xs_m)
        lo, eo, go = oracle.train(xs_o)
        for k in lo:
            np.testing.assert_allclose(float(lm[k]), float(lo[k]), rtol=2e-4, atol=2e-6, err_msg="%s ep%d" % (k, ep))
        for k in eo:
            np.testing.assert_allclose(float(em[k]), float(eo[k]), rtol=2e-4, atol=1e-6, err_msg="entropy %s" % k)
        np.testing.assert_allclose(float(gm["unclipped"]), float(go["unclipped"]), rtol=2e-3)
        np.testing.assert_allclose(float(gm["clipped"]), float(go["clipped"]), rtol=2e-3)
        if ep == 0:
            for name, p in oracle.policy_base.named_parameters():
                g = mine.flat.grad_of(name).cpu()
                assert p.grad is not None
                cos = torch.nn.functional.cosine_similarity(g.flatten(), p.grad.flatten(), dim=0)
                assert cos > 0.9999, (name, float(cos))
                np.testing.assert_allclose(float(g.norm()), float(p.grad.norm()), rtol=2e-3, err_msg=name)
    init = make_oracle(H, cell, S).policy_base.state_dict()
    dm = torch.cat([(a.cpu() - init[k]).flatten() for k, a in mine.policy_base.state_dict().items()])
    do = torch.cat([(b - init[k]).flatten() for k, b in oracle.policy_base.state_dict().items()])
    assert float(do.abs().max()) > 5e-5
    cos = torch.nn.functional.cosine_similarity(dm, do, dim=0)
    assert cos > 0.995, float(cos)
    assert float((dm - do).abs().max()) <= 3 * 2 * 5e-5 + 1e-6


def test_stacked_graph_replay_equals_launch_by_launch(tmp_path):
    """L = 2: train() replayed from the CUDA graph == launch by launch over five steps (parameters, exp_avg, adam_steps)."""
    S, B = 16, 6
    a = make_optimizer(128, "lstm", S, tmp_path)
    b = make_optimizer(128, "lstm", S, tmp_path)
    b.use_cuda_graph = False
    rollouts = [make_rollout(S, 40 + i) for i in range(B)]
    batch_a = a.batch_from_rollouts(copy.deepcopy(rollouts))
    batch_b = b.batch_from_rollouts(copy.deepcopy(rollouts))
    assert batch_a.h0.shape == batch_a.c0.shape == (2, B, 128)
    for step in range(5):
        la, _, ga = a.train(batch_a)
        lb, _, gb = b.train(batch_b)
        for k in la:
            np.testing.assert_allclose(float(la[k]), float(lb[k]), rtol=1e-6, atol=1e-9, err_msg="%s step %d" % (k, step))
        np.testing.assert_allclose(float(ga["unclipped"]), float(gb["unclipped"]), rtol=1e-6)
    assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"
    assert not any(isinstance(v, tuple) for v in b._graphs.values())
    torch.testing.assert_close(a.flat.param, b.flat.param, rtol=1e-6, atol=1e-9)
    torch.testing.assert_close(a.exp_avg, b.exp_avg, rtol=1e-5, atol=1e-12)
    assert torch.equal(a.adam_steps, b.adam_steps)


@pytest.mark.parametrize("H,cell", [(128, "lstm"), (256, "gru")])
def test_stacked_batch_from_rollouts_equals_stacked_sequences(H, cell, tmp_path):
    """L = 2: batch_from_rollouts == ExperienceBatch.from_sequences(experiences_from_rollout(...)), h0 / c0 [2, B, H]
    bit-identical; then the ragged (several chunks per rollout) path against experiences_from_rollouts."""
    from dotaclient_b200.optimizer import ExperienceBatch
    S = 16
    mine = make_optimizer(H, cell, S, tmp_path)
    rollouts = [make_rollout(S, 70 + i) for i in range(5)]
    fast = mine.batch_from_rollouts(copy.deepcopy(rollouts))
    slow = ExperienceBatch.from_sequences([s for r in rollouts for s in mine.experiences_from_rollout(copy.deepcopy(r))],
                                          P.dev())
    assert fast.h0.shape == (2, 5, H) and (fast.c0 is None) == (cell == "gru")
    for (_, ka, a), (_, kb, b) in zip(fast.tensors(), slow.tensors()):
        assert ka == kb and a.shape == b.shape, (ka, a.shape, b.shape)
        if a.dtype == torch.bool or ka in ("h0", "c0"):
            assert torch.equal(a, b), ka
        else:
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6, msg=ka)
    ragged = [make_rollout(L, 80 + i) for i, L in enumerate((S, 2 * S + 3, S - 5, 4 * S))]
    general = mine.batch_from_rollouts(copy.deepcopy(ragged))
    assert general.batch_size == 1 + 3 + 1 + 4 and general.h0.shape == (2, 9, H)
    slow2 = ExperienceBatch.from_sequences([s for grp in mine.experiences_from_rollouts(copy.deepcopy(ragged)) for s in grp],
                                           P.dev())
    for (_, ka, a), (_, kb, b) in zip(general.tensors(), slow2.tensors()):
        assert ka == kb and a.shape == b.shape, (ka, a.shape, b.shape)
        if a.dtype == torch.bool or ka in ("h0", "c0"):
            assert torch.equal(a, b), ka
        else:
            torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7, msg=ka)
    assert not torch.equal(general.h0[0], general.h0[1])           # the layers carry their own states


@pytest.mark.parametrize("H,cell", [(96, "gru"), (128, "lstm")])
def test_stacked_act_batched_pool_matches_per_agent_sequence(H, cell, tmp_path):
    """L = 2 actor pool step: A agents through one batched forward with carried [2, A, H] state + one selection launch ==
    each agent's own oracle sequence() followed by the pinned index function, over two steps."""
    from oracle.ref_policy import sample_index
    A = 37
    lstm = cell == "lstm"
    mine = make_optimizer(H, cell, 8, tmp_path).policy_base
    oracle = make_oracle(H, cell, 8).policy_base
    d = P.dev()
    g = torch.Generator().manual_seed(5)
    rolls = [make_rollout(2, 600 + a) for a in range(A)]
    z = torch.zeros(2, A, H, device=d)
    hid_m = (z, z.clone()) if lstm else z
    hid_o = [oracle.init_hidden() for _ in range(A)]
    for t in range(2):
        obs = {k: torch.stack([r["observations"][k][t] for r in rolls]) for k in mine.INPUT_KEYS}
        masks = {k: torch.rand(A, n, generator=g) < 0.7 for k, n in zip(P.HEADS, P.SIZES)}
        for k in masks:
            masks[k][:, 1 if k == "target_unit" else 0] = True
        u = torch.rand(A, 5, generator=g)
        chosen, logp, logits, value, hid_m = mine.act_batched(hid_m, {k: v.to(d) for k, v in obs.items()},
                                                              {k: v.to(d) for k, v in masks.items()}, u.to(d))
        follow = {0: (), 1: ("x", "y"), 2: ("target_unit",), 3: ("ability",)}
        for a in range(A):
            with torch.no_grad():
                lo, vo, hid_o[a] = oracle.sequence(hidden=hid_o[a], **{k: v[a:a + 1] for k, v in obs.items()})
            for k in P.HEADS:
                torch.testing.assert_close(logits[k][a].cpu(), lo[k][0, 0], rtol=1e-4, atol=3e-5)
            torch.testing.assert_close(value[a].cpu(), vo[0, 0, 0], rtol=1e-4, atol=3e-5)
            e = sample_index(logits["enum"][a].cpu(), masks["enum"][a], float(u[a, 0]))
            assert int(chosen["enum"][a]) == e
            for h, k in enumerate(P.HEADS):
                if k == "enum":
                    continue
                want = sample_index(logits[k][a].cpu(), masks[k][a], float(u[a, h])) if k in follow[e] else -1
                assert int(chosen[k][a]) == want, (t, a, k)
        for i, got in enumerate(hid_m if lstm else (hid_m,)):
            assert got.shape == (2, A, H)
            want = torch.cat([(h[i] if lstm else h) for h in hid_o], dim=1)
            torch.testing.assert_close(got.cpu(), want, rtol=1e-4, atol=3e-5)


def test_stacked_policy_forward_batch_first_matches_time_major(tmp_path):
    """L = 2: Policy.forward (batch-first inputs, [L, B, H] state) == forward_time_major, and == the stacked oracle."""
    mine = make_optimizer(128, "lstm", 8, tmp_path)
    oracle = make_oracle(128, "lstm", 8)
    B, S = 3, 8
    rolls = [make_rollout(S, 40 + i) for i in range(B)]
    obs_bf = {k: torch.stack([r["observations"][k] for r in rolls]) for k in mine.policy_base.INPUT_KEYS}
    h = torch.randn(2, B, 128) * 0.3
    c = torch.randn(2, B, 128) * 0.3
    d = P.dev()
    with torch.no_grad():
        lo, vo, (hn, cn) = oracle.policy_base(**obs_bf, hidden=(h, c))
        lm, vm, (hm, cm) = mine.policy_base(**{k: v.to(d) for k, v in obs_bf.items()}, hidden=(h.to(d), c.to(d)))
        lt, vt, (ht, ct) = mine.policy_base.forward_time_major(
            {k: v.transpose(0, 1).contiguous().to(d) for k, v in obs_bf.items()}, (h.to(d), c.to(d)))
    for k in P.HEADS:
        assert lm[k].shape == lo[k].shape
        torch.testing.assert_close(lm[k], lt[k].transpose(0, 1), rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(lm[k].cpu(), lo[k], rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(vm, vt.transpose(0, 1), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(hm, ht, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(cm, ct, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(vm.cpu(), vo, rtol=1e-4, atol=2e-5)
    assert hm.shape == cm.shape == (2, B, 128)
    torch.testing.assert_close(hm.cpu(), hn, rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(cm.cpu(), cn, rtol=1e-4, atol=2e-5)


# ------------------------------------------------------------------------------------------------ checkpoints
def test_stacked_checkpoint_loads_into_oracle_and_stock_torch(tmp_path):
    """L = 2: upload_model's bytes load strictly into the stacked oracle policy and, rnn.* part, into a stock
    nn.LSTM(num_layers=2)."""
    opt = make_optimizer(128, "lstm", 8, tmp_path, checkpoint=True)
    with open(os.path.join(str(tmp_path), "model_000000001.pt"), "rb") as f:
        body = f.read()
    assert body == opt.mq.latest_model()[0]
    sd = torch.load(io.BytesIO(body), map_location="cpu")
    assert len(sd) == 38 and "rnn.weight_hh_l1" in sd
    StackedRefPolicy(128, "lstm", 2).load_state_dict(sd, strict=True)
    stock = torch.nn.LSTM(input_size=128, hidden_size=128, num_layers=2, batch_first=True)
    stock.load_state_dict({k[4:]: v for k, v in sd.items() if k.startswith("rnn.")}, strict=True)
    for k, v in opt.policy_base.state_dict().items():
        assert torch.equal(v.cpu(), sd[k]), k


def test_stacked_resume_takes_the_same_next_step(tmp_path):
    """L = 2: a checkpoint (model_*.pt + adam_*.state) written after one step and resumed by a new optimizer takes the same
    next step as the optimizer that wrote it."""
    S = 16
    rollouts = [make_rollout(S, 500 + i) for i in range(4)]
    a = make_optimizer(256, "gru", S, tmp_path, checkpoint=True)
    a.use_cuda_graph = False
    batch = a.batch_from_rollouts(copy.deepcopy(rollouts))
    a.train(batch)
    a.upload_model(version=1)
    b = make_optimizer(256, "gru", S, tmp_path, checkpoint=True)
    b.use_cuda_graph = False
    assert b.iteration_start == 2
    assert torch.equal(a.flat.param, b.flat.param) and torch.equal(a.exp_avg, b.exp_avg)
    assert torch.equal(a.exp_avg_sq, b.exp_avg_sq) and torch.equal(a.adam_steps, b.adam_steps)
    batch2 = a.batch_from_rollouts(copy.deepcopy(rollouts))
    la, _, ga = a.train(batch2)
    lb, _, gb = b.train(batch2)
    for k in la:
        np.testing.assert_allclose(float(la[k]), float(lb[k]), rtol=1e-6, atol=1e-9, err_msg=k)
    np.testing.assert_allclose(float(ga["unclipped"]), float(gb["unclipped"]), rtol=1e-6)
    torch.testing.assert_close(a.flat.param, b.flat.param, rtol=1e-6, atol=1e-9)
    torch.testing.assert_close(a.exp_avg, b.exp_avg, rtol=1e-5, atol=1e-12)
    assert torch.equal(a.adam_steps, b.adam_steps) and int(b.adam_steps.max()) == 2


def test_single_layer_checkpoint_into_two_layer_optimizer(tmp_path):
    """pretrained_model keeps the reference's strict=False: a 1-layer checkpoint sets layer 0 (and every other tensor it
    has) of a 2-layer optimizer and leaves layer 1 at its seeded initial values."""
    S = 8
    one_dir, two_dir = tmp_path / "one", tmp_path / "two"
    one = make_optimizer(128, "lstm", S, one_dir, num_layers=1, checkpoint=True)
    one.train(one.batch_from_rollouts([make_rollout(S, 900 + i) for i in range(3)]))
    one.upload_model(version=1)
    path = os.path.join(str(one_dir), "model_000000001.pt")
    ckpt = torch.load(path, map_location="cpu")
    fresh = make_optimizer(128, "lstm", S, two_dir).policy_base.state_dict()
    loaded = make_optimizer(128, "lstm", S, two_dir, pretrained_model=path).policy_base.state_dict()
    assert set(ckpt) < set(loaded) and len(loaded) == len(ckpt) + 4
    for k, v in loaded.items():
        if k in ckpt:
            assert torch.equal(v.cpu(), ckpt[k]), k
        else:
            assert k.endswith("_l1") and torch.equal(v, fresh[k]), k
    assert not torch.equal(ckpt["rnn.weight_hh_l0"], fresh["rnn.weight_hh_l0"].cpu())    # layer 0 was changed


def test_single_layer_checkpoint_with_adam_state_into_checkpointing_two_layer_optimizer(tmp_path, caplog):
    """The entry point's setting (checkpoint=True, as main() passes on rank 0): the 1-layer run's adam_*.state lies next to
    its model_*.pt but is keyed by the 34-tensor layout, so the 2-layer optimizer loads the weights, logs that it does not
    restore the moments, starts them from zero and trains."""
    S = 8
    one_dir, two_dir = tmp_path / "one", tmp_path / "two"
    one = make_optimizer(128, "lstm", S, one_dir, num_layers=1, checkpoint=True)
    rollouts = [make_rollout(S, 900 + i) for i in range(3)]
    one.train(one.batch_from_rollouts(copy.deepcopy(rollouts)))
    one.upload_model(version=1)
    path = os.path.join(str(one_dir), "model_000000001.pt")
    assert os.path.isfile(os.path.join(str(one_dir), "adam_000000001.state"))
    ckpt = torch.load(path, map_location="cpu")
    with caplog.at_level("WARNING"):
        two = make_optimizer(128, "lstm", S, two_dir, checkpoint=True, pretrained_model=path)
    assert any("Not restoring Adam state" in r.getMessage() for r in caplog.records)
    assert two.iteration_start == 2
    assert not two.exp_avg.any() and not two.exp_avg_sq.any() and not two.adam_steps.any()
    sd = two.policy_base.state_dict()
    for k, v in ckpt.items():
        assert torch.equal(sd[k].cpu(), v), k
    losses, _, norms = two.train(two.batch_from_rollouts(copy.deepcopy(rollouts)))
    assert np.isfinite(float(losses["loss"])) and np.isfinite(float(norms["unclipped"]))
    assert int(two.adam_steps.max()) == 1
