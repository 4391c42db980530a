"""GPU tests of the schedulable PPO settings and the in-kernel PPO diagnostics: the statistics and the clipped value loss
against the CPU oracle (``ppo_controls_oracle.py``), the device-block entry points against the scalar ones (bitwise),
hyper-parameter schedules under CUDA-graph replay, non-default GAE settings, and value clipping through run_iteration."""
import copy
import math
import os
import pickle
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ppo_controls_oracle as PC  # noqa: E402
import test_gpu_parity as P  # noqa: E402
from oracle import ref_optimizer as RO  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS, SIZES = P.HEADS, P.SIZES


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=16, num_layers=1, epochs=1, min_seq=1, vf_coef=0.5, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="ppo", rmq_port=uuid.uuid4().int % 100000, epochs=epochs, min_seq_per_epoch=min_seq,
                         seq_len=seq_len, learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                         log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=vf_coef, run_local=True, hidden_size=hidden_size,
                         cell=cell, num_layers=num_layers, **kw)


def _stats_dict(t):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer._ppo_stats_dict(t.cpu().tolist())


def _check_stats(got, want):
    assert set(got) == set(want)
    for k in want:
        np.testing.assert_allclose(got[k], want[k], rtol=1e-4, atol=1e-6, err_msg=k)


# ------------------------------------------------------------------------------------------------ kernel vs oracle
@pytest.mark.parametrize("n_tokens,drop,pad", [(300, None, None), (1000, None, 900), (129, "ability", 100), (5, "x", None),
                                               (640, "target_unit", 517), (131072, None, None)])
@pytest.mark.parametrize("value_clip", [None, 0.05])
def test_stats_and_clipped_value_loss_vs_oracle(n_tokens, drop, pad, value_clip):
    """Several 128-token CTAs, a head without action rows, padding rows: losses, entropies, the diagnostics, dlogits and
    dvalue of dc_ppo_loss_fwd_bwd_dev against the oracle's autograd (clipped value loss when value_clip is set).
    131072 tokens are C2's batch: 1024 CTAs meet in the last-CTA ticket and the float64 atomics."""
    from dotaclient_b200 import ops
    e_clip, entropy_coef, vf_coef = 0.2, 5e-4, 0.5
    logits, masks, actions, old, values, adv, ret = P._random_loss_inputs(n_tokens, 11 + n_tokens, drop, pad)
    g = torch.Generator().manual_seed(n_tokens)
    old_values = values + 0.1 * torch.randn(n_tokens, generator=g)
    lg = {k: v.clone().unsqueeze(0).requires_grad_(True) for k, v in logits.items()}
    vg = values.clone().view(1, -1, 1).requires_grad_(True)
    loss, p_loss, e_loss, v_loss, ents = PC.ppo_loss(
        lg, vg, {k: v.unsqueeze(0) for k, v in actions.items()}, {k: v.unsqueeze(0) for k, v in masks.items()}, old,
        adv.view(1, -1), ret.view(1, -1), entropy_coef, vf_coef, e_clip, old_values=old_values.view(1, -1),
        value_clip=value_clip)
    loss.backward()
    want = PC.ppo_stats(logits, masks, actions, old, values, ret, e_clip)
    d = P.dev()
    dense_old = torch.zeros(n_tokens, 5)
    for h, k in enumerate(HEADS):
        dense_old[actions[k].any(dim=1), h] = old[k]
    hp = ops.hparam_block(d, lr=1e-3, e_clip=e_clip, entropy_coef=entropy_coef, vf_coef=vf_coef, max_grad_norm=0.5,
                          value_clip=value_clip)
    out, n_act, dlogits, dvalue, stats = ops.ppo_loss_fwd_bwd(
        [logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS], [actions[k].to(d) for k in HEADS],
        dense_old.to(d), adv.to(d), ret.to(d), values.to(d), None, None, None, hparams=hp, old_value=old_values.to(d))
    out = out.cpu().numpy()
    assert n_act.cpu().tolist() == [int(actions[k].any(dim=1).sum()) for k in HEADS]
    for i, ref in enumerate((loss, p_loss, e_loss, v_loss)):
        np.testing.assert_allclose(out[i], float(ref), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out[4:9], [float(ents[k]) for k in HEADS], rtol=1e-4, atol=1e-6)
    _check_stats(_stats_dict(stats), want)
    if drop is not None:
        assert _stats_dict(stats)["approx_kl/" + drop] == 0.0
    for h, k in enumerate(HEADS):
        g_ref = lg[k].grad[0] if lg[k].grad is not None else torch.zeros_like(logits[k])
        torch.testing.assert_close(dlogits[h].cpu(), g_ref, rtol=2e-4, atol=1e-8)
    gv = vg.grad.view(-1)
    torch.testing.assert_close(dvalue.cpu(), gv, rtol=1e-4, atol=1e-9)
    assert float(torch.nn.functional.cosine_similarity(dvalue.cpu(), gv, dim=0)) >= 0.9999
    if value_clip:                                   # the clipped branch really won somewhere, with a zero gradient
        vc = old_values + torch.clamp(values - old_values, -value_clip, value_clip)
        won = ((vc - ret).pow(2) > (values - ret).pow(2)) & ((values - old_values).abs() > value_clip)
        assert bool(won.any()) and bool((dvalue.cpu()[won] == 0).all())


# ------------------------------------------------------------------------------------------------ bitwise: device block
def test_dev_entry_points_are_bitwise_equal_to_the_scalar_ones():
    """At the same values the device-block forms (loss contiguous and packed, gradient finish) give bit-identical results:
    every value is rounded to the type the scalar argument has."""
    from dotaclient_b200 import ops
    d = P.dev()
    n = 1000
    logits, masks, actions, old, values, adv, ret = P._random_loss_inputs(n, 5, None, 900)
    dense_old = torch.zeros(n, 5)
    for h, k in enumerate(HEADS):
        dense_old[actions[k].any(dim=1), h] = old[k]
    L, M, A = [logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS], [actions[k].to(d) for k in HEADS]
    e_clip, ent, vf = 0.13, 3e-3, 0.7                   # none of them is exact in float
    hp = ops.hparam_block(d, lr=3e-4, e_clip=e_clip, entropy_coef=ent, vf_coef=vf, max_grad_norm=0.3)
    a = ops.ppo_loss_fwd_bwd(L, M, A, dense_old.to(d), adv.to(d), ret.to(d), values.to(d), e_clip, ent, vf)
    b = ops.ppo_loss_fwd_bwd(L, M, A, dense_old.to(d), adv.to(d), ret.to(d), values.to(d), None, None, None, hparams=hp,
                             old_value=values.to(d) + 1.0)     # old values are ignored while the value clip is 0
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[3], b[3])
    assert all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    # packed form (what DotaOptimizer runs): small heads + value as columns of one [N,128] tensor
    g = torch.Generator().manual_seed(9)
    packed = torch.randn(n, ops.PACK_WIDTH, generator=g).to(d)
    tu = logits["target_unit"].to(d)
    args = (packed, tu, M, A, dense_old.to(d), adv.to(d), ret.to(d))
    a = ops.ppo_loss_packed(*args, e_clip, ent, vf)
    b = ops.ppo_loss_packed(*args, None, None, None, hparams=hp)
    for x, y in zip(a, b[:4]):
        assert torch.equal(x, y)
    # gradient finish: 3 tensors, gradients large enough that the norm clip is active
    total, segs = 3000, [(0, 1000), (1024, 2000), (2048, 3000)]
    seg_lo = torch.tensor([s[0] for s in segs], dtype=torch.int64, device=d)
    seg_hi = torch.tensor([s[1] for s in segs], dtype=torch.int64, device=d)
    seg_head = torch.full((3,), -1, dtype=torch.int32, device=d)
    param = torch.randn(total, generator=g).to(d)
    grad = torch.cat([torch.randn(total, generator=g), torch.ones(3)]).to(d)
    m, v = (0.01 * torch.randn(total, generator=g)).to(d), (0.01 * torch.rand(total, generator=g)).to(d)
    steps = torch.tensor([0, 3, 7], dtype=torch.int32, device=d)
    loss_out = torch.zeros(16, device=d)
    res = []
    for use_dev in (False, True):
        bufs = [param.clone(), grad.clone(), m.clone(), v.clone(), steps.clone()]
        metrics = torch.zeros(4, device=d)
        ws = torch.zeros(1024, dtype=torch.uint8, device=d)
        ops.grad_finish(*bufs, seg_lo, seg_hi, seg_head, total, 3e-4 if not use_dev else None, (0.9, 0.999), 1e-8,
                        0.3 if not use_dev else None, loss_out, metrics, ws, hparams=hp if use_dev else None)
        res.append(bufs + [metrics])
    assert float(res[0][5][0]) > float(res[0][5][1]) > 0          # clipped
    for x, y in zip(*res):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ schedules
def _snapshot(opt):
    return [opt.flat.param.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.adam_steps.clone()]


def test_schedules_under_graph_replay_equal_launch_by_launch(tmp_path):
    """lr, e_clip, entropy_coef and MAX_GRAD_NORM change before every step; the optimizer that replays its captured graph
    and the one that launches kernel by kernel stay bitwise equal (parameters, Adam moments, losses, statistics), and
    every change shows in the result."""
    S, B = 16, 6
    a = make_optimizer(tmp_path)
    b = make_optimizer(tmp_path)
    b.use_cuda_graph = False
    rollouts = [make_rollout(S, 40 + i) for i in range(B)]
    batch_a = a.batch_from_rollouts(copy.deepcopy(rollouts))
    batch_b = b.batch_from_rollouts(copy.deepcopy(rollouts))
    schedule = [dict(),                                                    # eager on both ("seen")
                dict(learning_rate=1e-3, e_clip=1e-5),                     # a: captured, then replayed
                dict(lr_group=0.0, entropy_coef=0.05),                     # replay; lr 0 leaves the weights unchanged
                dict(learning_rate=2e-4, MAX_GRAD_NORM=1e-4, e_clip=10.0),
                dict(MAX_GRAD_NORM=1e6, entropy_coef=0.0, e_clip=1e-5)]
    results = {}
    for step, change in enumerate(schedule):
        for name, opt, batch in (("a", a, batch_a), ("b", b, batch_b)):
            for k, val in change.items():
                if k == "lr_group":
                    opt.optimizer.param_groups[0]["lr"] = val
                else:
                    setattr(opt, k, val)
            before = _snapshot(opt)
            losses, ents, norms = opt.train(batch)
            results[name, step] = (before, _snapshot(opt), losses, ents, norms, dict(opt.last_ppo_stats))
        ra, rb = results["a", step], results["b", step]
        for x, y in zip(ra[1], rb[1]):
            assert torch.equal(x, y), step
        for k in ra[2]:
            assert torch.equal(ra[2][k], rb[2][k]), (k, step)
        for k in ra[4]:
            assert torch.equal(ra[4][k], rb[4][k]), (k, step)
        assert ra[5] == rb[5], step
    assert isinstance(a._graphs.get((S, B, True)), tuple), "the step was never captured"
    assert not any(isinstance(v, tuple) for v in b._graphs.values())
    for name in ("a", "b"):
        before, after, losses, ents, norms, st = results[name, 2]
        assert torch.equal(before[0], after[0]) and not torch.equal(before[1], after[1])     # lr = 0: only the moments
        np.testing.assert_allclose(float(losses["entropy_loss"]), -0.05 * sum(float(v) for v in ents.values()), rtol=1e-5)
        _, _, _, _, norms, st = results[name, 3]
        assert st["clip_fraction"] == 0.0 and float(norms["clipped"]) < 1e-3 * float(norms["unclipped"])
        _, _, losses, _, norms, st = results[name, 4]
        assert st["clip_fraction"] > 0.5 and torch.equal(norms["clipped"], norms["unclipped"])
        assert float(losses["entropy_loss"]) == 0.0
        assert not torch.equal(results[name, 1][0][0], results[name, 1][1][0])             # lr 1e-3 moved the weights
    assert a.optimizer.state_dict()["param_groups"][0]["lr"] == 2e-4


def test_vf_coef_schedule_across_zero_gates_the_value_head(tmp_path):
    """vf_coef switched 0 -> 0.5 -> 0 between steps, replayed from the captured graph and launch by launch: while it is 0 the
    value head has no gradient, so Adam leaves its tensors and step counters alone (the reference's .grad = None); while it
    is > 0 they train.  Both runs stay bitwise equal."""
    S, B = 16, 6
    a = make_optimizer(tmp_path, vf_coef=0.0)
    b = make_optimizer(tmp_path, vf_coef=0.0)
    b.use_cuda_graph = False
    rollouts = [make_rollout(S, 140 + i) for i in range(B)]
    batch_a = a.batch_from_rollouts(copy.deepcopy(rollouts))
    batch_b = b.batch_from_rollouts(copy.deepcopy(rollouts))
    idx = [i for i, n in enumerate(a.flat.names) if n.startswith("affine_value")]
    assert len(idx) == 2

    def value_head(opt):
        return [opt.flat.param[opt.flat.starts[i]:opt.flat.ends[i]].clone() for i in idx], opt.adam_steps[idx].clone()

    for step, vf in enumerate([0.0, 0.0, 0.5, 0.5, 0.0, 0.0]):     # a: eager, captured, then replays
        res = []
        for opt, batch in ((a, batch_a), (b, batch_b)):
            opt.vf_coef = vf
            p0, s0 = value_head(opt)
            losses, _, norms = opt.train(batch)
            p1, s1 = value_head(opt)
            if vf > 0:
                assert all(not torch.equal(x, y) for x, y in zip(p0, p1)) and torch.equal(s1, s0 + 1), step
                assert float(losses["value_loss"]) > 0
            else:
                assert all(torch.equal(x, y) for x, y in zip(p0, p1)) and torch.equal(s1, s0), step
                assert float(losses["value_loss"]) == 0
            res.append((losses, norms))
        for k in res[0][0]:
            assert torch.equal(res[0][0][k], res[1][0][k]), (k, step)
        assert torch.equal(res[0][1]["unclipped"], res[1][1]["unclipped"]), step
        for x, y in zip(_snapshot(a), _snapshot(b)):
            assert torch.equal(x, y), step
    assert isinstance(a._graphs.get((S, B, True)), tuple), "the step was never captured"
    assert a.adam_steps[idx].tolist() == [2, 2] and int(a.adam_steps.max()) == 6


# ------------------------------------------------------------------------------------------------ GAE settings
def test_non_default_gamma_and_lambda_match_the_oracle(tmp_path):
    """gamma / gae_lambda reach the GAE scan of experience prep: per rollout, advantages and returns equal
    oracle.ref_optimizer.advantage_returns at those values (from the same values and rewards), and differ from the
    defaults."""
    S = 16
    opt = make_optimizer(tmp_path, gamma=0.995, gae_lambda=0.9)
    rollouts = P._rollouts(3, S, seed=77)
    groups = opt.experiences_from_rollouts(copy.deepcopy(rollouts))
    for seqs in groups:
        v = np.append(np.concatenate([s.values.reshape(-1).cpu().numpy() for s in seqs]), np.float32(0))
        r = np.append(np.concatenate([np.asarray(s.rewards).sum(axis=1) for s in seqs]), np.float32(0)).astype(np.float32)
        adv, ret = RO.advantage_returns(r, v.astype(np.float32), gamma=0.995, lam=0.9)
        got_adv = np.concatenate([s.advantages.cpu().numpy() for s in seqs])
        got_ret = np.concatenate([s.returns.cpu().numpy() for s in seqs])
        np.testing.assert_allclose(got_adv, adv, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(got_ret, ret, rtol=1e-5, atol=1e-6)
        d_adv, _ = RO.advantage_returns(r, v.astype(np.float32))
        assert np.abs(d_adv - adv).max() > 1e-3
    assert len(groups) == 3 and sum(len(g) for g in groups) > 3


# ------------------------------------------------------------------------------------------------ end to end
def test_step_statistics_match_the_oracle_on_ragged_rollouts(tmp_path):
    """The first train() step on ragged multi-chunk rollouts: explained variance and the (zero) clip fraction against the
    oracle's forward of the same batch; the approximate KL is ~0 (new and old policy are the same weights)."""
    S = 16
    mine = make_optimizer(tmp_path)
    oracle = P.make_oracle(128, "lstm", S)
    rollouts = P._rollouts(3, S, seed=31)
    xs_m = [s for grp in mine.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in grp]
    xs_o = [s for r in rollouts for s in oracle.experiences_from_rollout(copy.deepcopy(r))]
    _, logits, values = oracle.loss_only(xs_o)
    adv, ret, _, actions, masks, _, old = RO.stack_batch(xs_o)
    flat = {k: v.reshape(-1, v.shape[-1]) for k, v in logits.items()}
    want = PC.ppo_stats({k: v.detach() for k, v in flat.items()}, {k: v.reshape(flat[k].shape) for k, v in masks.items()},
                        {k: v.reshape(flat[k].shape) for k, v in actions.items()}, old, values.detach().reshape(-1),
                        ret.reshape(-1), 0.1)
    mine.train(xs_m)
    got = mine.last_ppo_stats
    assert set(got) == set(want)
    np.testing.assert_allclose(got["explained_variance"], want["explained_variance"], rtol=1e-4, atol=1e-5)
    for k in got:
        if k.startswith("approx_kl"):
            assert abs(got[k]) < 1e-6 and abs(want[k]) < 1e-6, k
        elif k.startswith("clip_fraction"):
            assert got[k] == want[k] == 0.0, k


def test_experience_batch_old_values_pin_to_and_value_clip_refusal(tmp_path):
    """batch_from_rollouts carries the prep-time values as old_values; pin_memory / to keep them; a batch without them
    trains as before, and is refused with ValueError when value clipping is on."""
    from dotaclient_b200.optimizer import ExperienceBatch
    S, B = 16, 4
    opt = make_optimizer(tmp_path, value_clip=0.2)
    rollouts = [make_rollout(S, 60 + i) for i in range(B)]
    batch = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    seqs = [s for r in rollouts for s in opt.experiences_from_rollout(copy.deepcopy(r))]
    assert batch.old_values.shape == (S, B)
    torch.testing.assert_close(batch.old_values, torch.stack([s.values.reshape(-1) for s in seqs], dim=1), rtol=1e-6,
                               atol=1e-7)
    host = batch.pin_memory()
    assert host.old_values.is_pinned() and torch.equal(host.old_values, batch.old_values.cpu())
    back = host.to(opt.device)
    torch.cuda.synchronize()
    assert torch.equal(back.old_values, batch.old_values)
    bare = ExperienceBatch(batch.observations, batch.masks, batch.actions, batch.old_logp, batch.advantages,
                           batch.returns, batch.h0, batch.c0)
    assert "old_values" not in [k for _, k, _ in bare.tensors()]
    with pytest.raises(ValueError, match="old_values"):
        opt.train(bare)
    losses, _, _ = opt.train(batch)
    assert math.isfinite(float(losses["value_loss"]))
    opt.value_clip = None
    bare_host = bare.pin_memory()
    assert bare_host.old_values is None and bare_host.to(opt.device).old_values is None
    losses, _, _ = opt.train(bare)
    assert math.isfinite(float(losses["loss"]))


@pytest.mark.parametrize("H,cell,L", [(128, "lstm", 2), (256, "gru", 1)])
def test_value_clip_run_iteration_reports_ppo_metrics(H, cell, L, tmp_path):
    """value_clip through a whole run_iteration (prep, epochs of train(), metrics) at L = 2 layers and at the reference's
    GRU-256: every ppo/* metric is present and finite, and the existing metric keys are unchanged."""
    from dotaclient_b200.optimizer import MessageQueue
    S = 16
    opt = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=L, epochs=3, min_seq=6, value_clip=0.2,
                         gamma=0.99, gae_lambda=0.95, clip_range=0.2, max_grad_norm=1.0)
    actor = MessageQueue(host="ppo", port=opt.rmq_port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for i in range(4):
        actor.publish_experience(pickle.dumps(make_rollout(40 + i, 90 + i, weight_version=1, with_canvas=True)))
    before = opt.flat.param.clone()
    metrics = opt.run_iteration(1)
    keys = ["ppo/approx_kl", "ppo/clip_fraction", "ppo/explained_variance"] + \
        ["ppo/%s/%s" % (s, k) for s in ("approx_kl", "clip_fraction") for k in HEADS]
    for k in keys:
        assert k in metrics and math.isfinite(metrics[k]), k
    assert 0.0 <= metrics["ppo/clip_fraction"] <= 1.0 and metrics["ppo/approx_kl"] >= -1e-6
    for k in ("loss/sum", "loss/policy", "loss/entropy", "loss/value", "entropy", "grad_norm/unclipped"):
        assert math.isfinite(float(metrics[k])), k
    assert not torch.equal(before, opt.flat.param)
