"""GPU tests of ``policy_ratio='joint'``: ``dc_ppo_loss_fwd_bwd_joint`` against the float64 CPU oracle
(``joint_ratio_oracle.py``) and against the per-head kernel, a joint train() step against the oracle's step, packed against
unpacked, graph replay with an ``e_clip`` schedule, and the metrics of run_iteration."""
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
import joint_ratio_oracle as JO  # noqa: E402
import padding_oracle as PO  # noqa: E402
import test_gpu_packing as PK  # noqa: E402
import test_gpu_parity as P  # noqa: E402
from oracle import ref_optimizer as RO  # noqa: E402
from stacked_oracle import StackedRefPolicy  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS = P.HEADS
E_CLIP = 0.1


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", num_layers=1, seq_len=16, epochs=1, min_seq=1, port=None,
                   **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="joint", rmq_port=port if port is not None else uuid.uuid4().int % 100000,
                         epochs=epochs, min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=5e-5, checkpoint=False,
                         pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4,
                         vf_coef=0.5, run_local=True, hidden_size=hidden_size, cell=cell, num_layers=num_layers, **kw)


# ------------------------------------------------------------------------------------------------ kernel inputs
def _inputs(n, seed, drop=None, pad=None, with_valid=False):
    """Random loss inputs whose joint ratios lie on both sides of 1 +- E_CLIP and, on every third token, at exactly 1:
    the old log-probs are the kernel's own selected log-probs (dc_selected_logp) plus per-head offsets, zero on those
    tokens.  Heads without an action row get an old log-prob of 99 (it must be ignored).  Tokens whose float64 ratio lies
    within 1e-4 of a clip bound are moved off it, so that the fp32 kernel and the oracle clip the same tokens."""
    from dotaclient_b200 import ops
    logits, masks, actions, _, values, adv, ret = P._random_loss_inputs(n, seed, drop, pad)
    d = P.dev()
    g = torch.Generator().manual_seed(seed + 1)
    lp = ops.selected_logp([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                           [actions[k].to(d) for k in HEADS]).cpu()
    acted = torch.stack([actions[k].any(dim=1) for k in HEADS], dim=1)
    offs = 0.3 * torch.rand(n, 5, generator=g) - 0.15
    offs[::3] = 0.0
    old = torch.where(acted, lp + offs, torch.full_like(lp, 99.0))
    valid = None
    if with_valid:
        valid = torch.rand(n, generator=g) < 0.8
        valid[: min(n, 3)] = True
    log_r, has, _ = JO.joint_log_ratio({k: v.double() for k, v in logits.items()}, actions, masks, old.double(), valid)
    r = torch.exp(log_r)
    near = has & (((r - (1 + E_CLIP)).abs() < 1e-4) | ((r - (1 - E_CLIP)).abs() < 1e-4))
    for t in torch.nonzero(near).flatten().tolist():
        h = int(torch.nonzero(acted[t])[0])
        old[t, h] -= 1e-3
    ov = values + 0.1 * torch.randn(n, generator=g)
    return logits, masks, actions, old, values, adv, ret, ov, valid


def _run(inputs, joint=True, value_clip=None, entropy_coef=5e-4, vf_coef=0.5):
    from dotaclient_b200 import ops
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    d = P.dev()
    hp = ops.hparam_block(d, e_clip=E_CLIP, entropy_coef=entropy_coef, vf_coef=vf_coef, value_clip=value_clip)
    return ops.ppo_loss_fwd_bwd([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                                [actions[k].to(d) for k in HEADS], old.to(d), adv.to(d), ret.to(d), values.to(d),
                                None, None, None, hparams=hp, old_value=ov.to(d),
                                valid=None if valid is None else valid.to(d), joint=joint)


def _stats(t, joint=True):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer._ppo_stats_dict(t.cpu().tolist(), joint=joint)


# ------------------------------------------------------------------------------------------------ kernel vs oracle
@pytest.mark.parametrize("n,drop,pad", [(300, None, None), (129, "ability", 100), (1000, "target_unit", 900),
                                        (131072, None, None)])
@pytest.mark.parametrize("with_valid", [False, True])
@pytest.mark.parametrize("value_clip", [None, 0.05])
def test_joint_kernel_vs_oracle(n, drop, pad, with_valid, value_clip):
    """Losses, entropies, per-head policy slots (0), n_actions, per-head and joint diagnostics, dlogits and dvalue of
    dc_ppo_loss_fwd_bwd_joint against the float64 oracle's autograd; a repeated call is bitwise equal.  Cases: a head
    without action rows, empty-mask rows (the padded tail), invalid tokens, and C2's 131072 tokens."""
    inputs = _inputs(n, 5 + n, drop, pad, with_valid)
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    lg = {k: v.double().requires_grad_(True) for k, v in logits.items()}
    vg = values.double().requires_grad_(True)
    loss, p_loss, e_loss, v_loss, ents = JO.joint_ppo_loss(lg, vg, actions, masks, old.double(), adv.double(),
                                                           ret.double(), 5e-4, 0.5, E_CLIP, valid=valid,
                                                           old_values=ov.double(), value_clip=value_clip)
    loss.backward()
    log_r, has, _ = JO.joint_log_ratio({k: v.double() for k, v in logits.items()}, actions, masks, old.double(), valid)
    r = torch.exp(log_r[has])
    assert bool((r > 1 + E_CLIP).any()) and bool((r < 1 - E_CLIP).any()) and bool(((r - 1).abs() < E_CLIP).any())
    res = _run(inputs, value_clip=value_clip)
    out, n_act, dlogits, dvalue, stats = res
    out = out.cpu().numpy()
    use = torch.ones(n, dtype=torch.bool) if valid is None else valid
    assert n_act.cpu().tolist() == [int((actions[k].any(dim=1) & use).sum()) for k in HEADS]
    for i, want in enumerate((loss, p_loss, e_loss, v_loss)):
        np.testing.assert_allclose(out[i], float(want.detach()), rtol=1e-4, atol=1e-6, err_msg=str(i))
    np.testing.assert_allclose(out[4:9], [float(ents[k].detach()) for k in HEADS], rtol=1e-4, atol=1e-6)
    assert (out[9:14] == 0).all()
    want_st = PO.masked_stats(logits, actions, masks, old, values, ret, use, E_CLIP)
    want_st.update(JO.joint_stats(logits, actions, masks, old, E_CLIP, valid))
    got_st = _stats(stats)
    assert set(got_st) == set(want_st)
    for k, w in want_st.items():
        np.testing.assert_allclose(got_st[k], w, rtol=1e-4, atol=1e-6, err_msg=k)
    assert float(stats[15]) == 0.0
    for h, k in enumerate(HEADS):
        g_ref = lg[k].grad.float() if lg[k].grad is not None else torch.zeros_like(logits[k])
        torch.testing.assert_close(dlogits[h].cpu(), g_ref, rtol=2e-4, atol=1e-8)
        if valid is not None:
            assert bool((dlogits[h].cpu()[~valid] == 0).all()), k
    if drop is not None:
        assert bool((dlogits[HEADS.index(drop)] == 0).all()) and got_st["approx_kl/" + drop] == 0.0
    if pad is not None:
        assert all(bool((dlogits[h][pad:] == 0).all()) for h in range(5))
    torch.testing.assert_close(dvalue.cpu(), vg.grad.float(), rtol=1e-4, atol=1e-9)
    again = _run(inputs, value_clip=value_clip)
    for a, b in zip(res, again):
        if isinstance(a, list):
            assert all(torch.equal(x, y) for x, y in zip(a, b))
        else:
            assert torch.equal(a, b)


def test_joint_kernel_without_action_rows():
    """T_a = 0: no action row anywhere, and action rows on invalid tokens only.  The policy loss, its gradient, the joint
    statistics and n_actions are 0; the value loss is unchanged."""
    inputs = list(_inputs(300, 41))
    logits, masks, actions = inputs[:3]
    no_act = {k: torch.zeros_like(a) for k, a in actions.items()}
    late = {k: a.clone() for k, a in actions.items()}           # actions on the invalid tokens 100.. only
    for a in late.values():
        a[:100] = False
    assert any(bool(a.any()) for a in late.values())
    for acts, valid in ((no_act, None), (late, torch.arange(300) < 100)):
        case = list(inputs)
        case[2], case[8] = acts, valid
        out, n_act, dlogits, dvalue, stats = _run(tuple(case), entropy_coef=0.0)
        assert float(out[1]) == 0.0 and n_act.cpu().tolist() == [0] * 5
        assert all(bool((g == 0).all()) for g in dlogits)
        st = _stats(stats)
        assert st["approx_kl/joint"] == 0.0 and st["clip_fraction/joint"] == 0.0 and st["approx_kl"] == 0.0
        v_loss = JO.joint_ppo_loss({k: v.double() for k, v in logits.items()}, case[4], acts, masks, case[3].double(),
                                   case[5], case[6], 0.0, 0.5, E_CLIP, valid=valid)[3]
        np.testing.assert_allclose(float(out[3]), float(v_loss), rtol=1e-5)
        assert float(out[0]) == float(out[3])


# ------------------------------------------------------------------------------------------------ per-head vs joint
@pytest.mark.parametrize("with_valid", [False, True])
def test_only_enum_sampled_joint_is_five_times_per_head(with_valid):
    """With only enum sampled and no entropy term, S_t = {enum}: the joint dlogits are 5x the per-head kernel's (rtol 1e-6:
    1/5 * 1/n and 1/T_a round differently; the taken entry g (1 - p) cancels when p is near 1, so its error is bounded
    relative to the largest gradient), and so is the policy loss; entropies, value loss, dvalue, n_actions and the
    per-head diagnostics are the same."""
    inputs = list(_inputs(4000, 9, with_valid=with_valid))
    inputs[2] = {k: (a if k == "enum" else torch.zeros_like(a)) for k, a in inputs[2].items()}
    inputs = tuple(inputs)
    j = _run(inputs, joint=True, entropy_coef=0.0)
    h = _run(inputs, joint=False, entropy_coef=0.0)
    assert float(h[0][1]) != 0.0
    np.testing.assert_allclose(float(j[0][1]), 5 * float(h[0][1]), rtol=1e-6)
    for a, b in zip(j[2], h[2]):
        torch.testing.assert_close(a, 5 * b, rtol=1e-6, atol=1e-6 * float((5 * b).abs().max()))
    assert float(j[2][0].abs().max()) > 0
    assert torch.equal(j[0][2:9], h[0][2:9]) and torch.equal(j[1], h[1]) and torch.equal(j[3], h[3])
    torch.testing.assert_close(j[4][:13], h[4][:13], rtol=1e-6, atol=0.0)


def test_per_head_diagnostics_keep_their_meaning():
    """Every head sampled: stats 0..12, entropies, value loss and dvalue of the joint kernel equal the per-head kernel's."""
    inputs = _inputs(3000, 13, with_valid=True)
    j, h = _run(inputs, joint=True), _run(inputs, joint=False)
    torch.testing.assert_close(j[4][:13], h[4][:13], rtol=1e-6, atol=1e-9)
    assert torch.equal(j[0][2:9], h[0][2:9]) and torch.equal(j[3], h[3]) and torch.equal(j[1], h[1])
    assert float(j[4][13]) > 0 and float(h[4][13]) == 0.0


# ------------------------------------------------------------------------------------------------ train step vs oracle
def _cpu_sequences(seqs):
    out = []
    for s in seqs:
        hid = tuple(x.cpu() for x in s.hidden) if isinstance(s.hidden, tuple) else s.hidden.cpu()
        out.append(RO.RefSequence(observations={k: torch.as_tensor(v).cpu() for k, v in s.observations.items()},
                                  actions={k: torch.as_tensor(v).cpu() for k, v in s.actions.items()},
                                  masks={k: torch.as_tensor(v).cpu() for k, v in s.masks.items()}, hidden=hid,
                                  log_probs_sel={k: v.cpu() for k, v in s.log_probs_sel.items()},
                                  advantages=s.advantages.cpu(), returns=s.returns.cpu(),
                                  valid=None if s.valid is None else s.valid.cpu()))
    return out


@pytest.mark.parametrize("H,cell", [(128, "lstm"), (256, "gru")])
@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
def test_joint_step_vs_oracle(H, cell, estimator, tmp_path):
    """Masked prep, then two joint train() steps against the oracle's joint step on the same sequences (the prep's
    advantages, returns, old log-probs, states and valid masks), at the parity suite's tolerances: losses, entropies,
    grad norms, per-tensor gradients, Adam moments."""
    torch.set_num_threads(8)
    S = 16
    mine = make_optimizer(tmp_path, hidden_size=H, cell=cell, mask_padding=True, advantage_estimator=estimator,
                          policy_ratio="joint")
    torch.manual_seed(7)
    oracle = JO.JointRefOptimizer(StackedRefPolicy(H, cell, 1), seq_len=S)
    rollouts = PK.ragged_rollouts(mine.policy_base, 6, estimator == "vtrace", False)
    xs_m = [s for grp in mine.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in grp]
    xs_o = _cpu_sequences(xs_m)
    assert any(not bool(s.valid.all()) for s in xs_o)
    for ep in range(2):
        lm, em, gm = mine.train(xs_m)
        lo, eo, go = oracle.train(xs_o)
        for k in lo:
            np.testing.assert_allclose(float(lm[k]), float(lo[k].detach()), rtol=2e-4, atol=2e-6, err_msg="%s %d" % (k, ep))
        for k in eo:
            np.testing.assert_allclose(float(em[k]), float(eo[k].detach()), rtol=2e-4, atol=1e-6, err_msg="entropy " + k)
        np.testing.assert_allclose(float(gm["unclipped"]), float(go["unclipped"]), rtol=2e-3)
        np.testing.assert_allclose(float(gm["clipped"]), float(go["clipped"]), rtol=2e-3)
        if ep == 0:
            for name, p in oracle.policy_base.named_parameters():
                g = mine.flat.grad_of(name).cpu()
                cos = torch.nn.functional.cosine_similarity(g.flatten(), p.grad.flatten(), dim=0)
                assert cos > 0.9999, (name, float(cos))
                np.testing.assert_allclose(float(g.norm()), float(p.grad.norm()), rtol=2e-3, err_msg=name)
    assert "approx_kl/joint" in mine.last_ppo_stats and mine.last_ppo_stats["approx_kl/joint"] >= 0
    sd = mine.optimizer.state_dict()["state"]
    want = P._adam_state_by_name(oracle)
    names = [n for n, _ in oracle.policy_base.named_parameters()]
    assert sorted(names[i] for i in sd) == sorted(want)
    for i, st in sd.items():
        w = want[names[i]]
        assert float(st["step"]) == float(w["step"]) == 2.0
        m_scale = float(w["exp_avg"].abs().max())
        v_scale = float(w["exp_avg_sq"].abs().max())
        torch.testing.assert_close(st["exp_avg"], w["exp_avg"], rtol=2e-3, atol=2e-3 * m_scale + 1e-12)
        torch.testing.assert_close(st["exp_avg_sq"], w["exp_avg_sq"], rtol=4e-3, atol=4e-3 * v_scale + 1e-20)


@pytest.mark.parametrize("H,cell", [(128, "lstm"), (256, "gru")])
@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
def test_packed_joint_step_equals_unpacked(H, cell, estimator, tmp_path):
    """The packed batch holds the unpacked masked batch's valid tokens: two joint steps on each agree to the packing
    suite's tolerances (losses, entropies, grad norms, statistics including the joint ones, gradients, weights)."""
    kw = dict(hidden_size=H, cell=cell, advantage_estimator=estimator, mask_padding=True, policy_ratio="joint",
              value_clip=0.2)
    unpacked = make_optimizer(tmp_path, **kw)
    packed = make_optimizer(tmp_path, pack_sequences=True, **kw)
    rollouts = PK.ragged_rollouts(unpacked.policy_base, 3, estimator == "vtrace", True)
    bu = unpacked.batch_from_rollouts(copy.deepcopy(rollouts))
    bp = packed.batch_from_rollouts(copy.deepcopy(rollouts))
    assert bp.batch_size < bu.batch_size
    for step in range(2):
        lu, eu, gu = unpacked.train(bu)
        lp, ep, gp = packed.train(bp)
        for k in lu:
            assert PK._close(lp[k], lu[k], 2e-4, 2e-6), (step, k, float(lp[k]), float(lu[k]))
        for k in eu:
            assert PK._close(ep[k], eu[k], 2e-4, 2e-6), (step, k)
        for k in gu:
            assert PK._close(gp[k], gu[k], 2e-3), (step, k)
        assert {"approx_kl/joint", "clip_fraction/joint"} <= set(unpacked.last_ppo_stats)
        for k, v in unpacked.last_ppo_stats.items():
            assert abs(packed.last_ppo_stats[k] - v) <= 2e-4 * abs(v) + 2e-5, (step, k, packed.last_ppo_stats[k], v)
        fu, fp = unpacked.flat, packed.flat
        for name, lo, hi in zip(fu.names, fu.starts, fu.ends):
            assert PK._close(fp.grad[lo:hi], fu.grad[lo:hi], 2e-3, 1e-9), (step, "grad", name)
        assert PK._close(fp.param, fu.param, 0.0, 1e-6), (step, "weights")


# ------------------------------------------------------------------------------------------------ graph replay
def test_graph_replayed_joint_step_equals_eager_and_follows_e_clip(tmp_path):
    """The joint step replayed from its captured graph is bit-identical to the launch-by-launch one, through an e_clip
    schedule that reaches the replays: a huge clip range clips no joint ratio, a tiny one nearly all."""
    a = make_optimizer(tmp_path, mask_padding=True, policy_ratio="joint", num_layers=2)
    b = make_optimizer(tmp_path, mask_padding=True, policy_ratio="joint", num_layers=2)
    b.use_cuda_graph = False
    rollouts = PK.ragged_rollouts(a.policy_base, 8, False, False)
    batch_a, batch_b = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    schedule = [dict(), dict(learning_rate=1e-3), dict(e_clip=10.0), dict(e_clip=1e-6), dict(e_clip=0.2)]
    stats = []
    for step, change in enumerate(schedule):
        rec = []
        for opt, batch in ((a, batch_a), (b, batch_b)):
            for k, v in change.items():
                setattr(opt, k, v)
            losses, ents, norms = opt.train(batch)
            rec.append(([float(v) for v in losses.values()], [float(v) for v in ents.values()],
                        [float(v) for v in norms.values()], dict(opt.last_ppo_stats)))
        assert rec[0] == rec[1], step
        assert torch.equal(a.flat.param, b.flat.param) and torch.equal(a.exp_avg_sq, b.exp_avg_sq), step
        stats.append(rec[0][3])
    assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"
    assert not any(isinstance(v, tuple) for v in b._graphs.values())
    assert stats[2]["clip_fraction/joint"] == 0.0 and stats[3]["clip_fraction/joint"] > 0.5
    assert 0.0 <= stats[4]["clip_fraction/joint"] < stats[3]["clip_fraction/joint"]


# ------------------------------------------------------------------------------------------------ run_iteration
def test_run_iteration_reports_the_joint_metrics(tmp_path):
    from dotaclient_b200.optimizer import MessageQueue
    rollouts = [make_rollout(L, 950 + i, game_id=i, weight_version=1, with_canvas=True) for i, L in enumerate((40, 23, 57))]
    base = uuid.uuid4().int % 100000
    metrics = {}
    for port, mode in ((base, "joint"), (base + 1, "per_head")):
        opt = make_optimizer(tmp_path, min_seq=6, port=port, epochs=2, mask_padding=True, policy_ratio=mode)
        actor = MessageQueue(host="joint", port=port, prefetch_count=1, use_model_exchange=False)
        actor.connect()
        for r in rollouts:
            actor.publish_experience(pickle.dumps(r))
        before = opt.flat.param.clone()
        metrics[mode] = opt.run_iteration(1)
        assert not torch.equal(before, opt.flat.param)
    assert set(metrics["joint"]) - set(metrics["per_head"]) == {"ppo/approx_kl/joint", "ppo/clip_fraction/joint"}
    assert set(metrics["per_head"]) <= set(metrics["joint"])
    for k in ("ppo/approx_kl/joint", "ppo/clip_fraction/joint", "loss/policy"):
        assert math.isfinite(float(metrics["joint"][k])), k
    assert 0.0 <= metrics["joint"]["ppo/clip_fraction/joint"] <= 1.0 and metrics["joint"]["ppo/approx_kl/joint"] >= -1e-7
