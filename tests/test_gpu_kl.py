"""GPU tests of KL control: ``dc_ppo_loss_fwd_bwd_kl`` against the float64 oracle (``kl_oracle.py``) in both ratio
modes, beta = 0 against the existing entry points bit for bit, the rows prep stores, the early stop of the gradient finish
(eager, replayed, and through ``train_epochs``), the adaptive coefficient over two iterations, and the metrics.

Tolerances are the suite's for the fused loss (``test_gpu_joint_ratio``): fp32 against float64, rtol 1e-4 on the losses and
statistics and 2e-4 on dlogits.  The KL gradient (beta / T_a)(p - p_old) is a difference of two fp32 probabilities that
carry about 1e-6 relative error each, so it adds at most ~1e-6 beta / T_a absolute to a dlogits entry: far under atol."""
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
import kl_oracle as KO  # noqa: E402
import test_gpu_joint_ratio as JR  # noqa: E402
import test_gpu_packing as PK  # noqa: E402
import test_gpu_parity as P  # noqa: E402
from stacked_oracle import StackedRefPolicy  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS = P.HEADS
E_CLIP = JR.E_CLIP
BETA = 0.7


def _old_rows(logits, masks, seed):
    """Prep-time rows of a policy near the current one: the masked log-softmax of perturbed logits, in fp32."""
    g = torch.Generator().manual_seed(seed)
    moved = {k: v.double() + 0.25 * torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in logits.items()}
    return KO.masked_log_rows(moved, masks).float()


def _run(inputs, rows, joint, beta, value_clip=None, value_norm=None, kl=True):
    from dotaclient_b200 import ops
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    d = P.dev()
    hp = ops.hparam_block(d, e_clip=E_CLIP, entropy_coef=5e-4, vf_coef=0.5, value_clip=value_clip, value_norm=value_norm,
                          kl_coef=beta)
    kl_out = torch.full((2,), -1.0, device=d) if kl else None
    res = ops.ppo_loss_fwd_bwd([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                               [actions[k].to(d) for k in HEADS], old.to(d), adv.to(d), ret.to(d), values.to(d),
                               None, None, None, hparams=hp, old_value=ov.to(d),
                               valid=None if valid is None else valid.to(d), joint=joint,
                               old_log_probs=rows.to(d) if kl else None, kl_out=kl_out)
    return res, kl_out


@pytest.mark.parametrize("n,drop,pad", [(300, None, None), (1000, "target_unit", 900), (131072, None, None)])
@pytest.mark.parametrize("joint", [False, True])
@pytest.mark.parametrize("with_valid", [False, True])
@pytest.mark.parametrize("value_clip", [None, 0.05])
@pytest.mark.parametrize("value_norm", [None, (0.3, 1.7)])
def test_kl_kernel_vs_oracle(n, drop, pad, joint, with_valid, value_clip, value_norm):
    """Loss, statistics, kl_out, dlogits and dvalue of dc_ppo_loss_fwd_bwd_kl (beta > 0) against the float64 oracle.  Under
    PopArt (value_norm = (mu, sigma)) the oracle's value targets and old values are (x - mu) / sigma, as the kernel reads
    them."""
    inputs = JR._inputs(n, 11 + n, drop, pad, with_valid)
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    rows = _old_rows(logits, masks, 3 + n)
    mu, sigma = value_norm if value_norm is not None else (0.0, 1.0)
    ret_n, ov_n = (ret.double() - mu) / sigma, (ov.double() - mu) / sigma
    lg = {k: v.double().requires_grad_(True) for k, v in logits.items()}
    vg = values.double().requires_grad_(True)
    loss, p_loss, e_loss, v_loss, ents, kl = KO.kl_ppo_loss(
        lg, vg, actions, masks, old.double(), rows.double(), adv.double(), ret_n, 5e-4, 0.5, E_CLIP, BETA,
        joint=joint, valid=valid, old_values=ov_n, value_clip=value_clip)
    loss.backward()
    _, kl_sum, t_a, per_head = KO.exact_kl({k: v.double() for k, v in logits.items()}, actions, masks, rows.double(), valid)
    (out, n_act, dlogits, dvalue, stats), kl_out = _run(inputs, rows, joint, BETA, value_clip, value_norm)
    out = out.cpu().numpy()
    st = stats.cpu()
    for i, want in enumerate((loss, p_loss, e_loss, v_loss)):
        np.testing.assert_allclose(out[i], float(want.detach()), rtol=1e-4, atol=1e-6, err_msg=str(i))
    assert float(kl.detach()) > 0
    np.testing.assert_allclose(float(st[16]), float(kl), rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(float(st[22]), BETA * float(kl), rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(st[17:22].numpy(), [per_head[k] for k in HEADS], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(float(kl_out[0]), float(kl_sum), rtol=1e-4)
    assert float(kl_out[1]) == t_a
    for h, k in enumerate(HEADS):
        g_ref = lg[k].grad.float() if lg[k].grad is not None else torch.zeros_like(logits[k])
        torch.testing.assert_close(dlogits[h].cpu(), g_ref, rtol=2e-4, atol=1e-8)
        if valid is not None:
            assert bool((dlogits[h].cpu()[~valid] == 0).all()), k
    if pad is not None:                            # empty-mask rows stay exactly 0
        assert all(bool((dlogits[h][pad:] == 0).all()) for h in range(5))
    # dvalue does not see the KL term.  Under the value clip, a token whose two value-loss branches tie within fp32
    # rounding may take the other branch in fp32 than in float64 (the KL-free entry points have the same property), so
    # such near-ties are left out of the comparison
    keep = torch.ones(n, dtype=torch.bool)
    if value_clip is not None:
        r, v, vo = ret_n, values.double(), ov_n
        l1, l2 = (v - r) ** 2, (vo + (v - vo).clamp(-value_clip, value_clip) - r) ** 2
        keep = (l1 - l2).abs() > 1e-5 * torch.maximum(l1, l2)
    torch.testing.assert_close(dvalue.cpu()[keep], vg.grad.float()[keep], rtol=1e-4, atol=1e-9)


@pytest.mark.parametrize("joint", [False, True])
@pytest.mark.parametrize("with_valid", [False, True])
@pytest.mark.parametrize("value_clip", [None, 0.05])
@pytest.mark.parametrize("value_norm", [None, (0.3, 1.7)])
def test_beta_zero_is_the_existing_entry_point_bitwise(joint, with_valid, value_clip, value_norm):
    n = 131072
    inputs = JR._inputs(n, 29, None, None, with_valid)
    rows = _old_rows(inputs[0], inputs[1], 31)
    (a, kl_out), (b, _) = _run(inputs, rows, joint, 0.0, value_clip, value_norm), \
        _run(inputs, rows, joint, 0.0, value_clip, value_norm, kl=False)
    out_a, n_a, dl_a, dv_a, st_a = a
    out_b, n_b, dl_b, dv_b, st_b = b
    assert torch.equal(out_a, out_b) and torch.equal(n_a, n_b) and torch.equal(dv_a, dv_b)
    assert all(torch.equal(x, y) for x, y in zip(dl_a, dl_b))
    assert torch.equal(st_a[:16], st_b[:16]) and bool((st_b[16:] == 0).all())
    assert float(st_a[16]) > 0 and float(st_a[22]) == 0.0 and float(kl_out[1]) > 0


def test_stored_rows_and_kl_at_the_prep_policy():
    """dc_selected_logp_rows: the selected log-probs bit for bit, rows equal to the oracle's masked log-softmax, and a KL of
    (about) 0 with a non-negative value when the loss sees the same logits; KL >= 0 once they move."""
    from dotaclient_b200 import ops
    n = 131072
    inputs = JR._inputs(n, 41, None, 120000, True)
    logits, masks, actions = inputs[0], inputs[1], inputs[2]
    d = P.dev()
    args = ([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS], [actions[k].to(d) for k in HEADS])
    sel, rows = ops.selected_logp_rows(*args)
    assert torch.equal(sel, ops.selected_logp(*args))
    want = KO.masked_log_rows({k: v.double() for k, v in logits.items()}, masks)
    torch.testing.assert_close(rows.cpu().double(), want, rtol=1e-5, atol=2e-5)
    legal = torch.cat([masks[k] for k in HEADS], dim=1)
    assert bool((rows.cpu()[~legal] == 0).all())
    col = 0
    for h, k in enumerate(HEADS):                   # the selected entry of a row is the selected log-prob, bit for bit
        acted = actions[k].any(dim=1)
        picked = (rows.cpu()[:, col:col + KO.SIZES[h]] * actions[k].float()).sum(dim=1)
        assert torch.equal(picked[acted], sel.cpu()[acted, h]), k
        col += KO.SIZES[h]
    (_, _, _, _, st), kl_out = _run(inputs, rows.cpu(), False, BETA)
    assert abs(float(st[16])) < 1e-6 and float(kl_out[1]) > 0
    (_, _, _, _, st), _ = _run(inputs, _old_rows(logits, masks, 5), True, BETA)
    assert float(st[16]) > 0 and bool((st[17:22] >= 0).all())


# ------------------------------------------------------------------------------------------------ the optimizer
def _snapshot(opt):
    return (opt.flat.param.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.adam_steps.clone())


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def test_prep_rows_survive_chunking_packing_and_gather(tmp_path):
    a = JR.make_optimizer(tmp_path, mask_padding=True, kl_coef=0.2)
    b = JR.make_optimizer(tmp_path, mask_padding=True, pack_sequences=True, kl_coef=0.2)
    rollouts = PK.ragged_rollouts(a.policy_base, 6, False, False)
    seqs = [s for r in a.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in r]
    chunked = a.batch_from_rollouts(copy.deepcopy(rollouts))
    assert chunked.old_log_probs.shape == chunked.old_logp.shape[:2] + (65,)
    for j, s in enumerate(seqs):
        assert torch.equal(chunked.old_log_probs[:, j], s.old_log_probs), j
    idx = [3, 0, 2]
    gathered = chunked.gather(idx)
    assert torch.equal(gathered.old_log_probs, chunked.old_log_probs[:, idx])
    packed = b.batch_from_rollouts(copy.deepcopy(rollouts))
    # every real token of the packed batch carries the row of the same (rollout, step) as the chunked batch
    rows_c = chunked.old_log_probs[chunked.valid]
    rows_p = packed.old_log_probs[packed.valid]
    key = lambda r: r[:, 0] * 1e3 + r[:, 13] + r[:, 64]      # noqa: E731
    assert torch.equal(torch.sort(key(rows_c)).values, torch.sort(key(rows_p)).values)
    # the KL at the prep-time weights is (about) 0 on the first step, and never negative beyond rounding
    a.train(chunked)
    st = a.last_ppo_stats
    assert -1e-6 <= st["kl"] < 1e-4 and st["kl_skipped"] == 0.0 and -1e-6 <= st["kl_all_ranks"] < 1e-4


def test_train_refuses_a_batch_without_rows(tmp_path):
    a = JR.make_optimizer(tmp_path, mask_padding=True, kl_stop=0.1)
    plain = JR.make_optimizer(tmp_path, mask_padding=True)
    rollouts = PK.ragged_rollouts(a.policy_base, 4, False, False)
    batch = plain.batch_from_rollouts(copy.deepcopy(rollouts))
    assert batch.old_log_probs is None and plain.flat.kl_tail is None
    with pytest.raises(ValueError, match="old_log_probs"):
        a.train(batch)
    plain.kl_coef = 0.3
    with pytest.raises(ValueError, match="KL control is off"):
        plain.train(batch)


@pytest.mark.parametrize("joint", [False, True])
def test_penalty_step_eager_equals_replayed_and_moves_with_beta(joint, tmp_path):
    """A train() step with kl_coef > 0: the graph replay is bit-identical to the eager step, and a beta schedule between
    steps reaches the replays (the loss moves by beta KL)."""
    mode = "joint" if joint else "per_head"
    a = JR.make_optimizer(tmp_path, mask_padding=True, policy_ratio=mode, kl_coef=0.5)
    b = JR.make_optimizer(tmp_path, mask_padding=True, policy_ratio=mode, kl_coef=0.5)
    b.use_cuda_graph = False
    rollouts = PK.ragged_rollouts(a.policy_base, 8, False, False)
    ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    schedule = [dict(learning_rate=3e-3), dict(), dict(), dict(kl_coef=4.0), dict(kl_coef=0.0)]
    pens = []
    for step, change in enumerate(schedule):
        rec = []
        for opt, batch in ((a, ba), (b, bb)):
            for k, v in change.items():
                setattr(opt, k, v)
            losses, _, norms = opt.train(batch)
            rec.append(([float(v) for v in losses.values()], [float(v) for v in norms.values()], dict(opt.last_ppo_stats)))
        assert rec[0] == rec[1], step
        assert _same(_snapshot(a), _snapshot(b)), step
        pens.append(rec[0][2])
    assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"
    assert pens[2]["kl"] > 0 and abs(pens[2]["kl_penalty"] - 0.5 * pens[2]["kl"]) <= 1e-5 * pens[2]["kl_penalty"]
    assert abs(pens[3]["kl_penalty"] - 4.0 * pens[3]["kl"]) <= 1e-5 * pens[3]["kl_penalty"]
    assert pens[4]["kl_penalty"] == 0.0


@pytest.mark.parametrize("graph", [False, True])
def test_early_stop_leaves_the_state_untouched(graph, tmp_path):
    """A limit the second step crosses: that step returns normally, says it skipped, and leaves the parameters, Adam
    moments and step counters bitwise unchanged; a later limit change reaches the (replayed) step."""
    a = JR.make_optimizer(tmp_path, mask_padding=True, kl_stop=1e-4)
    a.learning_rate = 1e-2
    a.use_cuda_graph = graph
    batch = a.batch_from_rollouts(copy.deepcopy(PK.ragged_rollouts(a.policy_base, 8, False, False)))
    a.train(batch)
    assert a.last_ppo_stats["kl_skipped"] == 0.0
    before = _snapshot(a)
    a.train(batch)
    st = a.last_ppo_stats
    assert st["kl_skipped"] == 1.0 and st["kl_all_ranks"] > 1e-4
    assert _same(before, _snapshot(a))
    a.train(batch)                                   # still above the limit: skipped again (graph replay when graph)
    assert a.last_ppo_stats["kl_skipped"] == 1.0 and _same(before, _snapshot(a))
    a.kl_stop = 10.0                                 # a limit change between steps reaches the replay
    a.train(batch)
    assert a.last_ppo_stats["kl_skipped"] == 0.0 and not torch.equal(before[0], a.flat.param)
    assert bool((a.adam_steps >= before[3]).all()) and int((a.adam_steps - before[3]).max()) == 1
    if graph:
        assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"


def test_train_epochs_stops_at_the_first_skip(tmp_path):
    a = JR.make_optimizer(tmp_path, mask_padding=True, kl_stop=1e-4, epochs=4, min_seq=4, num_minibatches=2)
    a.learning_rate = 1e-2
    batch = a.batch_from_rollouts(copy.deepcopy(PK.ragged_rollouts(a.policy_base, 8, False, False)))
    state = a.minibatch_rng.bit_generator.state
    losses, _, _, stats = a.train_epochs(batch)
    skipped = [s["kl_skipped"] for s in stats]
    assert skipped[-1] == 1.0 and all(v == 0.0 for v in skipped[:-1]) and len(stats) < 8
    run = len(stats) - 1
    assert a.last_kl_updates == (run, 8 - run)
    # the shuffles of the epochs that did not run were not drawn
    import numpy as np_
    from dotaclient_b200.optimizer import minibatch_indices
    rng = np_.random.default_rng()
    rng.bit_generator.state = state
    for _ in range((len(stats) + 1) // 2):
        list(minibatch_indices(batch.batch_size, 2, rng))
    assert rng.bit_generator.state == a.minibatch_rng.bit_generator.state


def test_run_iteration_adapts_beta_and_reports_the_metrics(tmp_path):
    """Two iterations with kl_target: beta moves by the rule from the mean all-ranks KL of each iteration's steps."""
    from dotaclient_b200.optimizer import MessageQueue, kl_coef_update
    port = uuid.uuid4().int % 100000
    opt = JR.make_optimizer(tmp_path, min_seq=6, port=port, epochs=3, mask_padding=True, kl_coef=0.3, kl_target=1e-6,
                            kl_stop=50.0)
    opt.learning_rate = 3e-3
    actor = MessageQueue(host="joint", port=port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for it in range(2):
        for i, L in enumerate((40, 23, 57)):
            actor.publish_experience(pickle.dumps(make_rollout(L, 970 + 10 * it + i, game_id=i, weight_version=1)))
    betas = [opt.kl_coef]
    for it in (1, 2):
        m = opt.run_iteration(it)
        assert m["kl/coef"] == betas[-1]
        assert m["kl/updates_run"] == 3 and m["kl/updates_skipped"] == 0
        for k in ["ppo/kl", "ppo/kl_penalty"] + ["ppo/kl/" + h for h in HEADS]:
            assert math.isfinite(m[k]) and m[k] >= -1e-6, k
        assert opt.kl_coef == kl_coef_update(betas[-1], m["kl/all_ranks"], 1e-6)
        betas.append(opt.kl_coef)
    assert betas == [0.3, 0.6, 1.2]                 # the KL after an update at lr 3e-3 is far above 1.5e-6


# ------------------------------------------------------------------------------------------------ whole steps vs the oracle
def _legal(masks):
    return torch.cat([masks[k].bool() for k in HEADS], dim=-1)


def _tempered_sequences(mine, rollouts):
    """Prep's sequences with their old rows replaced by a different policy's (``kl_oracle.temper_rows``), so that the KL
    term and its gradient are large from the first step; the oracle's CPU copies carry the same rows."""
    xs_m = [s for grp in mine.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in grp]
    for s in xs_m:
        s.old_log_probs = KO.temper_rows(s.old_log_probs, _legal(s.masks))
    xs_o = JR._cpu_sequences(xs_m)
    for o, s in zip(xs_o, xs_m):
        o.old_log_probs = s.old_log_probs.cpu()
    return xs_m, xs_o


def _check_step(lm, em, gm, lo, eo, go, tag):
    for k in lo:
        np.testing.assert_allclose(float(lm[k]), float(lo[k].detach()), rtol=2e-4, atol=2e-6, err_msg="%s %s" % (k, tag))
    for k in eo:
        np.testing.assert_allclose(float(em[k]), float(eo[k].detach()), rtol=2e-4, atol=1e-6, err_msg="entropy %s %s" % (k, tag))
    np.testing.assert_allclose(float(gm["unclipped"]), float(go["unclipped"]), rtol=2e-3, err_msg=tag)
    np.testing.assert_allclose(float(gm["clipped"]), float(go["clipped"]), rtol=2e-3, err_msg=tag)


def _check_grads(mine, oracle, tag):
    for name, p in oracle.policy_base.named_parameters():
        g = mine.flat.grad_of(name).cpu()
        cos = torch.nn.functional.cosine_similarity(g.flatten(), p.grad.flatten(), dim=0)
        assert cos > 0.9999, (tag, name, float(cos))
        np.testing.assert_allclose(float(g.norm()), float(p.grad.norm()), rtol=2e-3, err_msg="%s %s" % (tag, name))


def _check_adam(mine, oracle, steps):
    sd = mine.optimizer.state_dict()["state"]
    want = P._adam_state_by_name(oracle)
    names = [n for n, _ in oracle.policy_base.named_parameters()]
    assert sorted(names[i] for i in sd) == sorted(want)
    for i, st in sd.items():
        w = want[names[i]]
        assert float(st["step"]) == float(w["step"]) == float(steps)
        m_scale = float(w["exp_avg"].abs().max())
        v_scale = float(w["exp_avg_sq"].abs().max())
        torch.testing.assert_close(st["exp_avg"], w["exp_avg"], rtol=2e-3, atol=2e-3 * m_scale + 1e-12)
        torch.testing.assert_close(st["exp_avg_sq"], w["exp_avg_sq"], rtol=4e-3, atol=4e-3 * v_scale + 1e-20)


STEP_BETA = 1.0


@pytest.mark.parametrize("H,cell,joint,masked", [(128, "lstm", False, True), (128, "lstm", True, True),
                                                 (128, "lstm", False, False), (256, "gru", True, True)])
def test_kl_step_vs_oracle(H, cell, joint, masked, tmp_path):
    """Three train() steps with kl_coef > 0 against the reference optimizer whose loss adds beta * KL (kl_oracle), on the
    same sequences: the first step launch by launch, the next two replayed from the captured graph.  Losses (the total
    includes the penalty), entropies, grad norms, per-tensor gradients (cosine and norm) of the first and the last step,
    the KL, and the Adam moments after two steps, at the tolerances of the joint-ratio step test."""
    torch.set_num_threads(8)
    S = 16
    mine = JR.make_optimizer(tmp_path, hidden_size=H, cell=cell, mask_padding=masked,
                             policy_ratio="joint" if joint else "per_head", kl_coef=STEP_BETA)
    torch.manual_seed(7)
    oracle = KO.KLRefOptimizer(StackedRefPolicy(H, cell, 1), seq_len=S, kl_coef=STEP_BETA, joint=joint, masked=masked)
    xs_m, xs_o = _tempered_sequences(mine, PK.ragged_rollouts(mine.policy_base, 6, False, False))
    for ep in range(3):
        lm, em, gm = mine.train(xs_m)
        lo, eo, go = oracle.train(xs_o)
        _check_step(lm, em, gm, lo, eo, go, "step %d" % ep)
        st = mine.last_ppo_stats
        np.testing.assert_allclose(st["kl"], oracle.last_kl, rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(st["kl_penalty"], STEP_BETA * oracle.last_kl, rtol=1e-4, atol=1e-7)
        assert st["kl_penalty"] > 0.05 and st["kl_skipped"] == 0.0, st
        if ep in (0, 2):
            _check_grads(mine, oracle, "step %d" % ep)
        if ep == 1:                 # after a launch-by-launch and a replayed step, as the parity suite compares them
            _check_adam(mine, oracle, 2)
    assert any(isinstance(v, tuple) for v in mine._graphs.values()), "the step was never captured"


def test_kl_minibatch_steps_vs_oracle(tmp_path):
    """Minibatch steps: the chunked batch's columns gathered on the device (T_a and the advantage normalisation are the
    minibatch's) against the oracle trained on the same sequences, two steps on two different minibatches."""
    torch.set_num_threads(8)
    mine = JR.make_optimizer(tmp_path, mask_padding=True, kl_coef=STEP_BETA)
    torch.manual_seed(7)
    oracle = KO.KLRefOptimizer(StackedRefPolicy(128, "lstm", 1), seq_len=16, kl_coef=STEP_BETA)
    rollouts = PK.ragged_rollouts(mine.policy_base, 6, False, False)
    _, xs_o = _tempered_sequences(mine, rollouts)
    batch = mine.batch_from_rollouts(copy.deepcopy(rollouts))
    batch.old_log_probs = KO.temper_rows(batch.old_log_probs, _legal(batch.masks))
    B = batch.batch_size
    assert B >= 4
    for step, idx in enumerate((list(range(0, B, 2)), list(range(B - 1, 0, -2)))):
        lm, em, gm = mine.train(batch.gather(idx))
        lo, eo, go = oracle.train([xs_o[j] for j in idx])
        _check_step(lm, em, gm, lo, eo, go, "minibatch %d" % step)
        np.testing.assert_allclose(mine.last_ppo_stats["kl"], oracle.last_kl, rtol=1e-4, atol=1e-7)
        _check_grads(mine, oracle, "minibatch %d" % step)
    _check_adam(mine, oracle, 2)


@pytest.mark.parametrize("joint", [False, True])
def test_packed_kl_step_equals_unpacked(joint, tmp_path):
    """The packed batch holds the unpacked masked batch's valid tokens with the same old rows: two steps with the penalty
    on each agree to the packing suite's tolerances (losses, grad norms, statistics including the KL, gradients, weights)."""
    kw = dict(mask_padding=True, policy_ratio="joint" if joint else "per_head", kl_coef=STEP_BETA)
    unpacked = JR.make_optimizer(tmp_path, **kw)
    packed = JR.make_optimizer(tmp_path, pack_sequences=True, **kw)
    rollouts = PK.ragged_rollouts(unpacked.policy_base, 3, False, True)
    bu = unpacked.batch_from_rollouts(copy.deepcopy(rollouts))
    bp = packed.batch_from_rollouts(copy.deepcopy(rollouts))
    assert bp.batch_size < bu.batch_size
    for b in (bu, bp):
        b.old_log_probs = KO.temper_rows(b.old_log_probs, _legal(b.masks))
    for step in range(2):
        lu, eu, gu = unpacked.train(bu)
        lp, ep, gp = packed.train(bp)
        for k in lu:
            assert PK._close(lp[k], lu[k], 2e-4, 2e-6), (step, k, float(lp[k]), float(lu[k]))
        for k in gu:
            assert PK._close(gp[k], gu[k], 2e-3), (step, k)
        assert unpacked.last_ppo_stats["kl_penalty"] > 0.05
        for k, v in unpacked.last_ppo_stats.items():
            assert abs(packed.last_ppo_stats[k] - v) <= 2e-4 * abs(v) + 2e-5, (step, k, packed.last_ppo_stats[k], v)
        fu, fp = unpacked.flat, packed.flat
        for name, lo, hi in zip(fu.names, fu.starts, fu.ends):
            assert PK._close(fp.grad[lo:hi], fu.grad[lo:hi], 2e-3, 1e-9), (step, "grad", name)
        assert PK._close(fp.param, fu.param, 0.0, 1e-6), (step, "weights")


def test_run_iteration_reports_a_skip(tmp_path):
    """A limit the second step crosses: run_iteration returns, runs one update of the four planned, reports the skip, and
    its iteration means include the skipped step (its loss and KL were measured at the parameters it did not update)."""
    from dotaclient_b200.optimizer import MessageQueue
    port = uuid.uuid4().int % 100000
    opt = JR.make_optimizer(tmp_path, min_seq=6, port=port, epochs=4, mask_padding=True, kl_stop=1e-4)
    opt.learning_rate = 1e-2
    actor = MessageQueue(host="joint", port=port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for i, L in enumerate((40, 23, 57)):
        actor.publish_experience(pickle.dumps(make_rollout(L, 990 + i, game_id=i, weight_version=1)))
    steps_before = opt.adam_steps.clone()
    m = opt.run_iteration(1)
    assert (m["kl/updates_run"], m["kl/updates_skipped"]) == (1, 3)
    assert int((opt.adam_steps - steps_before).max()) == 1
    assert m["kl/all_ranks"] > 1e-4 / 2 and m["kl/coef"] == 0.0 and "ppo/kl_skipped" not in m
    assert math.isfinite(m["loss/sum"]) and m["ppo/kl"] > 0
