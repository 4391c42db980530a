"""GPU tests of dual-clip PPO (``DotaOptimizer(dual_clip=c)``): ``dc_ppo_loss_fwd_bwd_dual_clip`` against the float64
oracle (``dual_clip_oracle.py``) at C2's 131,072 tokens in both ratio modes, with and without ``valid``, alone, with the KL
penalty's rows, with the teacher's and with both; a c no ratio reaches against the entry point the call would otherwise be,
bit for bit; the zero gradient of bound rows; graph replays against eager steps and a changed c reaching the replays; the
default step and a step whose c binds nowhere; composition with value heads, PopArt and kl_stop; and two ranks over gloo.

The old log-probs are the kernel's own selected log-probs moved by up to +-3 nats, so ratios span about [0.05, 20] and a
sizeable share of the negative-advantage rows bind at c = 3.  Rows whose float64 ratio lies within 1e-4 of a clip bound or
of c are moved off it, so that the fp32 kernel and the oracle clip and bind the same rows.  Tolerances are the teacher
suite's (``test_gpu_teacher``): rtol 1e-4 on the losses and statistics, 2e-4 on dlogits."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dual_clip_oracle as DO  # noqa: E402
import joint_ratio_oracle as JO  # noqa: E402
import kl_oracle as KO  # noqa: E402
import test_gpu_joint_ratio as JR  # noqa: E402
import test_gpu_packing as PK  # noqa: E402
import test_gpu_parity as P  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS = P.HEADS
E_CLIP = JR.E_CLIP
C = 3.0
BETA, LAMBDA = 0.7, 1.3
N_C2 = 131072
COMBOS = [(False, False), (True, False), (False, True), (True, True)]     # (KL rows, teacher rows)


def _rows(logits, masks, seed, scale):
    """A policy's rows near the current one: the masked log-softmax of perturbed logits, in fp32."""
    g = torch.Generator().manual_seed(seed)
    moved = {k: v.double() + scale * torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in logits.items()}
    return KO.masked_log_rows(moved, masks).float()


def _inputs(n, seed, joint, with_valid):
    """Loss inputs whose ratios span about [0.05, 20]: the old log-probs are dc_selected_logp's plus offsets uniform in
    [-3, 3] (per head; under the joint ratio on the first head of the token's action only, so the joint ratio spans the
    same range), zero on every third token.  Heads without an action row get an old log-prob of 99.  Rows within 1e-4 of
    1 - e, 1 + e or c are moved off them."""
    from dotaclient_b200 import ops
    logits, masks, actions, _, values, adv, ret = P._random_loss_inputs(n, seed, None, None)
    d = P.dev()
    g = torch.Generator().manual_seed(seed + 1)
    lp = ops.selected_logp([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                           [actions[k].to(d) for k in HEADS]).cpu()
    acted = torch.stack([actions[k].any(dim=1) for k in HEADS], dim=1)
    offs = 6.0 * torch.rand(n, 5, generator=g) - 3.0
    if joint:
        first = acted.double().argmax(dim=1)
        offs = torch.where(torch.arange(5)[None, :] == first[:, None], offs, torch.zeros_like(offs))
    offs[::3] = 0.0
    old = torch.where(acted, lp + offs, torch.full_like(lp, 99.0))
    valid = None
    if with_valid:
        valid = torch.rand(n, generator=g) < 0.8
        valid[: min(n, 3)] = True
    lg = {k: v.double() for k, v in logits.items()}
    bounds = (1.0 - E_CLIP, 1.0 + E_CLIP, C)
    if joint:
        log_r, has, _ = JO.joint_log_ratio(lg, actions, masks, old.double(), valid)
        r = torch.exp(log_r)
        near = has & torch.stack([(r - b).abs() < 1e-4 * b for b in bounds]).any(dim=0)
        for t in torch.nonzero(near).flatten().tolist():
            old[t, int(torch.nonzero(acted[t])[0])] -= 1e-3
    else:
        from oracle.ref_policy import masked_softmax
        for h, k in enumerate(HEADS):
            lpk = masked_softmax(lg[k], masks[k].bool(), dim=1)
            sel = lpk.masked_fill(~actions[k].bool(), 0.0).sum(dim=1)
            r = torch.exp(sel - old[:, h].double())
            near = acted[:, h] & torch.stack([(r - b).abs() < 1e-4 * b for b in bounds]).any(dim=0)
            old[near, h] -= 1e-3
    ov = values + 0.1 * torch.randn(n, generator=g)
    return logits, masks, actions, old, values, adv, ret, ov, valid


def _run(inputs, joint, old_rows, teacher_rows, c, entropy_coef=5e-4, beta=BETA):
    """One loss call: ``_dual_clip`` when c is given, else the entry point the same operands select without it."""
    from dotaclient_b200 import ops
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    d = P.dev()
    hp = ops.hparam_block(d, e_clip=E_CLIP, entropy_coef=entropy_coef, vf_coef=0.5, kl_coef=beta)
    kl_out = torch.full((2,), -1.0, device=d) if old_rows is not None else None
    kw = {}
    if teacher_rows is not None:
        kw.update(teacher_log_probs=teacher_rows.to(d),
                  teacher_coef=torch.tensor([LAMBDA], dtype=torch.float64, device=d))
    if c is not None:
        kw.update(dual_clip=torch.tensor([c], dtype=torch.float64, device=d))
    res = ops.ppo_loss_fwd_bwd([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                               [actions[k].to(d) for k in HEADS], old.to(d), adv.to(d), ret.to(d), values.to(d),
                               None, None, None, hparams=hp, old_value=ov.to(d),
                               valid=None if valid is None else valid.to(d), joint=joint,
                               old_log_probs=None if old_rows is None else old_rows.to(d), kl_out=kl_out, **kw)
    return res, kl_out


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("joint", [False, True])
@pytest.mark.parametrize("with_valid", [False, True])
@pytest.mark.parametrize("with_kl,with_teacher", COMBOS)
def test_dual_clip_kernel_vs_oracle(joint, with_valid, with_kl, with_teacher):
    """Loss, its terms, dual_clip_stats, kl_out, teacher_stats, dlogits and dvalue of dc_ppo_loss_fwd_bwd_dual_clip (c = 3)
    at 131,072 tokens against the float64 oracle."""
    inputs = _inputs(N_C2, 41, joint, with_valid)
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    old_rows = _rows(logits, masks, 3, 0.25) if with_kl else None
    t_rows = _rows(logits, masks, 5, 1.0) if with_teacher else None
    lg = {k: v.double().requires_grad_(True) for k, v in logits.items()}
    vg = values.double().requires_grad_(True)
    loss, p_loss, e_loss, v_loss, ents, fr = DO.dual_clip_ppo_loss(
        lg, vg, actions, masks, old.double(), adv.double(), ret.double(), 5e-4, 0.5, E_CLIP, C, joint=joint, valid=valid,
        old_rows=None if old_rows is None else old_rows.double(), kl_coef=BETA,
        teacher_rows=None if t_rows is None else t_rows.double(), teacher_coef=LAMBDA, old_values=ov.double())
    loss.backward()
    res, kl_out = _run(inputs, joint, old_rows, t_rows, C)
    out, n_act, dlogits, dvalue, stats = res[:5]
    dst = res[-1].cpu()
    out = out.cpu().numpy()
    for i, want in enumerate((loss, p_loss, e_loss, v_loss)):
        np.testing.assert_allclose(out[i], float(want.detach()), rtol=1e-4, atol=1e-6, err_msg=str(i))
    # a sizeable share binds, and the kernel binds the same rows as float64
    key = "fraction/joint" if joint else "fraction"
    assert fr[key] > 0.02, fr
    want = [fr["fraction"]] + [fr["fraction/" + k] for k in HEADS] + [fr["fraction/joint"]]
    np.testing.assert_allclose(dst.numpy(), want, rtol=1e-6, atol=1e-7)
    if with_kl:
        _, kl_sum, t_a, _ = KO.exact_kl({k: v.double() for k, v in logits.items()}, actions, masks, old_rows.double(), valid)
        assert float(kl_out[1]) == t_a
        np.testing.assert_allclose(float(kl_out[0]), float(kl_sum), rtol=1e-4)
    if with_teacher:
        kl_t = float(KO.exact_kl({k: v.double() for k, v in logits.items()}, actions, masks, t_rows.double(), valid)[0])
        np.testing.assert_allclose(float(res[5][0]), kl_t, rtol=1e-4, atol=1e-7)
    for h, k in enumerate(HEADS):
        g_ref = lg[k].grad.float() if lg[k].grad is not None else torch.zeros_like(logits[k])
        torch.testing.assert_close(dlogits[h].cpu(), g_ref, rtol=2e-4, atol=1e-8)
        if valid is not None:
            assert bool((dlogits[h].cpu()[~valid] == 0).all()), k
    torch.testing.assert_close(dvalue.cpu(), vg.grad.float(), rtol=1e-4, atol=1e-9)


@pytest.mark.parametrize("joint", [False, True])
@pytest.mark.parametrize("with_valid", [False, True])
@pytest.mark.parametrize("with_kl,with_teacher", COMBOS)
def test_unreached_c_is_the_other_entry_point_bitwise(joint, with_valid, with_kl, with_teacher):
    """c = 1e6, beyond every ratio: loss, n_actions, dlogits, dvalue, stats, kl_out and teacher_stats equal those of
    _masked / _dev / _joint / _kl / _teacher bit for bit, and nothing binds."""
    inputs = _inputs(N_C2, 43, joint, with_valid)
    old_rows = _rows(inputs[0], inputs[1], 31, 0.25) if with_kl else None
    t_rows = _rows(inputs[0], inputs[1], 37, 1.0) if with_teacher else None
    (a, kl_a), (b, kl_b) = _run(inputs, joint, old_rows, t_rows, 1e6), _run(inputs, joint, old_rows, t_rows, None)
    assert len(a) == len(b) + 1
    for x, y in zip(a[:len(b)], b):
        if isinstance(x, list):
            assert all(torch.equal(p, q) for p, q in zip(x, y))
        else:
            assert torch.equal(x, y)
    if with_kl:
        assert torch.equal(kl_a, kl_b)
    assert bool((a[-1] == 0).all())


@pytest.mark.parametrize("joint", [False, True])
def test_bound_rows_get_exactly_zero_gradient(joint):
    """entropy_coef = 0 and no KL or teacher: every row whose cap binds has a dlogits row of exactly 0, and a row that does
    not bind has a nonzero one."""
    from oracle.ref_policy import masked_softmax
    inputs = _inputs(N_C2, 47, joint, True)
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    res, _ = _run(inputs, joint, None, None, C, entropy_coef=0.0)
    dlogits = [x.cpu() for x in res[2]]
    a = DO.normalised_advantage(adv, valid)
    lg = {k: v.double() for k, v in logits.items()}
    use = valid.bool()
    if joint:
        log_r, has, _ = JO.joint_log_ratio(lg, actions, masks, old.double(), valid)
        _, bound = DO.dual_clip_term(torch.exp(log_r), a, E_CLIP, C)
        bound &= has
        rows = {k: bound & actions[k].any(dim=1) for k in HEADS}
        free = has & ~bound & (a > 0) & (torch.exp(log_r) < 1.0 + E_CLIP)
        free_rows = {k: free & actions[k].any(dim=1) for k in HEADS}
    else:
        rows, free_rows = {}, {}
        for h, k in enumerate(HEADS):
            act = actions[k].bool() & use[:, None]
            sel = masked_softmax(lg[k], masks[k].bool(), dim=1).masked_fill(~act, 0.0).sum(dim=1)
            r = torch.exp(sel - old[:, h].double())
            _, bound = DO.dual_clip_term(r, a, E_CLIP, C)
            rows[k] = bound & act.any(dim=1)
            free_rows[k] = act.any(dim=1) & ~bound & (a > 0) & (r < 1.0 + E_CLIP)
    n_bound = sum(int(v.sum()) for v in rows.values())
    assert n_bound > 1000, n_bound
    for h, k in enumerate(HEADS):
        assert bool((dlogits[h][rows[k]] == 0).all()), k
        if int(free_rows[k].sum()):
            assert bool((dlogits[h][free_rows[k]].abs().sum(dim=1) > 0).all()), k


# ------------------------------------------------------------------------------------------------ the optimizer
def _snapshot(opt):
    return (opt.flat.param.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.adam_steps.clone())


def _keys(stats):
    return {k for k in stats if "dual_clip" in k}


@pytest.mark.parametrize("joint", [False, True])
def test_replays_equal_eager_steps_and_pick_up_a_new_c(joint, tmp_path):
    """KL control with kl_stop, mask_padding + pack_sequences, 2 minibatches and both refreshes under dual clip: the
    epochs replayed from captured graphs equal the eager ones bit for bit (losses, statistics, parameters, Adam state);
    assigning opt.dual_clip between replays reaches the replayed step; an invalid value is refused at the next train()."""
    ratio = "joint" if joint else "per_head"
    kw = dict(mask_padding=True, pack_sequences=True, policy_ratio=ratio, kl_coef=0.3, kl_stop=10.0, num_minibatches=2,
              recompute_advantages=True, recompute_states=True, epochs=3, min_seq=4, dual_clip=1.5)
    a = JR.make_optimizer(tmp_path, **kw)
    b = JR.make_optimizer(tmp_path, **kw)
    b.use_cuda_graph = False
    for o in (a, b):
        o.learning_rate = 3e-3
    rollouts = PK.ragged_rollouts(a.policy_base, 9, False, True)
    ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    fractions = []
    for rep, c in enumerate((1.5, 1.5, 1.05)):       # the second pass replays every shape; the third changes c
        a.dual_clip = b.dual_clip = c
        ra, rb = a.train_epochs(ba), b.train_epochs(bb)
        assert [dict(s) for s in ra[3]] == [dict(s) for s in rb[3]], rep
        assert [{k: float(v) for k, v in x.items()} for x in ra[0]] == [{k: float(v) for k, v in x.items()} for x in rb[0]]
        assert all(torch.equal(x, y) for x, y in zip(_snapshot(a), _snapshot(b))), rep
        want = {"dual_clip_fraction"} | {"dual_clip_fraction/" + k for k in HEADS}
        assert all(_keys(s) == (want | {"dual_clip_fraction/joint"} if joint else want) for s in ra[3])
        fractions.append(max(s["dual_clip_fraction/joint" if joint else "dual_clip_fraction"] for s in ra[3]))
        assert a.last_dual_clip_stats["fraction"] == ra[3][-1]["dual_clip_fraction"]
    assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"
    print("\nlargest bound fraction per pass (c = 1.5, 1.5, 1.05): %s" % fractions)
    assert fractions[1] > 0 and fractions[2] > fractions[1]      # a smaller c binds more rows, replayed
    for bad in (1.0, float("nan"), None):
        a.dual_clip = bad
        with pytest.raises(ValueError, match="dual_clip="):
            a.train(ba)
    off = JR.make_optimizer(tmp_path, mask_padding=True)
    off.dual_clip = 3.0                              # fixed off at construction
    with pytest.raises(ValueError, match="dual_clip="):
        off.train(off.batch_from_rollouts(copy.deepcopy(rollouts)))


def test_default_step_and_an_unreached_c_are_the_same_step(tmp_path):
    """The default optimizer (dual_clip=None) runs the parent's kernels and host code; a c no ratio reaches runs the
    dual-clip instantiation and must give the same step bit for bit: losses, statistics, parameters and Adam state over two
    epochs of replayed steps.  The default reports no dual-clip keys and attaches nothing."""
    kw = dict(mask_padding=True, epochs=2, min_seq=4)
    a = JR.make_optimizer(tmp_path, **kw)
    b = JR.make_optimizer(tmp_path, dual_clip=1e6, **kw)
    assert a._dual_clip_stats is None and a._hparams_dev_flat.numel() == 10 and a.last_dual_clip_stats is None
    rollouts = PK.ragged_rollouts(a.policy_base, 5, False, False)
    ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    for rep in range(2):
        ra, rb = a.train_epochs(ba), b.train_epochs(bb)
        assert [{k: float(v) for k, v in x.items()} for x in ra[0]] == [{k: float(v) for k, v in x.items()} for x in rb[0]]
        for sa, sb in zip(ra[3], rb[3]):
            assert not _keys(sa) and sb["dual_clip_fraction"] == 0.0
            assert dict(sa) == {k: v for k, v in sb.items() if "dual_clip" not in k}
        assert all(torch.equal(x, y) for x, y in zip(_snapshot(a), _snapshot(b))), rep
    assert a.last_dual_clip_stats is None


def _move_old_logp(*batches):
    """Moves every batch's prep-time log-probs by the same offsets, uniform in [-2, 2], so that the first step already
    has ratios far from 1 and the cap binds on some rows."""
    torch.cuda.synchronize()
    g = torch.Generator().manual_seed(5)
    offs = 4.0 * torch.rand(batches[0].old_logp.shape, generator=g) - 2.0
    for b in batches:
        b.old_logp.add_(offs.to(b.old_logp.device))


@pytest.mark.parametrize("kw", [dict(value_heads=True), dict(value_norm=True), dict(kl_coef=0.2, kl_stop=1e-6)],
                         ids=["value_heads", "popart", "kl_stop"])
def test_composition_leaves_the_value_side_alone(kw, tmp_path):
    """Value heads, PopArt and kl_stop with c = 1.5 on a batch whose ratios start far from 1: the step runs, the cap binds,
    and the value loss, the explained variance and the value heads' losses and explained variances equal those of the
    same step without dual clip bit for bit (the value term does not depend on the policy term).  Under kl_stop (a limit
    every later step exceeds) the second step is skipped by both and leaves parameters and Adam state alone."""
    from dotaclient_b200.optimizer import REWARD_KEYS
    kw = dict(kw)
    if "value_heads" in kw:
        kw["value_heads"] = {"win": ["win"], "rest": [k for k in REWARD_KEYS if k != "win"]}
    a = JR.make_optimizer(tmp_path, mask_padding=True, **kw)
    b = JR.make_optimizer(tmp_path, mask_padding=True, dual_clip=1.5, **kw)
    for o in (a, b):
        o.learning_rate = 3e-3
    rollouts = PK.ragged_rollouts(a.policy_base, 7, False, False)
    ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    _move_old_logp(ba, bb)
    la, lb = a.train(ba)[0], b.train(bb)[0]
    sa, sb = a.last_ppo_stats, b.last_ppo_stats
    assert sb["dual_clip_fraction"] > 0 and "dual_clip_fraction" not in sa
    assert float(la["value_loss"]) == float(lb["value_loss"])
    vkeys = [k for k in sa if k.startswith(("explained_variance", "loss/value"))]
    assert vkeys and all(sa[k] == sb[k] or (np.isnan(sa[k]) and np.isnan(sb[k])) for k in vkeys), vkeys
    assert float(la["policy_loss"]) != float(lb["policy_loss"])
    if "kl_stop" in kw:
        snaps = _snapshot(a), _snapshot(b)
        a.train(ba)
        b.train(bb)
        assert a.last_ppo_stats["kl_skipped"] == b.last_ppo_stats["kl_skipped"] == 1.0
        assert all(torch.equal(x, y) for x, y in zip(snaps[0], _snapshot(a)))
        assert all(torch.equal(x, y) for x, y in zip(snaps[1], _snapshot(b)))


def test_run_iteration_reports_the_fractions_and_c(tmp_path):
    """run_iteration reports ppo/dual_clip_fraction, per head and dual_clip/coef only when the feature is on."""
    import pickle
    import uuid
    from dotaclient_b200.optimizer import MessageQueue
    from dotaclient_b200.synthetic import make_rollout
    seen = {}
    for c in (None, 3.0):
        port = uuid.uuid4().int % 100000
        opt = JR.make_optimizer(tmp_path, port=port, mask_padding=True, dual_clip=c)
        actor = MessageQueue(host="joint", port=port, prefetch_count=1, use_model_exchange=False)
        actor.connect()
        for i, L in enumerate((40, 23)):
            actor.publish_experience(pickle.dumps(make_rollout(L, 600 + i, game_id=i, weight_version=1)))
        m = opt.run_iteration(1)
        seen[c] = {k for k in m if "dual_clip" in k}
        if c is not None:
            assert m["dual_clip/coef"] == c
        opt.close()
    assert seen[None] == set()
    assert seen[3.0] == {"dual_clip/coef", "ppo/dual_clip_fraction"} | {"ppo/dual_clip_fraction/" + k for k in HEADS}


def test_two_ranks_gloo_keep_identical_weights(tmp_path):
    import dual_clip_multi_rank as DM
    a, b = DM.run(tmp_path)
    assert torch.equal(a["param"], b["param"]) and torch.equal(a["steps"], b["steps"])
    assert a["coef"] == b["coef"] == [DM.C, DM.C]
    assert all(0.0 <= f <= 1.0 for f in a["fraction"] + b["fraction"])
