"""GPU tests of behaviour cloning (``DotaOptimizer(objective='bc')``): ``dc_ppo_loss_fwd_bwd_bc`` against the float64 oracle
(``bc_oracle.py``) at C2's token count; its value gradient against the default objective's, bit for bit; a student of
another architecture learning a seeded demonstrator's actions; replayed steps against eager ones; the published model; and
two ranks over gloo.

Tolerances are the KL control and teacher suites': fp32 against float64, rtol 1e-4 on the losses and statistics and 2e-4
on dlogits."""
import copy
import os
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bc_oracle as BO  # noqa: E402
import test_gpu_joint_ratio as JR  # noqa: E402
import test_gpu_packing as PK  # noqa: E402
import test_gpu_parity as P  # noqa: E402
from dotaclient_b200.synthetic import demonstration_rollout, make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS = P.HEADS
N_C2 = 131072


def _inputs(n, seed, with_valid):
    logits, masks, actions, _, values, adv, ret = P._random_loss_inputs(n, seed)
    g = torch.Generator().manual_seed(seed + 1)
    valid = None
    if with_valid:
        valid = torch.rand(n, generator=g) < 0.8
        valid[:3] = True
    ov = values + 0.1 * torch.randn(n, generator=g)
    return logits, masks, actions, values, adv, ret, ov, valid


def _run(inputs, bc, value_clip=None, entropy_coef=5e-4, vf_coef=0.5, value_norm=None):
    """One loss call: ``_bc`` or (old log-probs all 0) ``_masked`` / ``_dev``."""
    from dotaclient_b200 import ops
    logits, masks, actions, values, adv, ret, ov, valid = inputs
    d = P.dev()
    hp = ops.hparam_block(d, e_clip=0.2, entropy_coef=entropy_coef, vf_coef=vf_coef, value_clip=value_clip,
                          value_norm=value_norm)
    n = values.numel()
    return ops.ppo_loss_fwd_bwd([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                                [actions[k].to(d) for k in HEADS], None if bc else torch.zeros(n, 5, device=d),
                                adv.to(d), ret.to(d), values.to(d), None, None, None, hparams=hp, old_value=ov.to(d),
                                valid=None if valid is None else valid.to(d), bc=bc)


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("with_valid", [False, True])
@pytest.mark.parametrize("value_clip", [None, 0.2])
def test_bc_kernel_vs_oracle(with_valid, value_clip):
    """Loss terms, entropies, per-head NLL shares, n_actions, bc_stats, dlogits and dvalue of dc_ppo_loss_fwd_bwd_bc at
    C2's 131,072 tokens against the float64 oracle."""
    inputs = _inputs(N_C2, 41, with_valid)
    logits, masks, actions, values, adv, ret, ov, valid = inputs
    lg = {k: v.double().requires_grad_(True) for k, v in logits.items()}
    vg = values.double().requires_grad_(True)
    loss, l_nll, e_loss, v_loss, ents = BO.bc_loss(lg, vg, actions, masks, ret.double(), 5e-4, 0.5, valid=valid,
                                                   old_values=ov.double(), value_clip=value_clip)
    loss.backward()
    _, t_a, sums, counts = BO.nll({k: v.double() for k, v in logits.items()}, actions, masks, valid)
    acc, acc_h = BO.accuracy({k: v.double() for k, v in logits.items()}, actions, masks, valid)
    out, n_act, dlogits, dvalue, stats, bst = _run(inputs, True, value_clip)
    out, st, bst = out.cpu().numpy(), stats.cpu(), bst.cpu().numpy()
    for i, want in enumerate((loss, l_nll, e_loss, v_loss)):
        np.testing.assert_allclose(out[i], float(want.detach()), rtol=1e-4, atol=1e-6, err_msg=str(i))
    np.testing.assert_allclose(out[4:9], [float(ents[k]) for k in HEADS], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(out[9:14], [sums[k] / t_a for k in HEADS], rtol=1e-4, atol=1e-7)
    assert n_act.cpu().tolist() == [counts[k] for k in HEADS]
    np.testing.assert_allclose(bst[0], float(l_nll.detach()), rtol=1e-4)
    np.testing.assert_allclose(bst[1:6], [sums[k] / counts[k] for k in HEADS], rtol=1e-4)
    np.testing.assert_allclose(bst[6], acc, rtol=1e-6)
    np.testing.assert_allclose(bst[7:12], [acc_h[k] for k in HEADS], rtol=1e-6)
    assert 0.05 < acc < 0.95 and bool((st[:12] == 0).all()) and bool((st[13:] == 0).all())
    for h, k in enumerate(HEADS):
        g_ref = lg[k].grad.float()
        torch.testing.assert_close(dlogits[h].cpu(), g_ref, rtol=2e-4, atol=1e-8)
        if valid is not None:
            assert bool((dlogits[h].cpu()[~valid] == 0).all()), k
    torch.testing.assert_close(dvalue.cpu(), vg.grad.float(), rtol=1e-4, atol=1e-9)


def test_bc_kernel_without_entropy_is_the_closed_form():
    inputs = _inputs(4096, 43, True)
    logits, masks, actions, values, adv, ret, ov, valid = inputs
    out, _, dlogits, _, _, bst = _run(inputs, True, entropy_coef=0.0)
    closed = BO.nll_dlogits({k: v.double() for k, v in logits.items()}, actions, masks, valid)
    for h, k in enumerate(HEADS):
        torch.testing.assert_close(dlogits[h].cpu().double(), closed[k], rtol=2e-4, atol=1e-9)
    assert float(out[2]) == 0.0 and float(out[1]) == float(bst[0])


@pytest.mark.parametrize("value_norm", [None, (0.3, 1.7)])
@pytest.mark.parametrize("with_valid", [False, True])
def test_value_gradient_is_the_default_objectives_bitwise(value_norm, with_valid):
    """Same inputs under 'bc' and 'ppo': dvalue, the value loss, the entropies, n_actions and the explained variance are
    bit-identical (the value and entropy terms are the same code)."""
    inputs = _inputs(N_C2, 47, with_valid)
    a = _run(inputs, True, 0.2, value_norm=value_norm)
    b = _run(inputs, False, 0.2, value_norm=value_norm)
    assert torch.equal(a[3], b[3]) and torch.equal(a[1], b[1])
    assert torch.equal(a[0][2:9], b[0][2:9])
    assert torch.equal(a[4][12], b[4][12])


def test_value_heads_columns_are_the_default_objectives_bitwise():
    """K = 3 value heads on the packed GEMM output, as the step runs them: the loss with its value term off, then
    dc_value_heads_loss.  The K value columns of the gradient and the value loss are bit-identical under 'bc' and 'ppo'."""
    from dotaclient_b200 import _lib, ops
    d = P.dev()
    n, K = N_C2, 3
    logits, masks, actions, values, adv, ret, ov, valid = _inputs(n, 53, True)
    g = torch.Generator().manual_seed(5)
    packed = torch.zeros(n, ops.PACK_WIDTH)
    for k in ("enum", "x", "y", "ability"):
        lo, hi = ops.PACK_COLS[k]
        packed[:, lo:hi] = logits[k]
    packed[:, 25:25 + K] = torch.randn(n, K, generator=g)
    rets = torch.randn(n, K, generator=g)
    olds = packed[:, 25:25 + K] + 0.1 * torch.randn(n, K, generator=g)
    packed, tu = packed.to(d), logits["target_unit"].to(d)
    hp_full = ops.hparam_block(d, entropy_coef=5e-4, vf_coef=0.5, value_clip=0.2)
    hp_pol = ops.hparam_block(d, e_clip=0.2, entropy_coef=5e-4)
    res = []
    for bc in (True, False):
        r = ops.ppo_loss_packed(packed, tu, [masks[k].to(d) for k in HEADS], [actions[k].to(d) for k in HEADS],
                                None if bc else torch.zeros(n, 5, device=d), adv.to(d), adv.to(d), None, None, None,
                                hparams=hp_pol, valid=valid.to(d), bc=bc)
        out, _, d_packed = r[0], r[1], r[2]
        hs = torch.empty(_lib.VALUE_HEADS_STATS_SLOTS, device=d)
        ops.value_heads_loss(packed, d_packed, rets.to(d), hp_full, out, hs, old_value=olds.to(d), valid=valid.to(d),
                             stats=r[4])
        res.append((out.clone(), d_packed[:, 25:25 + K].clone(), hs.clone()))
    (oa, da, ha), (ob, db, hb) = res
    assert torch.equal(da, db) and torch.equal(ha, hb) and oa[3] == ob[3] and bool((da != 0).any())


# ------------------------------------------------------------------------------------------------ learning
def _demonstrator():
    """A seeded GRU-256 with habits: its head layers' weights are scaled by DEMO_SHARPEN and their biases drawn with a
    standard deviation of DEMO_BIAS, so that its actions have preferences a student can learn from a few thousand steps on
    top of their dependence on the observations."""
    from dotaclient_b200.policy import Policy
    torch.manual_seed(21)
    pol = Policy(hidden_size=256, cell="gru")
    with torch.no_grad():
        for layer in (pol.affine_head_enum, pol.affine_move_x, pol.affine_move_y, pol.affine_head_ability,
                      pol.affine_unit_attention):
            layer.weight.mul_(DEMO_SHARPEN)
            layer.bias.copy_(DEMO_BIAS * torch.randn(layer.bias.shape))
    return pol.to(P.dev())


def _held_out_metrics(pol, demos):
    """NLL and token accuracy of ``pol`` on the demonstrations, in float64 from its fp32 logits (forward from the zero
    state over every rollout)."""
    d = P.dev()
    lg, acts, masks = {k: [] for k in HEADS}, {k: [] for k in HEADS}, {k: [] for k in HEADS}
    with torch.no_grad():
        for r in demos:
            obs = {k: torch.as_tensor(v).unsqueeze(0).to(d) for k, v in r["observations"].items()}
            h = pol.init_hidden()
            h = tuple(x.to(d) for x in h) if isinstance(h, tuple) else h.to(d)
            logits, _, _ = pol(**obs, hidden=h)
            for k in HEADS:
                lg[k].append(logits[k][0].double().cpu())
                acts[k].append(r["actions"][k])
                masks[k].append(r["masks"][k])
    cat = [{k: torch.cat(v[k]) for k in HEADS} for v in (lg, acts, masks)]
    nll = float(BO.nll(*cat)[0])
    return nll, BO.accuracy(*cat)[0]


# Measured on an H100 with these settings (32 training rollouts of 64 steps, learning rate 3e-4, 60 steps): the LSTM-128
# student's held-out NLL fell from 5.865 to 2.822 and its token accuracy rose from 0.000 to 0.223.  The bars ask for about
# half of each gain.
DEMO_SHARPEN, DEMO_BIAS = 2.0, 3.0
BC_STEPS = 60
NLL_DROP = 1.5
ACC_GAIN = 0.1


def test_a_student_learns_the_demonstrators_actions(tmp_path):
    """Demonstrations of a seeded GRU-256 (demonstration_rollout) train an LSTM-128 student with BC: after BC_STEPS steps
    its NLL on held-out demonstrations is lower by NLL_DROP and its token accuracy higher by ACC_GAIN."""
    demo = _demonstrator()
    train = [demonstration_rollout(demo, 64, 900 + i, game_id=i) for i in range(32)]
    held = [demonstration_rollout(demo, 64, 950 + i, game_id=100 + i) for i in range(4)]
    opt = JR.make_optimizer(tmp_path, mask_padding=True, objective="bc")
    opt.learning_rate, opt.entropy_coef = 3e-4, 0.0
    batch = opt.batch_from_rollouts(copy.deepcopy(train))
    nll0, acc0 = _held_out_metrics(opt.policy_base, held)
    train_nll = []
    for _ in range(BC_STEPS):
        opt.train(batch)
        train_nll.append(opt.last_bc_stats["nll"])
    nll1, acc1 = _held_out_metrics(opt.policy_base, held)
    print("\nheld-out NLL %.4f -> %.4f, accuracy %.4f -> %.4f; training NLL %.4f -> %.4f"
          % (nll0, nll1, acc0, acc1, train_nll[0], train_nll[-1]))
    assert nll1 < nll0 - NLL_DROP and acc1 > acc0 + ACC_GAIN


def test_demonstration_rollout_is_a_valid_seeded_demonstration():
    from dotaclient_b200.optimizer import check_demonstrations
    demo = _demonstrator()
    a, b = demonstration_rollout(demo, 48, 3), demonstration_rollout(demo, 48, 3)
    check_demonstrations([a])
    assert all(torch.equal(a["actions"][k], b["actions"][k]) and torch.equal(a["masks"][k], b["masks"][k]) for k in HEADS)
    plain = make_rollout(48, 3)
    assert all(torch.equal(a["observations"][k], plain["observations"][k]) for k in plain["observations"])
    kinds = a["actions"]["enum"].int().argmax(dim=1)
    assert len(set(kinds.tolist())) >= 2


# ------------------------------------------------------------------------------------------------ the optimizer
def _snapshot(opt):
    return (opt.flat.param.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.adam_steps.clone())


def test_replayed_steps_equal_eager_steps(tmp_path):
    """mask_padding + pack_sequences, 2 minibatches, 3 epochs, both refreshes: the epochs replayed from captured graphs
    equal the eager ones bit for bit (losses, statistics, parameters, Adam state)."""
    kw = dict(mask_padding=True, pack_sequences=True, num_minibatches=2, recompute_advantages=True,
              recompute_states=True, epochs=3, min_seq=4, objective="bc")
    a = JR.make_optimizer(tmp_path, **kw)
    b = JR.make_optimizer(tmp_path, **kw)
    b.use_cuda_graph = False
    for o in (a, b):
        o.learning_rate = 1e-3
    rollouts = PK.ragged_rollouts(a.policy_base, 9, False, False)
    ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    for rep in range(2):                             # the second pass replays every minibatch shape
        ra, rb = a.train_epochs(ba), b.train_epochs(bb)
        assert [dict(s) for s in ra[3]] == [dict(s) for s in rb[3]], rep
        assert [{k: float(v) for k, v in x.items()} for x in ra[0]] == [{k: float(v) for k, v in x.items()} for x in rb[0]]
        assert all(torch.equal(x, y) for x, y in zip(_snapshot(a), _snapshot(b))), rep
        assert a.last_bc_stats == b.last_bc_stats and a.last_bc_stats["nll"] > 0
        assert all("approx_kl" not in s and "bc/accuracy" in s for s in ra[3])
    assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"


def test_published_model_is_the_reference_network_and_a_teacher(tmp_path):
    """After BC steps the published model loads strictly into the reference's Policy, and a 'ppo' optimizer of another
    architecture takes it as its teacher."""
    from dotaclient_b200.optimizer import DotaOptimizer
    from oracle.ref_policy import RefPolicy
    log_dir = tmp_path / "run"
    opt = DotaOptimizer(rmq_host="bc", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=1, seq_len=16,
                        learning_rate=1e-3, checkpoint=True, pretrained_model=None, mq_prefetch_count=1,
                        log_dir=str(log_dir), entropy_coef=5e-4, vf_coef=0.5, run_local=True, objective="bc")
    batch = opt.batch_from_rollouts([make_rollout(L, 60 + i, game_id=i) for i, L in enumerate((40, 23, 57))])
    for _ in range(3):
        opt.train(batch)
    opt.upload_model(2)
    path = str(log_dir / "model_000000002.pt")
    published = torch.load(path)
    ref = RefPolicy(256, "gru")
    ref.load_state_dict(published, strict=True)
    assert all(torch.equal(published[k], v.cpu()) for k, v in opt.policy_base.state_dict().items())
    student = JR.make_optimizer(tmp_path, mask_padding=True, teacher_model=path)
    b = student.batch_from_rollouts([make_rollout(40, 70)])
    student.train(b)
    assert student.last_ppo_stats["teacher/kl"] > 0


def test_prep_refuses_a_malformed_demonstration(tmp_path):
    opt = JR.make_optimizer(tmp_path, objective="bc")
    bad = make_rollout(30, 3, game_id=5)
    t = int(torch.nonzero(bad["actions"]["enum"][:, 0])[0])
    bad["actions"]["x"][t, 4] = True
    bad["masks"]["x"][t, 4] = True
    with pytest.raises(ValueError, match="game_id=5 .*step %d, head 'x'" % t):
        opt.batch_from_rollouts([bad])


def test_two_ranks_gloo_keep_identical_weights(tmp_path):
    import bc_multi_rank as BM
    a, b = BM.run(tmp_path)
    assert torch.equal(a["param"], b["param"]) and torch.equal(a["steps"], b["steps"])
    assert a["nll"] != b["nll"] and min(a["nll"] + b["nll"]) > 0      # different demonstrations, rank-local NLLs
