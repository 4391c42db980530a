"""GPU tests of kickstarting (``DotaOptimizer(teacher_model=...)``): ``dc_ppo_loss_fwd_bwd_teacher`` against the float64
oracle (``teacher_oracle.py``) in both ratio modes, with and without the KL penalty's rows; lambda = 0 against the entry
point the call would otherwise be, bit for bit; prep's teacher rows against a float64 forward of the reference network;
a teacher equal to the student's initial weights; the term doing its job; graph replay with every option it combines with
and the anneal retiring the teacher; checkpoint and resume; and two ranks over gloo.

Tolerances are the KL control suite's (``test_gpu_kl``): fp32 against float64, rtol 1e-4 on the losses and statistics and
2e-4 on dlogits."""
import copy
import os
import pickle
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kl_oracle as KO  # noqa: E402
import teacher_oracle as TO  # noqa: E402
import test_gpu_joint_ratio as JR  # noqa: E402
import test_gpu_packing as PK  # noqa: E402
import test_gpu_parity as P  # noqa: E402
from dotaclient_b200.synthetic import make_rollout, split_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS = P.HEADS
E_CLIP = JR.E_CLIP
BETA, LAMBDA = 0.7, 1.3
N_C2 = 131072


def _rows(logits, masks, seed, scale):
    """A policy's rows near the current one: the masked log-softmax of perturbed logits, in fp32."""
    g = torch.Generator().manual_seed(seed)
    moved = {k: v.double() + scale * torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in logits.items()}
    return KO.masked_log_rows(moved, masks).float()


def _run(inputs, old_rows, teacher_rows, joint, beta, lam):
    """One loss call: ``_teacher`` when teacher_rows is given, else ``_kl`` (old_rows) or ``_masked`` / ``_joint``."""
    from dotaclient_b200 import ops
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    d = P.dev()
    hp = ops.hparam_block(d, e_clip=E_CLIP, entropy_coef=5e-4, vf_coef=0.5, kl_coef=beta)
    kl_out = torch.full((2,), -1.0, device=d) if old_rows is not None else None
    kw = {}
    if teacher_rows is not None:
        kw = dict(teacher_log_probs=teacher_rows.to(d), teacher_coef=torch.tensor([lam], dtype=torch.float64, device=d))
    res = ops.ppo_loss_fwd_bwd([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                               [actions[k].to(d) for k in HEADS], old.to(d), adv.to(d), ret.to(d), values.to(d),
                               None, None, None, hparams=hp, old_value=ov.to(d),
                               valid=None if valid is None else valid.to(d), joint=joint,
                               old_log_probs=None if old_rows is None else old_rows.to(d), kl_out=kl_out, **kw)
    return res, kl_out


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("joint", [False, True])
@pytest.mark.parametrize("with_valid", [False, True])
@pytest.mark.parametrize("with_kl", [False, True])
def test_teacher_kernel_vs_oracle(joint, with_valid, with_kl):
    """Loss, statistics, teacher_stats, kl_out, dlogits and dvalue of dc_ppo_loss_fwd_bwd_teacher (lambda > 0) at C2's
    131,072 tokens against the float64 oracle."""
    n = N_C2
    inputs = JR._inputs(n, 17, None, None, with_valid)
    logits, masks, actions, old, values, adv, ret, ov, valid = inputs
    old_rows = _rows(logits, masks, 3, 0.25) if with_kl else None
    t_rows = _rows(logits, masks, 5, 1.0)                       # a teacher further away than the prep-time policy
    lg = {k: v.double().requires_grad_(True) for k, v in logits.items()}
    vg = values.double().requires_grad_(True)
    loss, p_loss, e_loss, v_loss, ents, kl_t = TO.teacher_ppo_loss(
        lg, vg, actions, masks, old.double(), None if old_rows is None else old_rows.double(), t_rows.double(),
        adv.double(), ret.double(), 5e-4, 0.5, E_CLIP, BETA, LAMBDA, joint=joint, valid=valid, old_values=ov.double())
    loss.backward()
    _, t_sum, t_a, per_head = TO.teacher_kl({k: v.double() for k, v in logits.items()}, actions, masks, t_rows.double(),
                                            valid)
    (out, n_act, dlogits, dvalue, stats, tst), kl_out = _run(inputs, old_rows, t_rows, joint, BETA, LAMBDA)
    out, st, tst = out.cpu().numpy(), stats.cpu(), tst.cpu()
    for i, want in enumerate((loss, p_loss, e_loss, v_loss)):
        np.testing.assert_allclose(out[i], float(want.detach()), rtol=1e-4, atol=1e-6, err_msg=str(i))
    kl_t = float(kl_t.detach())
    assert kl_t > 0.05
    np.testing.assert_allclose(float(tst[0]), kl_t, rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(tst[1:6].numpy(), [per_head[k] for k in HEADS], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(float(tst[6]), LAMBDA * kl_t, rtol=1e-4, atol=1e-7)
    if with_kl:
        _, kl_sum, t_a_kl, per_kl = KO.exact_kl({k: v.double() for k, v in logits.items()}, actions, masks,
                                                old_rows.double(), valid)
        assert t_a_kl == t_a and float(kl_out[1]) == t_a
        np.testing.assert_allclose(float(kl_out[0]), float(kl_sum), rtol=1e-4)
        np.testing.assert_allclose(st[17:22].numpy(), [per_kl[k] for k in HEADS], rtol=1e-4, atol=1e-7)
    else:
        assert bool((st[16:] == 0).all())
    for h, k in enumerate(HEADS):
        g_ref = lg[k].grad.float() if lg[k].grad is not None else torch.zeros_like(logits[k])
        torch.testing.assert_close(dlogits[h].cpu(), g_ref, rtol=2e-4, atol=1e-8)
        if valid is not None:
            assert bool((dlogits[h].cpu()[~valid] == 0).all()), k
    torch.testing.assert_close(dvalue.cpu(), vg.grad.float(), rtol=1e-4, atol=1e-9)


@pytest.mark.parametrize("joint", [False, True])
@pytest.mark.parametrize("with_valid", [False, True])
@pytest.mark.parametrize("with_kl", [False, True])
def test_lambda_zero_is_the_other_entry_point_bitwise(joint, with_valid, with_kl):
    """lambda = 0: loss, n_actions, dlogits, dvalue, stats and kl_out equal _kl (old rows) or _masked / _joint (none) bit
    for bit, and teacher_stats still reports the KL."""
    inputs = JR._inputs(N_C2, 29, None, None, with_valid)
    old_rows = _rows(inputs[0], inputs[1], 31, 0.25) if with_kl else None
    t_rows = _rows(inputs[0], inputs[1], 37, 1.0)
    (a, kl_a), (b, kl_b) = _run(inputs, old_rows, t_rows, joint, BETA, 0.0), _run(inputs, old_rows, None, joint, BETA, 0.0)
    out_a, n_a, dl_a, dv_a, st_a, ts = a
    out_b, n_b, dl_b, dv_b, st_b = b
    assert torch.equal(out_a, out_b) and torch.equal(n_a, n_b) and torch.equal(dv_a, dv_b) and torch.equal(st_a, st_b)
    assert all(torch.equal(x, y) for x, y in zip(dl_a, dl_b))
    if with_kl:
        assert torch.equal(kl_a, kl_b)
    assert float(ts[0]) > 0 and float(ts[6]) == 0.0


# ------------------------------------------------------------------------------------------------ experience prep
def _save(pol, path):
    torch.save({k: v.detach().cpu() for k, v in pol.state_dict().items()}, path)
    return path


def _reference_teacher(tmp_path):
    """The reference's GRU-256 at its seeded initialisation, saved as a published model."""
    from dotaclient_b200.policy import Policy
    torch.manual_seed(7)
    return _save(Policy(), str(tmp_path / "teacher_gru256.pt"))


def _rollouts(seed, carried):
    """Four rollouts; with ``carried`` the first is cut from a longer game and carries an 'initial_hidden' of an LSTM-128
    actor."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, L in enumerate((40, 23, 57, 16)):
        cut = carried and i == 0
        r = make_rollout(L + (1 if cut else 0), 100 * seed + i, game_id=i)
        if cut:
            r = split_rollout(r, [L])[0]
            h = 0.5 * torch.randn(1, 1, 128, generator=g)
            r["initial_hidden"] = (h, 0.5 * torch.randn(h.shape, generator=g))
        out.append(r)
    return out


def test_prep_teacher_rows_vs_float64_reference(tmp_path):
    """A GRU-256 teacher (the reference's initialisation) for an LSTM-128 student: prep's teacher rows of every rollout
    against RefPolicy in float64 loaded with the teacher's weights, run over the rollout from the zero state -- also for the
    cut rollout, whose 'initial_hidden' is the student's."""
    from oracle.ref_policy import RefPolicy
    path = _reference_teacher(tmp_path)
    opt = JR.make_optimizer(tmp_path, mask_padding=True, teacher_model=path)
    rollouts = _rollouts(3, True)
    p = opt._prepare_rollouts(copy.deepcopy(rollouts))
    rows = p["teacher_log_probs"]
    assert rows.shape == (p["Lmax"], len(rollouts), 65)
    ref = RefPolicy(256, "gru")
    ref.load_state_dict(torch.load(path))
    ref = ref.double()
    worst = 0.0
    for i, d in enumerate(rollouts):
        L = p["Ls"][i]
        obs = {k: torch.as_tensor(v[:L]).double().unsqueeze(0) for k, v in d["observations"].items()}
        with torch.no_grad():
            lg, _, _ = ref(**obs, hidden=torch.zeros(1, 1, 256, dtype=torch.float64))
        masks = {k: torch.as_tensor(d["masks"][k][:L]).bool() for k in HEADS}
        want = TO.masked_log_rows({k: lg[k][0] for k in HEADS}, masks)
        got = rows[:L, i].cpu().double()
        legal = torch.cat([masks[k] for k in HEADS], dim=1)
        assert bool((got[~legal] == 0).all())
        err = float((got - want)[legal].abs().max())
        worst = max(worst, err)
        assert err < 1e-4, (i, err)
    print("\nteacher rows vs float64: max abs error %.3g" % worst)
    batch = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    assert batch.teacher_log_probs.shape == batch.old_logp.shape[:2] + (65,)
    for c in range(3):                               # rollout 0 (40 steps) fills columns 0..2 of the unpacked batch
        assert torch.equal(batch.teacher_log_probs[:, c], rows[16 * c:16 * (c + 1), 0]), c


def test_teacher_equal_to_the_student_gives_the_old_rows(tmp_path):
    """The teacher is the student's own initial weights and prep also stores the KL penalty's rows: the same kernels on the
    same inputs, so teacher_log_probs equals old_log_probs bit for bit (chunked, packed and as Sequences)."""
    from dotaclient_b200.policy import Policy
    torch.manual_seed(7)
    path = _save(Policy(hidden_size=128, cell="lstm"), str(tmp_path / "self.pt"))
    kw = dict(mask_padding=True, kl_coef=0.2, teacher_model=path)
    a = JR.make_optimizer(tmp_path, **kw)
    b = JR.make_optimizer(tmp_path, pack_sequences=True, **kw)
    sd_a, sd_t = a.policy_base.state_dict(), a.teacher.state_dict()
    assert all(torch.equal(sd_a[k], sd_t[k]) for k in sd_a)
    rollouts = _rollouts(5, False)
    chunked = a.batch_from_rollouts(copy.deepcopy(rollouts))
    assert torch.equal(chunked.teacher_log_probs, chunked.old_log_probs)
    packed = b.batch_from_rollouts(copy.deepcopy(rollouts))
    assert torch.equal(packed.teacher_log_probs, packed.old_log_probs)
    seqs = [s for r in a.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in r]
    assert all(torch.equal(s.teacher_log_probs, s.old_log_probs) for s in seqs)
    a.train(chunked)                                 # the teacher is the prep-time policy: KL_T is the KL, about 0
    st = a.last_ppo_stats
    assert st["teacher/kl"] == st["kl"] and -1e-6 <= st["teacher/kl"] < 1e-4


# ------------------------------------------------------------------------------------------------ the optimizer
# The first run (H100): teacher/kl 0.0101 before the first update, 0.0013 after the twelfth (0.13x; the first update at
# this learning rate overshoots to 0.14 and the next ones bring it down).  The bound leaves a factor of 4 of room.
TEACHER_FACTOR = 0.5


def test_the_term_pulls_the_student_toward_the_teacher(tmp_path):
    """A large lambda and a GRU-256 teacher for an LSTM-128 student: a few steps on synthetic rollouts cut the KL to the
    teacher by at least TEACHER_FACTOR."""
    from dotaclient_b200.policy import Policy
    torch.manual_seed(11)
    path = _save(Policy(hidden_size=256, cell="gru"), str(tmp_path / "t.pt"))
    opt = JR.make_optimizer(tmp_path, mask_padding=True, teacher_model=path, teacher_coef=20.0)
    opt.learning_rate = 3e-3
    batch = opt.batch_from_rollouts(copy.deepcopy(_rollouts(7, False)))
    kls = []
    for _ in range(12):
        opt.train(batch)
        kls.append(opt.last_ppo_stats["teacher/kl"])
        assert opt.last_ppo_stats["loss/teacher"] == pytest.approx(20.0 * kls[-1], rel=1e-5)
    print("\nteacher/kl over 12 steps: %s (last / first %.3f)" % (["%.4f" % k for k in kls], kls[-1] / kls[0]))
    assert kls[0] > 0.005 and kls[-1] < TEACHER_FACTOR * kls[0]


def _snapshot(opt):
    return (opt.flat.param.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.adam_steps.clone())


def test_every_option_replays_as_it_runs_eagerly_and_the_anneal_retires_the_teacher(tmp_path):
    """Joint ratio, the KL penalty, mask_padding + pack_sequences, 2 minibatches and both refreshes with a teacher: the
    epochs replayed from captured graphs equal the eager ones bit for bit (losses, statistics, parameters, Adam state).
    Then run_iteration anneals lambda to 0 over two iterations: the third retires the teacher and its batch has no rows."""
    from dotaclient_b200.optimizer import MessageQueue
    from dotaclient_b200.policy import Policy
    torch.manual_seed(13)
    path = _save(Policy(hidden_size=256, cell="gru", num_layers=2), str(tmp_path / "t.pt"))
    port = uuid.uuid4().int % 100000
    kw = dict(mask_padding=True, pack_sequences=True, policy_ratio="joint", kl_coef=0.3, num_minibatches=2,
              recompute_advantages=True, recompute_states=True, epochs=3, min_seq=4, teacher_model=path,
              teacher_coef=2.0, teacher_anneal_iterations=2)
    a = JR.make_optimizer(tmp_path, port=port, **kw)
    b = JR.make_optimizer(tmp_path, **kw)
    b.use_cuda_graph = False
    for o in (a, b):
        o.learning_rate = 1e-3
    rollouts = PK.ragged_rollouts(a.policy_base, 9, False, True)
    ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    assert ba.teacher_log_probs is not None and torch.equal(ba.teacher_log_probs, bb.teacher_log_probs)
    for rep in range(2):                             # the second pass replays every minibatch shape
        ra, rb = a.train_epochs(ba), b.train_epochs(bb)
        assert [dict(s) for s in ra[3]] == [dict(s) for s in rb[3]], rep
        assert [{k: float(v) for k, v in x.items()} for x in ra[0]] == [{k: float(v) for k, v in x.items()} for x in rb[0]]
        assert all(torch.equal(x, y) for x, y in zip(_snapshot(a), _snapshot(b))), rep
        assert all(s["loss/teacher"] > 0 for s in ra[3])
    assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"
    # the anneal: lambda = 2 (n = 0), 1 (n = 1), then 0 -> retired
    actor = MessageQueue(host="joint", port=port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for it in range(3):
        for i, L in enumerate((40, 23, 57)):
            actor.publish_experience(pickle.dumps(make_rollout(L, 970 + 10 * it + i, game_id=i, weight_version=1)))
    seen = []
    a.batch_from_rollouts, prepare = (lambda datas: seen.append(prepare(datas)) or seen[-1]), a.batch_from_rollouts
    for it, lam in ((1, 2.0), (2, 1.0), (3, 0.0)):
        m = a.run_iteration(it)
        assert m["teacher/coef"] == lam and a.teacher_iterations == min(it, 2)
        if lam > 0:
            assert seen[-1].teacher_log_probs is not None and m["teacher/kl"] > 0 and m["loss/teacher"] > 0
        else:
            assert seen[-1].teacher_log_probs is None and "teacher/kl" not in m and a.teacher is None


def test_checkpoint_and_resume_restore_the_schedule(tmp_path):
    """upload_model writes the teacher's side file and prunes it like the others; a resumed run restores n and lambda.  The
    published model has exactly the keys and shapes of a teacher-less run of the same architecture, and no teacher."""
    from dotaclient_b200.optimizer import DotaOptimizer
    from dotaclient_b200.policy import Policy
    torch.manual_seed(17)
    path = _save(Policy(hidden_size=256, cell="gru"), str(tmp_path / "t.pt"))
    log_dir = tmp_path / "run"

    def make(**kw):
        return DotaOptimizer(rmq_host="teacher", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=1,
                             seq_len=16, learning_rate=5e-5, checkpoint=True, pretrained_model=None, mq_prefetch_count=1,
                             log_dir=str(log_dir), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=128,
                             cell="lstm", **kw)
    a = make(teacher_model=path, teacher_coef=3.0, teacher_anneal_iterations=10)
    for version, n in ((5, 4), (6, 5), (7, 6), (8, 7)):
        a.teacher_iterations, a.teacher_coef = n, 3.0 * (1 - n / 10)
        a.upload_model(version)
    side = sorted(f for f in os.listdir(str(log_dir)) if f.startswith("teacher_"))
    assert side == ["teacher_%09d.state" % v for v in (6, 7, 8)], side
    st = torch.load(str(log_dir / "teacher_000000008.state"))
    assert st == {"iterations": 7, "teacher_coef": 3.0 * (1 - 7 / 10), "teacher_model": path}
    published = torch.load(str(log_dir / "model_000000008.pt"))
    plain_dir = tmp_path / "plain"
    os.makedirs(str(plain_dir))
    plain = JR.make_optimizer(plain_dir)
    want = plain.policy_base.state_dict()
    assert list(published) == list(want) and all(published[k].shape == want[k].shape for k in want)
    assert all(torch.equal(published[k], v.cpu()) for k, v in a.policy_base.state_dict().items())
    b = make(teacher_model=path, teacher_coef=3.0, teacher_anneal_iterations=10)
    assert b.iteration_start == 9 and b.teacher_iterations == 7 and b.teacher_coef == 3.0 * (1 - 7 / 10)
    b.teacher_anneal()
    assert b.teacher_coef == pytest.approx(0.9, rel=1e-15) and b.teacher is not None
    c = make()                                       # a run without a teacher ignores the file
    assert c.teacher_model is None and c.teacher_iterations == 0


def test_constructor_refuses_a_bad_teacher_file(tmp_path):
    torch.save(torch.nn.Linear(3, 3).state_dict(), str(tmp_path / "linear.pt"))
    with pytest.raises(ValueError, match="no such file"):
        JR.make_optimizer(tmp_path, teacher_model=str(tmp_path / "missing.pt"))
    with pytest.raises(ValueError, match="not a Policy state_dict"):
        JR.make_optimizer(tmp_path, teacher_model=str(tmp_path / "linear.pt"))


def test_train_refuses_a_batch_without_rows(tmp_path):
    from dotaclient_b200.policy import Policy
    path = _save(Policy(hidden_size=64), str(tmp_path / "t.pt"))
    a = JR.make_optimizer(tmp_path, mask_padding=True, teacher_model=path)
    plain = JR.make_optimizer(tmp_path, mask_padding=True)
    batch = plain.batch_from_rollouts(copy.deepcopy(_rollouts(2, False)))
    with pytest.raises(ValueError, match="teacher_log_probs"):
        a.train(batch)
    a.teacher_coef = 0.0                             # lambda = 0: the batch trains without the term
    a.train(batch)
    assert "teacher/kl" not in a.last_ppo_stats


def test_two_ranks_gloo_keep_identical_weights(tmp_path):
    import teacher_multi_rank as TM
    a, b = TM.run(tmp_path)
    assert torch.equal(a["param"], b["param"]) and torch.equal(a["steps"], b["steps"])
    assert a["coef"] == b["coef"] and a["n"] == b["n"] == 2
    assert a["kl"] != b["kl"] and min(a["kl"] + b["kl"]) > 0      # different batches, rank-local KLs
