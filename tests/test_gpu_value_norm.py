"""GPU tests of ``value_norm`` (PopArt): the three new kernels against numpy float64 at 131,072 tokens, the value-normalised
loss of all three entry points against a float64 restatement and bitwise against the plain loss at slot 7 = 0 and at
(0, 1), preservation of the critic's output across an update, whole iterations against the CPU oracle
(``value_norm_oracle.py``), graph replay, checkpoints and resume, and the feature being off by default."""
import copy
import os
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_parity as P  # noqa: E402
import test_gpu_vtrace as V  # noqa: E402
import value_norm_oracle as VO  # noqa: E402
from stacked_oracle import StackedRefPolicy  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS, SIZES = P.HEADS, P.SIZES
N_C2 = 131072


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=16, epochs=1, min_seq=1, port=None, checkpoint=False,
                   pretrained_model=None, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="value_norm", rmq_port=port if port is not None else uuid.uuid4().int % 100000,
                         epochs=epochs, min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=5e-5,
                         checkpoint=checkpoint, pretrained_model=pretrained_model, mq_prefetch_count=1, log_dir=str(tmp_path),
                         entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=hidden_size, cell=cell, **kw)


def _scaled(rollouts, scale=25.0, offset=4.0):
    """Rewards rescaled and offset, so that the value statistics land far from (0, 1)."""
    for r in rollouts:
        r["rewards"] = (np.asarray(r["rewards"], np.float32) * scale + offset).astype(np.float32)
    return rollouts


def _hidden(pol):
    h = pol.init_hidden()
    return tuple(t.to(P.dev()) for t in h) if isinstance(h, tuple) else h.to(P.dev())


def _rollouts(seed, lengths=(40, 23, 48, 7, 33), scale=25.0, offset=4.0, **kw):
    return _scaled([make_rollout(L, 1300 + 10 * seed + i, game_id=i, **kw) for i, L in enumerate(lengths)], scale, offset)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("masked", [False, True])
def test_stats_kernel_vs_numpy_and_bitwise_repeatable(masked):
    from dotaclient_b200 import ops
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(N_C2, generator=g) * 30.0 + 12.0).float()
    valid = torch.rand(N_C2, generator=g) < 0.8 if masked else None
    d = P.dev()
    a = ops.value_norm_stats(x.to(d), None if valid is None else valid.to(d))
    b = ops.value_norm_stats(x.to(d), None if valid is None else valid.to(d))
    assert torch.equal(a, b)
    n, s1, s2 = VO.batch_sums(x.numpy(), None if valid is None else valid.numpy())
    got = a.cpu().tolist()
    assert got[0] == n
    assert got[1] == pytest.approx(s1, rel=1e-12) and got[2] == pytest.approx(s2, rel=1e-12)
    empty = ops.value_norm_stats(x[:0].to(d))
    assert empty.cpu().tolist() == [0.0, 0.0, 0.0]


def test_denorm_kernel_is_numpys_fp64_then_round_on_a_packed_column():
    from dotaclient_b200 import ops
    g = torch.Generator().manual_seed(12)
    packed = torch.randn(N_C2, ops.PACK_WIDTH, generator=g).to(P.dev())
    col = packed[:, ops.PACK_COLS["value"][0]:ops.PACK_COLS["value"][1]]           # pitch 128
    for mu, sigma in ((0.0, 1.0), (13.7, 41.3), (-0.3, 0.01)):
        got = ops.value_denorm(col, mu, sigma).cpu().numpy()
        want = VO.denorm(col.cpu().numpy(), mu, sigma)
        np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(ops.value_denorm(col, 0.0, 1.0).cpu().numpy(), col.cpu().numpy())


def test_head_rescale_kernel_vs_numpy():
    from dotaclient_b200 import ops
    w = torch.randn(1, 256, generator=torch.Generator().manual_seed(13)) * 0.05
    b = torch.tensor([0.7])
    for old, new in (((0.0, 1.0), (6.0, 30.0)), ((6.0, 30.0), (5.5, 29.0)), ((-1.0, 0.01), (2.0, 3.0))):
        wd, bd = w.to(P.dev()), b.to(P.dev())
        ops.value_head_rescale(wd, bd, old, new)
        ww, bb = VO.rescale(w.numpy(), b.numpy(), old, new)
        np.testing.assert_array_equal(wd.cpu().numpy(), ww)
        np.testing.assert_array_equal(bd.cpu().numpy(), bb)


# ------------------------------------------------------------------------------------------------ the loss
def _loss_inputs(n, seed):
    import test_padding_host as H
    logits, values, actions, masks, old, adv, ret, valid = H._case(n, seed, invalid_actions=True)
    g = torch.Generator().manual_seed(seed)
    ret = ret * 40.0 + 9.0                                       # raw targets, far from the normalised head's units
    ov = ret + 15.0 * torch.randn(n, generator=g)                # raw old values
    return logits, values, actions, masks, old, adv, ret, ov, valid


def _call(inp, entry, clip, norm, masked=True):
    from dotaclient_b200 import ops
    logits, values, actions, masks, old, adv, ret, ov, valid = inp
    d = P.dev()
    hp = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5, value_clip=clip, value_norm=norm)
    v = valid.to(d) if (masked and entry != "dev") else None
    return ops.ppo_loss_fwd_bwd([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                                [actions[k].to(d) for k in HEADS], old.to(d), adv.to(d), ret.to(d), values.to(d),
                                0.0, 0.0, 0.0, hparams=hp, old_value=ov.to(d), valid=v, joint=entry == "joint")


def _same(a, b):
    out_a, na, dl_a, dv_a, st_a = a
    out_b, nb, dl_b, dv_b, st_b = b
    assert torch.equal(out_a, out_b) and torch.equal(na, nb) and torch.equal(dv_a, dv_b)
    assert all(torch.equal(x, y) for x, y in zip(dl_a, dl_b))
    assert torch.equal(st_a.nan_to_num(7.0), st_b.nan_to_num(7.0))


@pytest.mark.parametrize("entry", ["dev", "masked", "joint"])
@pytest.mark.parametrize("clip", [None, 0.2])
def test_normalised_loss_vs_float64(entry, clip):
    """Value loss, dvalue, the clipped branch and the explained variance against float64 on normalised targets; the policy
    and entropy terms are the plain loss's, bit for bit."""
    mu, sigma = 31.0, 17.5
    inp = _loss_inputs(N_C2, 21)
    logits, values, actions, masks, old, adv, ret, ov, valid = inp
    got = _call(inp, entry, clip, (mu, sigma))
    plain = _call(inp, entry, clip, None)
    out, dv, st = got[0].cpu().double(), got[3].cpu().double(), got[4].cpu().double()
    v = valid.bool() if entry != "dev" else torch.ones(N_C2, dtype=torch.bool)
    r_n = torch.from_numpy(VO.normalise(ret.numpy(), mu, sigma)).double()
    o_n = torch.from_numpy(VO.normalise(ov.numpy(), mu, sigma)).double()
    val = values.double().clone().requires_grad_(True)
    if clip:
        vc = o_n + torch.clamp(val - o_n, -clip, clip)
        per = torch.maximum((val - r_n) ** 2, (vc - r_n) ** 2)
    else:
        per = (val - r_n) ** 2
    v_loss = 0.5 * 0.5 * per[v].sum() / v.sum()
    v_loss.backward()
    np.testing.assert_allclose(float(out[3]), float(v_loss), rtol=1e-5)
    np.testing.assert_allclose(dv.numpy(), val.grad.numpy(), rtol=1e-4, atol=1e-9)
    rv, dd = r_n[v], (r_n - values.double())[v]
    ev = 1.0 - float(dd.var(unbiased=False)) / float(rv.var(unbiased=False))
    np.testing.assert_allclose(float(st[12]), ev, rtol=1e-4, atol=1e-5)
    # the policy and entropy terms do not see the value normalisation
    for i in list(range(1, 3)) + list(range(4, 16)):
        assert got[0].cpu()[i] == plain[0].cpu()[i], i
    assert all(torch.equal(a, b) for a, b in zip(got[2], plain[2]))
    assert not torch.equal(got[3], plain[3])


@pytest.mark.parametrize("entry", ["dev", "masked", "joint"])
@pytest.mark.parametrize("clip", [None, 0.2])
def test_slot7_zero_and_identity_are_the_plain_loss_bitwise(entry, clip):
    inp = _loss_inputs(N_C2, 22)
    plain = _call(inp, entry, clip, None)
    _same(plain, _call(inp, entry, clip, (0.0, 1.0)))
    _same(plain, _call(inp, entry, clip, (123.0, 0.0)))       # slot 7 = 0: off whatever slot 6 holds


# ------------------------------------------------------------------------------------------------ optimizer
def test_off_by_default_leaves_slots_6_and_7_zero(tmp_path):
    from dotaclient_b200 import _lib
    opt = make_optimizer(tmp_path)
    batch = opt.batch_from_rollouts(_rollouts(1))
    opt.train(batch)
    hp = opt._hparams_dev.cpu()
    assert hp[_lib.HP_VALUE_NORM_MEAN] == 0.0 and hp[_lib.HP_VALUE_NORM_STD] == 0.0
    assert opt.value_norm_stats is None


def test_update_preserves_the_critic_and_reaches_the_hparams(tmp_path):
    """Value before the update == sigma_new v' + mu_new after it, within rtol 1e-6; the next step uploads (mu, sigma)."""
    from dotaclient_b200 import _lib
    opt = make_optimizer(tmp_path, value_norm=True, value_norm_decay=0.9)
    probe = _rollouts(2)[0]
    obs = {k: torch.as_tensor(probe["observations"][k][:16]).unsqueeze(1).to(P.dev()) for k in opt.policy_base.INPUT_KEYS}

    def critic():
        with torch.no_grad():
            _, v, _ = opt.policy_base.forward_time_major(obs, _hidden(opt.policy_base))
        return v.double().cpu().reshape(-1)
    for it in range(3):
        mu0, s0 = opt._value_norm_moments()
        before = s0 * critic() + mu0
        batch = opt.batch_from_rollouts(_rollouts(30 + it, scale=25.0 * (1 + it), offset=4.0 - 3 * it))
        mu1, s1 = opt._value_norm_moments()
        after = s1 * critic() + mu1
        assert (mu1, s1) != (mu0, s0)
        np.testing.assert_allclose(after.numpy(), before.numpy(), rtol=1e-6, atol=1e-6 * s1)
        opt.train(batch)
        hp = opt._hparams_dev.cpu()
        assert (float(hp[_lib.HP_VALUE_NORM_MEAN]), float(hp[_lib.HP_VALUE_NORM_STD])) == (mu1, s1)
    st = opt.value_norm_stats
    assert abs(st["mean"]) > 10 and st["std"] > 10 and st["weight"] == pytest.approx(1 - 0.9 ** 3)


def _stats_of_batch(batch, valid):
    ret = batch.returns.cpu().numpy()
    return VO.batch_sums(ret, None if valid is None else valid.cpu().numpy())


@pytest.mark.parametrize("mask", [False, True])
def test_prep_updates_from_the_counting_tokens(mask, tmp_path):
    opt = make_optimizer(tmp_path, value_norm=True, value_norm_decay=0.0, mask_padding=mask)
    batch = opt.batch_from_rollouts(_rollouts(3))
    n, s1, s2 = _stats_of_batch(batch, batch.valid)
    assert n == (sum((40, 23, 48, 7, 33)) if mask else 12 * 16)
    mu, sigma = opt._value_norm_moments()
    assert mu == pytest.approx(s1 / n, rel=1e-12)
    assert sigma == pytest.approx(np.sqrt(s2 / n - (s1 / n) ** 2), rel=1e-9)


def test_packed_prep_has_the_statistics_of_the_unpacked_one(tmp_path):
    a = make_optimizer(tmp_path, value_norm=True, mask_padding=True)
    b = make_optimizer(tmp_path, value_norm=True, mask_padding=True, pack_sequences=True)
    rollouts = _rollouts(4)
    for it in range(2):
        ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
        if it == 0:                       # same weights, same prep: the same statistics and head, bit for bit
            assert a._value_norm == b._value_norm
            assert torch.equal(a.policy_base.affine_value.weight, b.policy_base.affine_value.weight)
        else:                             # after a packed and an unpacked step: equal up to summation order
            assert a._value_norm == pytest.approx(b._value_norm, rel=1e-5)
        assert bb.batch_size < ba.batch_size
        la, lb = a.train(ba)[0], b.train(bb)[0]
        assert np.isfinite(float(la["value_loss"])) and np.isfinite(float(lb["value_loss"]))


def test_cut_rollouts_read_the_critic_in_raw_units(tmp_path):
    """Identity statistics give exactly the plain prep; after an update the values and V(s_L) bootstraps of a prep with
    the feature match the plain optimizer's within the rescale's rounding."""
    a = make_optimizer(tmp_path, value_norm=True, mask_padding=True)
    b = make_optimizer(tmp_path, mask_padding=True)
    from dotaclient_b200.synthetic import split_rollout
    rollouts = _scaled(split_rollout(make_rollout(60, 1500, game_id=1), [25]) + [make_rollout(33, 1501, game_id=2)])
    assert not rollouts[0]["terminal"]
    pa, pb = a._prepare_rollouts(copy.deepcopy(rollouts)), b._prepare_rollouts(copy.deepcopy(rollouts))
    for k in ("values_lr", "adv_c", "ret_c", "bootstrap"):
        assert torch.equal(pa[k], pb[k]), k
    assert a.value_norm_stats["weight"] > 0
    pa, pb = a._prepare_rollouts(copy.deepcopy(rollouts)), b._prepare_rollouts(copy.deepcopy(rollouts))
    sigma = a.value_norm_stats["std"]
    for k in ("values_lr", "bootstrap", "ret_c"):
        torch.testing.assert_close(pa[k], pb[k], rtol=1e-5, atol=1e-5 * sigma)


CONFIGS = {
    "gae": dict(),
    "vtrace": dict(advantage_estimator="vtrace"),
    "gae_masked": dict(mask_padding=True),
    "vtrace_masked_clip": dict(advantage_estimator="vtrace", mask_padding=True, value_clip=0.2),
    "gae_clip": dict(value_clip=0.2),
}


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_iterations_vs_oracle(name, tmp_path):
    """Three iterations (prep + one step each) against the CPU oracle, at the step parity tests' tolerances: losses,
    mu and sigma, the value head and every parameter."""
    torch.set_num_threads(8)
    kw = CONFIGS[name]
    S, H, cell = 16, 128, "lstm"
    mine = make_optimizer(tmp_path, hidden_size=H, cell=cell, value_norm=True, value_norm_decay=0.9, **kw)
    torch.manual_seed(7)
    oracle = VO.ValueNormRefOptimizer(StackedRefPolicy(H, cell, 1), seq_len=S, decay=0.9,
                                      estimator=kw.get("advantage_estimator", "gae"),
                                      mask_padding=kw.get("mask_padding", False), value_clip=kw.get("value_clip"))
    for it in range(3):
        rollouts = _rollouts(10 + it)
        if kw.get("advantage_estimator") == "vtrace":
            rollouts = V._stale_behaviour(mine, rollouts, 20 + it)
        xs_m = [s for grp in mine.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in grp]
        xs_o = oracle.prepare(copy.deepcopy(rollouts))
        for a, b in zip(xs_m, xs_o):
            V._close(a.values.reshape(-1).cpu(), b.values.reshape(-1), 2e-4)
            V._close(a.returns.cpu(), b.returns, 2e-4)
        mu_m, s_m = mine._value_norm_moments()
        mu_o, s_o = oracle.stats
        assert mu_m == pytest.approx(mu_o, rel=1e-4) and s_m == pytest.approx(s_o, rel=1e-4), it
        assert abs(mu_m) > 5 and s_m > 5
        lm, em, gm = mine.train(xs_m)
        lo, eo, go = oracle.train(xs_o)
        for k in lo:
            np.testing.assert_allclose(float(lm[k]), float(lo[k]), rtol=2e-4, atol=2e-6, err_msg="%s it%d" % (k, it))
        np.testing.assert_allclose(float(gm["unclipped"]), float(go["unclipped"]), rtol=2e-3)
    for name_, p in oracle.policy_base.named_parameters():
        mp = dict(mine.policy_base.named_parameters())[name_].detach().cpu()
        # three Adam steps of lr 5e-5: a parameter can differ by at most a few steps' size where its gradient is ~0
        torch.testing.assert_close(mp, p.detach(), rtol=1e-4, atol=3e-4, msg=name_)
    hw = mine.policy_base.affine_value.weight.detach().cpu()
    torch.testing.assert_close(hw, oracle.policy_base.affine_value.weight.detach(), rtol=2e-3, atol=3e-4)


def test_minibatches_equal_index_select_batches(tmp_path):
    from dotaclient_b200.optimizer import minibatch_indices
    a = make_optimizer(tmp_path, epochs=2, min_seq=3, num_minibatches=2, value_norm=True)
    b = make_optimizer(tmp_path, epochs=2, min_seq=3, value_norm=True)
    rollouts = _rollouts(5)
    batch_a, batch_b = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    assert a._value_norm == b._value_norm
    rng = copy.deepcopy(a.minibatch_rng)
    la = a.train_epochs(batch_a)[0]
    lb = []
    for _ in range(2):
        for idx in minibatch_indices(batch_b.batch_size, 2, rng):
            mb = batch_b.map(lambda v: v.index_select(1, torch.as_tensor(idx, device=v.device)))
            lb.append(b.train(mb)[0])
    assert [[float(v) for v in x.values()] for x in la] == [[float(v) for v in x.values()] for x in lb]
    assert torch.equal(a.flat.param, b.flat.param)


def test_graph_replay_after_a_stats_update_equals_launch_by_launch(tmp_path):
    a = make_optimizer(tmp_path, value_norm=True)
    b = make_optimizer(tmp_path, value_norm=True)
    a.use_cuda_graph, b.use_cuda_graph = False, True
    rollouts = _rollouts(6, (32, 16, 48))
    for it in range(3):                    # same shape every iteration: b captures in it 0 and replays after each update
        ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
        assert a._value_norm == b._value_norm
        for _ in range(2):
            ra, rb = a.train(ba), b.train(bb)
            assert [float(v) for v in ra[0].values()] == [float(v) for v in rb[0].values()], it
    assert any(not isinstance(v, str) for v in b._graphs.values())
    assert torch.equal(a.flat.param, b.flat.param) and torch.equal(a.exp_avg, b.exp_avg)


def test_published_model_is_denormalised_and_resume_is_bit_identical(tmp_path):
    from dotaclient_b200.optimizer import DotaOptimizer
    from dotaclient_b200.policy import Policy
    d1 = tmp_path / "run"
    a = make_optimizer(d1, checkpoint=True, value_norm=True, value_norm_decay=0.8)
    rollouts = [_rollouts(7 + k, (32, 16, 48)) for k in range(3)]
    for k in range(2):
        a.train(a.batch_from_rollouts(copy.deepcopy(rollouts[k])))
    a.upload_model(version=2)
    names = sorted(os.listdir(d1))
    assert "model_000000002.pt" in names and "value_norm_000000002.state" in names
    # a plain Policy from the published weights gives the trainer's raw-scale values
    sd = torch.load(d1 / "model_000000002.pt", map_location="cpu")
    assert len(sd) == len(a.policy_base.state_dict())
    plain = Policy(hidden_size=128, cell="lstm")
    plain.load_state_dict(sd)
    plain.to(P.dev())
    r = rollouts[2][0]
    obs = {k: torch.as_tensor(r["observations"][k][:16]).unsqueeze(1).to(P.dev()) for k in Policy.INPUT_KEYS}
    with torch.no_grad():
        v_pub = plain.forward_time_major(obs, _hidden(plain))[1].double().cpu()
        v_norm = a.policy_base.forward_time_major(obs, _hidden(a.policy_base))[1].double().cpu()
    mu, sigma = a._value_norm_moments()
    torch.testing.assert_close(v_pub, sigma * v_norm + mu, rtol=1e-5, atol=1e-5 * sigma)
    # resume: the next iteration of the resumed optimizer is bit-identical to the uninterrupted one
    b = make_optimizer(d1, checkpoint=True, value_norm=True, value_norm_decay=0.8)
    assert b.iteration_start == 3 and b._value_norm == a._value_norm
    assert torch.equal(b.flat.param, a.flat.param) and torch.equal(b.exp_avg_sq, a.exp_avg_sq)
    la = a.train(a.batch_from_rollouts(copy.deepcopy(rollouts[2])))[0]
    lb = b.train(b.batch_from_rollouts(copy.deepcopy(rollouts[2])))[0]
    assert [float(v) for v in la.values()] == [float(v) for v in lb.values()]
    assert torch.equal(a.flat.param, b.flat.param) and torch.equal(a.exp_avg, b.exp_avg)
    # without the feature the side file is ignored and the published (raw-scale) head is used as is
    sd3 = torch.load(d1 / "model_000000003.pt", map_location="cpu")        # what b published when it was constructed
    c = make_optimizer(d1, checkpoint=True)
    assert isinstance(c, DotaOptimizer) and c.iteration_start == 4 and c.value_norm_stats is None
    assert torch.equal(c.policy_base.affine_value.weight.cpu(), sd3["affine_value.weight"])
    assert torch.equal(c.policy_base.affine_value.bias.cpu(), sd3["affine_value.bias"])


def test_run_iteration_reports_the_statistics(tmp_path):
    import pickle
    from dotaclient_b200.optimizer import MessageQueue
    port = uuid.uuid4().int % 100000
    opt = make_optimizer(tmp_path, min_seq=6, port=port, value_norm=True)
    actor = MessageQueue(host="value_norm", port=port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for r in _scaled([make_rollout(L, 900 + i, game_id=i, weight_version=1, with_canvas=True)
                      for i, L in enumerate((40, 23, 57))]):
        actor.publish_experience(pickle.dumps(r))
    met = opt.run_iteration(1)
    st = opt.value_norm_stats
    assert met["value_norm/mean"] == st["mean"] and met["value_norm/std"] == st["std"] and st["weight"] > 0
