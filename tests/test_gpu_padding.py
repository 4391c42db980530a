"""GPU tests of ``mask_padding``: ``dc_ppo_loss_fwd_bwd_masked`` against the CPU oracle and bitwise against ``_dev``,
experience prep with the terminal bootstrap at each rollout's real end (GAE and V-trace), the whole masked step against the
CPU oracle, and the bit-identities that define the feature: whole-chunk rollouts train exactly as without masking, and
the padded tail's observations reach no loss, gradient or weight bit."""
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
import padding_oracle as PO  # noqa: E402
import test_gpu_parity as P  # noqa: E402
import test_gpu_vtrace as V  # noqa: E402
import vtrace_oracle as VT  # noqa: E402
from stacked_oracle import StackedRefPolicy  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS, SIZES = P.HEADS, P.SIZES


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=16, epochs=1, min_seq=1, port=None, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="padding", rmq_port=port if port is not None else uuid.uuid4().int % 100000,
                         epochs=epochs, min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=5e-5, checkpoint=False,
                         pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5,
                         run_local=True, hidden_size=hidden_size, cell=cell, **kw)


RAGGED = (40, 23, 48, 7, 33)          # 3 + 2 + 3 + 1 + 3 = 12 sequences of 16; 48 fills its chunks


def _ragged(seed=0, lengths=RAGGED):
    return [make_rollout(L, 700 + 10 * seed + i, game_id=i) for i, L in enumerate(lengths)]


# ------------------------------------------------------------------------------------------------ the kernel
def _kernel(inputs, clip, valid, packed=False):
    from dotaclient_b200 import ops
    logits, values, actions, masks, old, adv, ret, ov = inputs
    d = P.dev()
    hp = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5, value_clip=clip)
    v = None if valid is None else valid.to(d)
    if not packed:
        return ops.ppo_loss_fwd_bwd([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                                    [actions[k].to(d) for k in HEADS], old.to(d), adv.to(d), ret.to(d), values.to(d),
                                    0.0, 0.0, 0.0, hparams=hp, old_value=ov.to(d), valid=v)
    n = values.numel()
    pk = torch.zeros(n, ops.PACK_WIDTH)
    for k in ("enum", "x", "y", "ability"):
        lo, hi = ops.PACK_COLS[k]
        pk[:, lo:hi] = logits[k]
    pk[:, ops.PACK_COLS["value"][0]] = values
    return ops.ppo_loss_packed(pk.to(d), logits["target_unit"].to(d), [masks[k].to(d) for k in HEADS],
                               [actions[k].to(d) for k in HEADS], old.to(d), adv.to(d), ret.to(d), 0.0, 0.0, 0.0,
                               hparams=hp, old_value=ov.to(d), valid=v)


def _inputs(n, seed):
    import test_padding_host as H
    logits, values, actions, masks, old, adv, ret, valid = H._case(n, seed, invalid_actions=True)
    ov = values + 0.2 * torch.randn(n, generator=torch.Generator().manual_seed(seed))
    return (logits, values, actions, masks, old, adv, ret, ov), valid


@pytest.mark.parametrize("n", [129, 300, 1000])
@pytest.mark.parametrize("clip", [None, 0.2])
def test_masked_kernel_vs_oracle(n, clip):
    """Multi-CTA batches whose invalid rows hold actions: losses, entropies, advantage mean / std, n_actions (bit-exact),
    diagnostics, dlogits and dvalue against the oracle's autograd; invalid rows exactly 0."""
    inputs, valid = _inputs(n, 11 + n)
    logits, values, actions, masks, old, adv, ret, ov = inputs
    lg = {k: t.clone().requires_grad_(True) for k, t in logits.items()}
    vg = values.clone().requires_grad_(True)
    loss, p_loss, e_loss, v_loss, ents = PO.masked_ppo_loss(lg, vg, actions, masks, old, adv, ret, valid, 5e-4, 0.5, 0.1,
                                                            old_values=ov, value_clip=clip)
    loss.backward()
    out, n_act, dlogits, dvalue, stats = _kernel(inputs, clip, valid)
    out = out.cpu().numpy()
    assert n_act.cpu().tolist() == [int((actions[k].any(dim=1) & valid).sum()) for k in HEADS]
    assert any(bool((actions[k].any(dim=1) & ~valid).any()) for k in HEADS)       # invalid rows with actions exist
    for i, want in enumerate((loss, p_loss, e_loss, v_loss)):
        np.testing.assert_allclose(out[i], float(want), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out[4:9], [float(ents[k]) for k in HEADS], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out[14], float(adv[valid].mean()), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(out[15], float(adv[valid].std()), rtol=1e-5)
    st = PO.masked_stats(logits, actions, masks, old, values, ret, valid, 0.1)
    from dotaclient_b200.optimizer import DotaOptimizer
    got = DotaOptimizer._ppo_stats_dict(stats.cpu().tolist())
    for k, w in st.items():
        np.testing.assert_allclose(got[k], w, rtol=1e-4, atol=1e-6, err_msg=k)
    for h, k in enumerate(HEADS):
        g = dlogits[h].cpu()
        g_ref = lg[k].grad if lg[k].grad is not None else torch.zeros_like(g)
        torch.testing.assert_close(g, g_ref, rtol=2e-4, atol=1e-8)
        assert bool((g[~valid] == 0).all()), k
    dv = dvalue.cpu()
    torch.testing.assert_close(dv, vg.grad, rtol=1e-4, atol=1e-9)
    assert bool((dv[~valid] == 0).all())


def _same_result(got, want, packed):
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]) and torch.equal(got[4], want[4])
    if packed:
        assert torch.equal(got[2], want[2]) and torch.equal(got[3], want[3])
    else:
        assert all(torch.equal(a, b) for a, b in zip(got[2], want[2])) and torch.equal(got[3], want[3])


@pytest.mark.parametrize("packed", [False, True])
def test_masked_kernel_without_mask_or_all_valid_is_dev_bitwise(packed, monkeypatch):
    """dc_ppo_loss_fwd_bwd_masked with a NULL mask and with an all-true mask == dc_ppo_loss_fwd_bwd_dev, bit for bit:
    losses, statistics, n_actions and every gradient, with and without value clipping."""
    from dotaclient_b200 import _lib
    lib = _lib.load()
    inputs, _ = _inputs(1000, 3)
    for clip in (None, 0.2):
        want = _kernel(inputs, clip, None, packed)                   # valid=None: the _dev entry point
        _same_result(_kernel(inputs, clip, torch.ones(1000, dtype=torch.bool), packed), want, packed)
        masked, calls = lib.dc_ppo_loss_fwd_bwd_masked, []

        def masked_null(*a):
            calls.append(1)
            return masked(*a[:10], None, *a[10:])
        with monkeypatch.context() as m:                             # the masked entry point with valid = NULL
            m.setattr(lib, "dc_ppo_loss_fwd_bwd_dev", masked_null)
            _same_result(_kernel(inputs, clip, None, packed), want, packed)
        assert calls == [1]


def test_masked_kernel_with_no_or_one_valid_token_has_a_nan_std():
    inputs, _ = _inputs(300, 5)
    for n_valid in (0, 1):
        valid = torch.zeros(300, dtype=torch.bool)
        valid[:n_valid] = True
        out = _kernel(inputs, None, valid)[0].cpu()
        assert math.isnan(float(out[15])), n_valid


# ------------------------------------------------------------------------------------------------ prep
def _prep_check(opt, rollouts, vtrace):
    batch = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    groups = opt.experiences_from_rollouts(copy.deepcopy(rollouts))
    S, col = opt.seq_len, 0
    for r, seqs in zip(rollouts, groups):
        L = int(r["rewards"].shape[0])
        n = len(seqs)
        values = batch.old_values[:, col:col + n].t().reshape(-1).cpu().numpy()
        rewards = np.sum(np.asarray(r["rewards"], dtype=np.float32), axis=1)
        if vtrace:
            old = batch.old_logp[:, col:col + n].transpose(0, 1).reshape(-1, 5).cpu().numpy()[:L]
            acted = np.stack([np.asarray(r["actions"][k]).any(axis=1) for k in HEADS], axis=1)
            pg, vs = VT.vtrace(rewards, values[:L], VT.log_rho(old, np.where(acted, r["behaviour_logp"], 0.0)), 0.98, 0.97)
            want_adv, want_ret = pg, vs
        else:
            want_adv, want_ret = PO.real_advantage_returns(rewards, values[:L])
        adv = batch.advantages[:, col:col + n].t().reshape(-1).cpu().numpy()
        ret = batch.returns[:, col:col + n].t().reshape(-1).cpu().numpy()
        V._close(adv[:L], want_adv)
        V._close(ret[:L], want_ret)
        assert (adv[L:] == 0).all() and (ret[L:] == 0).all()
        valid = batch.valid[:, col:col + n].t().reshape(-1).cpu()
        assert valid.tolist() == [True] * L + [False] * (n * S - L)
        for j, s in enumerate(seqs):
            assert torch.equal(s.valid, batch.valid[:, col + j])
            assert torch.equal(s.advantages, batch.advantages[:, col + j]) and torch.equal(s.returns, batch.returns[:, col + j])
        col += n
    assert col == batch.batch_size
    return batch


def test_prep_bootstraps_at_each_rollouts_real_end(tmp_path):
    """GAE: real rows equal advantage_returns(r[:L] + [0], V[:L] + [0]) on prep's own values, padded rows are 0."""
    opt = make_optimizer(tmp_path, mask_padding=True)
    batch = _prep_check(opt, _ragged(1), vtrace=False)
    assert batch.valid.dtype == torch.bool and batch.valid.shape == (16, 12)


def test_vtrace_prep_on_the_real_length(tmp_path):
    opt = make_optimizer(tmp_path, mask_padding=True, advantage_estimator="vtrace")
    rollouts = V._stale_behaviour(opt, _ragged(2), 2)
    _prep_check(opt, rollouts, vtrace=True)
    got = opt.last_vtrace_stats
    ref = make_optimizer(tmp_path, advantage_estimator="vtrace")
    ref.batch_from_rollouts(copy.deepcopy(rollouts))
    assert opt._vtrace_seg_stats.shape[0] == 2 * len(rollouts)
    for k, v in ref.last_vtrace_stats.items():          # the statistics already covered the real steps only
        assert got[k] == pytest.approx(v, rel=1e-12, abs=1e-15), k


# ------------------------------------------------------------------------------------------------ bit-identities
def _train_record(opt, batch, steps=2):
    rec = []
    for _ in range(steps):
        l, e, g = opt.train(batch)
        rec.append(([float(v) for v in l.values()], [float(v) for v in e.values()], [float(v) for v in g.values()],
                    dict(opt.last_ppo_stats)))
    return rec


def _same_rec(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x[:3] == y[:3]
        assert all(x[3][k] == y[3][k] or (x[3][k] != x[3][k] and y[3][k] != y[3][k]) for k in x[3])


@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
def test_whole_chunk_rollouts_train_as_without_masking(estimator, tmp_path):
    a = make_optimizer(tmp_path, advantage_estimator=estimator)
    b = make_optimizer(tmp_path, advantage_estimator=estimator, mask_padding=True)
    rollouts = _ragged(3, (32, 16, 48))
    if estimator == "vtrace":
        rollouts = V._stale_behaviour(a, rollouts, 3)
    ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    assert ba.valid is None and bool(bb.valid.all())
    for (_, k, x), (_, _, y) in zip(ba.tensors(), bb.tensors()):
        assert torch.equal(x, y), k
    _same_rec(_train_record(a, ba, 3), _train_record(b, bb, 3))
    assert torch.equal(a.flat.param, b.flat.param) and torch.equal(a.exp_avg_sq, b.exp_avg_sq)


@pytest.mark.parametrize("H,cell,layers", [(256, "gru", 1), (128, "lstm", 2)])
def test_padded_observations_reach_no_bit(H, cell, layers, tmp_path):
    """With masking, random finite observations in the padded tail change no loss, gradient, weight or moment bit."""
    a = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers, mask_padding=True)
    b = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers, mask_padding=True)
    batch = a.batch_from_rollouts(_ragged(4))
    noisy = batch.map(lambda v: v.clone())
    g = torch.Generator(device=P.dev()).manual_seed(5)
    pad = ~noisy.valid
    for k, t in noisy.observations.items():
        t[pad] = 3.0 * torch.randn(t[pad].shape, generator=g, device=t.device)
    assert not torch.equal(noisy.observations["env"], batch.observations["env"])
    for step in range(2):
        ra, rb = _train_record(a, batch, 1), _train_record(b, noisy, 1)
        _same_rec(ra, rb)
        assert torch.equal(a.flat.grad_full, b.flat.grad_full), step
    assert torch.equal(a.flat.param, b.flat.param)
    assert torch.equal(a.exp_avg, b.exp_avg) and torch.equal(a.exp_avg_sq, b.exp_avg_sq)


def test_graph_replay_equals_launch_by_launch(tmp_path):
    a = make_optimizer(tmp_path, mask_padding=True)
    b = make_optimizer(tmp_path, mask_padding=True)
    a.use_cuda_graph, b.use_cuda_graph = False, True
    batch = a.batch_from_rollouts(_ragged(5))
    _same_rec(_train_record(a, batch, 4), _train_record(b, batch, 4))
    assert any(isinstance(v, tuple) and k[-1] == "valid" for k, v in b._graphs.items())
    assert torch.equal(a.flat.param, b.flat.param) and torch.equal(a.exp_avg, b.exp_avg)


def test_train_epochs_minibatches_equal_index_select_batches(tmp_path):
    from dotaclient_b200.optimizer import minibatch_indices
    a = make_optimizer(tmp_path, epochs=2, min_seq=3, num_minibatches=3, mask_padding=True)
    b = make_optimizer(tmp_path, epochs=2, min_seq=3, mask_padding=True)
    rollouts = _ragged(6)
    batch_a, batch_b = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    rng = copy.deepcopy(a.minibatch_rng)
    la, ea, ga, sa = a.train_epochs(batch_a)
    got = [([float(v) for v in l.values()], [float(v) for v in e.values()], [float(v) for v in g.values()], s)
           for l, e, g, s in zip(la, ea, ga, sa)]
    want = []
    for _ in range(2):
        for idx in minibatch_indices(batch_b.batch_size, 3, rng):
            mb = batch_b.map(lambda v: v.index_select(1, torch.as_tensor(idx, device=v.device)))
            want += _train_record(b, mb, 1)
    _same_rec(got, want)
    assert torch.equal(a.flat.param, b.flat.param) and torch.equal(a.exp_avg_sq, b.exp_avg_sq)


# ------------------------------------------------------------------------------------------------ the step vs the oracle
@pytest.mark.parametrize("H,cell,layers", [(256, "gru", 1), (128, "lstm", 2)])
def test_masked_step_vs_oracle(H, cell, layers, tmp_path):
    """Masked prep + two train() steps against the CPU oracle on ragged multi-chunk rollouts, at the parity suite's
    tolerances: prep outputs, losses, entropies, grad norms, per-tensor gradient cosine, Adam moments."""
    torch.set_num_threads(8)
    S = 16
    mine = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers, mask_padding=True)
    torch.manual_seed(7)
    oracle = PO.MaskedRefOptimizer(StackedRefPolicy(H, cell, layers), seq_len=S)
    rollouts = _ragged(7)
    xs_m = [s for grp in mine.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in grp]
    xs_o = [s for r in rollouts for s in oracle.experiences_from_rollout(copy.deepcopy(r))]
    P._compare_sequences(xs_m, xs_o, cell)
    for a, b in zip(xs_m, xs_o):
        assert torch.equal(a.valid.cpu(), b.valid)
    for ep in range(2):
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
                cos = torch.nn.functional.cosine_similarity(g.flatten(), p.grad.flatten(), dim=0)
                assert cos > 0.9999, (name, float(cos))
                np.testing.assert_allclose(float(g.norm()), float(p.grad.norm()), rtol=2e-3, err_msg=name)
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
        cos = torch.nn.functional.cosine_similarity(st["exp_avg"].flatten(), w["exp_avg"].flatten(), dim=0)
        assert cos > 0.9999, (names[i], float(cos))


# ------------------------------------------------------------------------------------------------ train / run_iteration
def test_train_refuses_batches_it_cannot_mask(tmp_path):
    opt = make_optimizer(tmp_path, mask_padding=True)
    plain = make_optimizer(tmp_path).batch_from_rollouts(_ragged(8, (40,)))
    with pytest.raises(ValueError, match="mask_padding"):
        opt.train(plain)
    batch = opt.batch_from_rollouts(_ragged(8, (40,)))
    batch.valid = torch.zeros_like(batch.valid)              # no valid token: NaN advantage std -> the NaN-loss error
    before = opt.flat.param.clone()
    with pytest.raises(ValueError, match="loss=nan"):
        opt.train(batch)
    assert torch.equal(opt.flat.param, before) and int(opt.adam_steps.max()) == 0


def _run_iteration(tmp_path, port, rollouts, **kw):
    from dotaclient_b200.optimizer import MessageQueue
    opt = make_optimizer(tmp_path, min_seq=6, port=port, **kw)
    actor = MessageQueue(host="padding", port=port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for r in rollouts:
        actor.publish_experience(pickle.dumps(r))
    return opt, opt.run_iteration(1)


def test_run_iteration_reports_padding_fraction(tmp_path):
    rollouts = [make_rollout(L, 900 + i, game_id=i, weight_version=1, with_canvas=True) for i, L in enumerate((40, 23, 57))]
    base = uuid.uuid4().int % 100000
    m1, met1 = _run_iteration(tmp_path, base, rollouts, mask_padding=True, num_minibatches=2)
    m0, met0 = _run_iteration(tmp_path, base + 1, rollouts)
    assert set(met1) - set(met0) == {"padding_fraction"} and set(met0) <= set(met1)
    assert met1["padding_fraction"] == pytest.approx((9 * 16 - (40 + 23 + 57)) / (9 * 16), rel=1e-12)
    assert int(m1.adam_steps.max()) == 2
    assert not torch.equal(m1.flat.param, m0.flat.param)
