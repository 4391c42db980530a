"""GPU tests of the V-trace advantage estimator: ``dc_vtrace_scan`` against the float64 numpy oracle (``vtrace_oracle.py``)
and against ``dc_gae_scan`` through the on-policy identities, ``DotaOptimizer(advantage_estimator='vtrace')`` experience
prep, train step and ``run_iteration`` against the CPU oracle on rollouts from a stale policy, the untouched default, and
the actor's ``act_batched`` log-probabilities against prep's."""
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
import test_gpu_parity as P  # noqa: E402
import vtrace_oracle as VT  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS, SIZES = P.HEADS, P.SIZES


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=16, epochs=1, min_seq=1, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="vtrace", rmq_port=uuid.uuid4().int % 100000, epochs=epochs, min_seq_per_epoch=min_seq,
                         seq_len=seq_len, learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                         log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=hidden_size,
                         cell=cell, **kw)


def _close(got, want, tol=1e-6):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    err = np.abs(got - want) / (1.0 + np.abs(want))
    assert err.max(initial=0.0) <= tol, (float(err.max()), int(err.argmax()))


# ------------------------------------------------------------------------------------------------ kernel vs oracle
LENS = [1, 31, 32, 33, 517, 1380]


def _kernel_inputs(n_sub, seed):
    """Segments of LENS rows.  Per row one of: log rho exactly 0, log rho spread over +-6, +800 (exp overflows to inf),
    -800 (rho = 0); heads without an action carry 0 in both log-prob arrays."""
    rng = np.random.RandomState(seed)
    off = np.concatenate([[0], np.cumsum(LENS)]).astype(np.int64)
    n = int(off[-1])
    rewards = (rng.randn(n, n_sub) * 0.1).astype(np.float32)
    values = rng.randn(n).astype(np.float32)
    acted = rng.rand(n, 5) < 0.6
    acted[:, 0] = True
    lt = np.where(acted, -3.0 * rng.rand(n, 5), 0.0).astype(np.float32)
    kind = rng.randint(0, 4, size=n)
    lb = lt.copy()
    spread = np.where(acted, rng.uniform(-6.0, 6.0, size=(n, 5)) / acted.sum(axis=1, keepdims=True), 0.0)
    lb[kind == 1] = (lt - spread).astype(np.float32)[kind == 1]
    lb[kind == 2, 0] = lt[kind == 2, 0] - 800.0
    lb[kind == 3, 0] = lt[kind == 3, 0] + 800.0
    return rewards, values, lt, lb, off


@pytest.mark.parametrize("n_sub", [10, 1])
@pytest.mark.parametrize("clips", [(1.0, 1.0), (2.0, 0.5)])
@pytest.mark.parametrize("extras", [False, True])
def test_vtrace_kernel_vs_oracle(n_sub, clips, extras):
    from dotaclient_b200 import ops
    d = P.dev()
    gamma, lam = 0.98, 0.95
    rewards, values, lt, lb, off = _kernel_inputs(n_sub, 11 * n_sub + int(clips[0]))
    lr = VT.log_rho(lt, lb)
    assert (lr == 0).any() and (lr > 710).any() and (lr < -710).any() and (np.abs(lr[np.abs(lr) < 100]) > 3).any()
    rng = np.random.RandomState(1)
    boot = rng.randn(len(LENS)).astype(np.float32) if extras else None
    valid = np.array([rng.randint(0, L + 1) for L in LENS[:-1]] + [LENS[-1]], np.int64) if extras else None
    args = (torch.from_numpy(rewards if n_sub > 1 else rewards[:, 0]).to(d), torch.from_numpy(values).to(d),
            torch.from_numpy(lt).to(d), torch.from_numpy(lb).to(d), torch.from_numpy(off).to(d), gamma, lam, *clips)
    kw = dict(boot_value=None if boot is None else torch.from_numpy(boot).to(d),
              valid_len=None if valid is None else torch.from_numpy(valid).to(d), stats=True)
    pg, vs, st = ops.vtrace_scan(*args, **kw)
    pg2, vs2, st2 = ops.vtrace_scan(*args, **kw)
    assert torch.equal(pg, pg2) and torch.equal(vs, vs2) and torch.equal(st, st2)          # deterministic, bitwise
    pg, vs, st = pg.cpu().numpy(), vs.cpu().numpy(), st.cpu().numpy()
    assert st.shape == (len(LENS), VT.STATS_SLOTS) and np.isfinite(pg).all() and np.isfinite(vs).all()
    for s, (lo, hi) in enumerate(zip(off[:-1], off[1:])):
        want_pg, want_vs = VT.vtrace(rewards[lo:hi], values[lo:hi], lr[lo:hi], gamma, lam, *clips,
                                     boot=0.0 if boot is None else boot[s])
        _close(pg[lo:hi], want_pg)
        _close(vs[lo:hi], want_vs)
        n_valid = hi - lo if valid is None else valid[s]
        want_st = VT.stats(lr[lo:lo + n_valid], *clips)
        scale = 1.0 + np.abs(lr[lo:lo + n_valid]).sum() + np.abs(want_st)
        assert (np.abs(st[s] - want_st) <= 1e-9 * scale).all(), (s, st[s], want_st)
    # without the statistics the outputs are the same
    pg3, vs3 = ops.vtrace_scan(*args, boot_value=kw["boot_value"], valid_len=kw["valid_len"])
    assert np.array_equal(pg3.cpu().numpy(), pg) and np.array_equal(vs3.cpu().numpy(), vs)


@pytest.mark.parametrize("n_sub", [10, 1])
def test_vtrace_identities_against_gae_scan(n_sub):
    """log rho = 0: vs - V equals dc_gae_scan's GAE(0.97) advantage; at lambda = 1, vs equals its returns and A its
    GAE(1) advantage."""
    from dotaclient_b200 import ops
    d = P.dev()
    rewards, values, lt, _, off = _kernel_inputs(n_sub, 5)
    r = torch.from_numpy(rewards if n_sub > 1 else rewards[:, 0]).to(d)
    v, seg, logp = torch.from_numpy(values).to(d), torch.from_numpy(off).to(d), torch.from_numpy(lt).to(d)
    adv, _ = ops.gae_scan(r, v, seg, gamma=0.98, lam=0.97)
    pg, vs = ops.vtrace_scan(r, v, logp, logp, seg, 0.98, 0.97, 1.0, 1.0)
    _close((vs.double() - v.double()).cpu().numpy(), adv.cpu().numpy())
    adv1, ret1 = ops.gae_scan(r, v, seg, gamma=0.98, lam=1.0)
    pg, vs = ops.vtrace_scan(r, v, logp, logp, seg, 0.98, 1.0, 1.0, 1.0)
    _close(vs.cpu().numpy(), ret1.cpu().numpy())
    _close(pg.cpu().numpy(), adv1.cpu().numpy())


# ------------------------------------------------------------------------------------------------ experience prep
def _stale_behaviour(opt, rollouts, seed, scale=0.05):
    """behaviour_logp of each rollout under a stale policy: the optimizer's weights plus seeded noise, the whole rollout
    run from the zero state, the taken actions' log-probs from ops.selected_logp."""
    from dotaclient_b200 import ops
    from dotaclient_b200.policy import Policy
    base = opt.policy_base
    stale = Policy(hidden_size=base.hidden_size, cell=base.cell, num_layers=base.num_layers)
    stale.load_state_dict({k: v.detach().cpu() for k, v in base.state_dict().items()})
    stale.to(P.dev())
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in stale.parameters():
            p.add_(scale * torch.randn(p.shape, generator=g).to(p.device))
    d = P.dev()
    for r in rollouts:
        L = r["rewards"].shape[0]
        obs = {k: v.unsqueeze(1).to(d) for k, v in r["observations"].items()}
        h = torch.zeros(stale.num_layers, 1, stale.hidden_size, device=d)
        with torch.no_grad():
            logits, _, _ = stale.forward_time_major(obs, (h, h.clone()) if stale.cell == "lstm" else h)
        lp = ops.selected_logp([logits[k][:, 0] for k in HEADS], [r["masks"][k].to(d) for k in HEADS],
                               [r["actions"][k].to(d) for k in HEADS])
        r["behaviour_logp"] = lp.cpu().numpy().reshape(L, 5)
    return rollouts


def _dense(seqs, per_seq):
    """Concatenation over a rollout's chunks of a dense [S, 5] per-head array (0 where the head took no action)."""
    out = []
    for s in seqs:
        dense = np.zeros((s.rewards.shape[0], 5), np.float32)
        for h, k in enumerate(HEADS):
            step = np.asarray(s.actions[k].cpu()).any(axis=-1).reshape(-1)
            dense[step, h] = np.asarray(per_seq(s, k)).reshape(-1)
        out.append(dense)
    return np.concatenate(out)


def _oracle_vtrace(oracle, rollouts, gamma=0.98, lam=0.97, rho_clip=1.0, c_clip=1.0):
    """The CPU oracle: reference prep (values, old log-probs) per rollout, then numpy V-trace over the padded rollout.
    Returns the oracle's sequences (advantages / returns replaced by V-trace's) and the per-rollout statistics."""
    seqs, stats = [], []
    for r in rollouts:
        xs = oracle.experiences_from_rollout(copy.deepcopy(r))
        L = r["rewards"].shape[0]
        old = _dense(xs, lambda s, k: s.log_probs_sel[k].numpy())
        acted = np.stack([np.asarray(r["actions"][k]).any(axis=1) for k in HEADS], axis=1)
        blp = np.zeros_like(old)
        blp[:L] = np.where(acted, r["behaviour_logp"], 0.0)
        lr = VT.log_rho(old, blp)
        rewards = np.concatenate([s.rewards for s in xs]).astype(np.float32)
        values = np.concatenate([s.values.reshape(-1).numpy() for s in xs])
        pg, vs = VT.vtrace(rewards, values, lr, gamma, lam, rho_clip, c_clip)
        S = xs[0].rewards.shape[0]
        for j, s in enumerate(xs):
            s.advantages = torch.from_numpy(pg[j * S:(j + 1) * S].astype(np.float32))
            s.returns = torch.from_numpy(vs[j * S:(j + 1) * S].astype(np.float32))
        seqs.append(xs)
        stats.append(VT.stats(lr[:L], rho_clip, c_clip))
    return seqs, stats


def _prep_fixture(tmp_path, seed=31, n=4, S=16):
    mine = make_optimizer(tmp_path, advantage_estimator="vtrace")
    oracle = P.make_oracle(128, "lstm", S)
    rollouts = _stale_behaviour(mine, P._rollouts(n, S, seed=seed), seed)
    assert max(r["rewards"].shape[0] for r in rollouts) > 2 * S and len({r["rewards"].shape[0] for r in rollouts}) > 1
    return mine, oracle, rollouts


def test_vtrace_prep_matches_the_oracle(tmp_path):
    """Ragged multi-chunk rollouts with a stale behaviour policy: batch_from_rollouts' advantages and returns equal numpy
    V-trace of the prep's own values and log-probs (1e-6 relative), and the CPU oracle's V-trace (reference prep values
    and log-probs, which the GPU prep reproduces to the parity tolerance); experiences_from_rollouts agrees with the
    batch sequence by sequence; the statistics match."""
    mine, oracle, rollouts = _prep_fixture(tmp_path)
    batch = mine.batch_from_rollouts(copy.deepcopy(rollouts))
    groups = mine.experiences_from_rollouts(copy.deepcopy(rollouts))
    oseqs, ostats = _oracle_vtrace(oracle, rollouts)
    col = 0
    for r, seqs, oxs in zip(rollouts, groups, oseqs):
        L = r["rewards"].shape[0]
        assert len(seqs) == len(oxs)
        # numpy V-trace of the GPU prep's own values and old log-probs
        old = np.concatenate([s.old_logp.cpu().numpy() for s in seqs])
        blp = np.zeros_like(old)
        acted = np.stack([np.asarray(r["actions"][k]).any(axis=1) for k in HEADS], axis=1)
        blp[:L] = np.where(acted, r["behaviour_logp"], 0.0)
        values = np.concatenate([s.values.reshape(-1).cpu().numpy() for s in seqs])
        rewards = np.concatenate([s.rewards for s in seqs]).astype(np.float32)
        pg, vs = VT.vtrace(rewards, values, VT.log_rho(old, blp), 0.98, 0.97)
        got_adv = np.concatenate([s.advantages.cpu().numpy() for s in seqs])
        got_ret = np.concatenate([s.returns.cpu().numpy() for s in seqs])
        _close(got_adv, pg)
        _close(got_ret, vs)
        assert np.abs(VT.log_rho(old, blp)[:L]).max() > 1e-2            # the behaviour policy really is stale
        for j, (s, o) in enumerate(zip(seqs, oxs)):
            torch.testing.assert_close(batch.advantages[:, col + j], s.advantages, rtol=1e-6, atol=1e-7)
            torch.testing.assert_close(batch.returns[:, col + j], s.returns, rtol=1e-6, atol=1e-7)
            torch.testing.assert_close(s.advantages.cpu(), o.advantages, rtol=1e-4, atol=2e-5)
            torch.testing.assert_close(s.returns.cpu(), o.returns, rtol=1e-4, atol=2e-5)
        col += len(seqs)
    assert col == batch.batch_size
    got, want = mine.last_vtrace_stats, VT.summary(ostats)
    assert set(got) == {"mean_log_rho", "mean_clipped_rho", "rho_clip_fraction", "c_clip_fraction"}
    n_tok = sum(r["rewards"].shape[0] for r in rollouts)
    np.testing.assert_allclose(got["mean_log_rho"], want["mean_log_rho"], rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(got["mean_clipped_rho"], want["mean_clipped_rho"], rtol=1e-4, atol=1e-5)
    for k in ("rho_clip_fraction", "c_clip_fraction"):
        assert abs(got[k] - want[k]) <= 1.5 / n_tok and 0.0 < got[k] < 1.0, k


def test_vtrace_train_step_matches_the_oracle(tmp_path):
    """One train() step on the V-trace batch, launch by launch and replayed from the captured graph, against the oracle's
    train step fed the oracle's V-trace advantages and returns."""
    eager, oracle, rollouts = _prep_fixture(tmp_path, seed=12)
    graphed = make_optimizer(tmp_path, advantage_estimator="vtrace")
    eager.use_cuda_graph = False
    oseqs, _ = _oracle_vtrace(oracle, rollouts)
    lo, eo, go = oracle.train([s for xs in oseqs for s in xs])
    lo, eo, go = ({k: float(v.detach()) for k, v in dd.items()} for dd in (lo, eo, go))
    for opt in (eager, graphed):
        batch = opt.batch_from_rollouts(copy.deepcopy(rollouts))
        if opt is graphed:
            # a warm-up step at lr = 0 runs launch by launch and leaves the weights as they are; the next step of the same
            # shape is captured and replayed
            opt.learning_rate = 0.0
            opt.train(batch)
            opt.learning_rate = 5e-5
        lm, em, gm = opt.train(batch)
        for k in lo:
            np.testing.assert_allclose(float(lm[k]), float(lo[k]), rtol=2e-4, atol=2e-6, err_msg=k)
        for k in eo:
            np.testing.assert_allclose(float(em[k]), float(eo[k]), rtol=2e-4, atol=1e-6, err_msg="entropy " + k)
        np.testing.assert_allclose(float(gm["unclipped"]), float(go["unclipped"]), rtol=2e-3)
        np.testing.assert_allclose(float(gm["clipped"]), float(go["clipped"]), rtol=2e-3)
    assert isinstance(graphed._graphs.get(batch.graph_key()), tuple), "the step was not replayed from a graph"
    assert not any(isinstance(v, tuple) for v in eager._graphs.values())


def test_vtrace_run_iteration_reports_metrics_and_refuses_rollouts_without_behaviour_logp(tmp_path):
    from dotaclient_b200.optimizer import MessageQueue
    S = 16
    lens = [40, 23, 57]
    opt = make_optimizer(tmp_path, epochs=2, min_seq=sum((L + S - 1) // S for L in lens), advantage_estimator="vtrace",
                         vtrace_rho_clip=1.5, vtrace_c_clip=0.9)
    oracle = P.make_oracle(128, "lstm", S)
    rollouts = [make_rollout(L, 300 + i, game_id=10 + i, weight_version=1) for i, L in enumerate(lens)]
    rollouts = _stale_behaviour(opt, rollouts, 8)
    _, ostats = _oracle_vtrace(oracle, rollouts, rho_clip=1.5, c_clip=0.9)
    actor = MessageQueue(host="vtrace", port=opt.rmq_port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for r in rollouts:
        actor.publish_experience(pickle.dumps(r))
    metrics = opt.run_iteration(1)
    want = VT.summary(ostats)
    n_tok = sum(lens)
    for k, w in want.items():
        got = metrics["vtrace/" + k]
        assert isinstance(got, float) and math.isfinite(got), k
        tol = 1.5 / n_tok if k.endswith("fraction") else 1e-3 * abs(w) + 1e-5
        assert abs(got - w) <= tol, (k, got, w)
    assert math.isfinite(float(metrics["loss/sum"])) and "ppo/approx_kl" in metrics
    bad = make_rollout(10 * S, 999, game_id=4242)         # enough sequences for one iteration on its own
    actor.publish_experience(pickle.dumps(bad))
    with pytest.raises(ValueError, match="game_id=4242"):
        opt.run_iteration(2)


def test_gae_default_ignores_behaviour_logp(tmp_path):
    """With the default estimator a rollout's behaviour_logp changes nothing: the batch is bitwise the one built without it,
    and run_iteration's metrics have no vtrace/ keys."""
    opt = make_optimizer(tmp_path)
    assert opt.advantage_estimator == "gae" and opt.last_vtrace_stats is None
    plain = P._rollouts(3, 16, seed=12)
    tagged = copy.deepcopy(plain)
    for r in tagged:
        r["behaviour_logp"] = np.full((r["rewards"].shape[0], 5), float("nan"), np.float32)
    a = opt.batch_from_rollouts(copy.deepcopy(plain))
    b = opt.batch_from_rollouts(tagged)
    names_a, names_b = [k for _, k, _ in a.tensors()], [k for _, k, _ in b.tensors()]
    assert names_a == names_b
    for (_, k, x), (_, _, y) in zip(a.tensors(), b.tensors()):
        assert x.dtype == y.dtype and torch.equal(x, y), k
    assert opt.last_vtrace_stats is None


def test_actor_logp_equals_prep_logp_at_the_same_weights(tmp_path):
    """A pool of agents plays step by step with act_batched (recurrence S = 1, expf) at the optimizer's own weights; prep
    recomputes the same log-probs over the whole rollout (S = L, __expf).  log rho per token stays within 1e-4."""
    S, A, L = 16, 4, 45
    opt = make_optimizer(tmp_path, advantage_estimator="vtrace")
    pol, d = opt.policy_base, P.dev()
    g = torch.Generator().manual_seed(17)
    rolls = [make_rollout(L, 700 + a, game_id=a) for a in range(A)]
    h = torch.zeros(pol.num_layers, A, pol.hidden_size, device=d)
    hidden = (h, h.clone())
    chosen_all, logp_all, legal_all = [], [], []
    for t in range(L):
        obs = {k: torch.stack([r["observations"][k][t] for r in rolls]).to(d) for k in pol.INPUT_KEYS}
        legal = {k: torch.ones(A, n, dtype=torch.bool) for k, n in zip(HEADS, SIZES)}
        legal["target_unit"] = torch.rand(A, 40, generator=g) < 0.5
        legal["target_unit"][:, 0] = False
        legal["target_unit"][:, 1] = True
        u = torch.rand(A, 5, generator=g)
        chosen, logp, _, _, hidden = pol.act_batched(hidden, obs, {k: v.to(d) for k, v in legal.items()}, u.to(d))
        chosen_all.append({k: v.cpu() for k, v in chosen.items()})
        logp_all.append(logp.cpu())
        legal_all.append(legal)
    for a, r in enumerate(rolls):
        for h_i, k in enumerate(HEADS):
            n = SIZES[h_i]
            acts = torch.zeros(L, n, dtype=torch.bool)
            masks = torch.zeros(L, n, dtype=torch.bool)
            for t in range(L):
                c = int(chosen_all[t][k][a])
                if c >= 0:
                    acts[t, c] = True
                    masks[t] = legal_all[t][k][a]                  # the mask of a head the agent used
            r["actions"][k], r["masks"][k] = acts, masks
        r["behaviour_logp"] = torch.stack([logp_all[t][a] for t in range(L)]).numpy()
    groups = opt.experiences_from_rollouts(copy.deepcopy(rolls))
    worst = 0.0
    for r, seqs in zip(rolls, groups):
        old = np.concatenate([s.old_logp.cpu().numpy() for s in seqs])[:L]
        acted = np.stack([r["actions"][k].numpy().any(axis=1) for k in HEADS], axis=1)
        assert acted[:, 1:].any() and (old[~acted] == 0).all()
        worst = max(worst, float(np.abs(VT.log_rho(old, np.where(acted, r["behaviour_logp"], 0.0))).max()))
    print("act_batched vs prep: max |log rho| per token = %.3g" % worst)
    assert worst <= 1e-4
    st = opt.last_vtrace_stats
    assert abs(st["mean_log_rho"]) <= 1e-4 and abs(st["mean_clipped_rho"] - 1.0) <= 1e-4
