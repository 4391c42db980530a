"""GPU tests of UPGO (``DotaOptimizer(upgo_coef=c)``): ``dc_upgo_scan`` against the float64 oracle (``upgo_oracle.py``)
on ragged segments and at the benchmark's token count, its identities against ``dc_gae_scan``, the indexed form against
the plain one, and experience prep, the advantage refresh and ``run_iteration`` with every option UPGO composes with."""
import copy
import os
import pickle
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_continuation as C  # noqa: E402
import test_gpu_packing as PK  # noqa: E402
import test_gpu_parity as P  # noqa: E402
import test_gpu_vtrace as V  # noqa: E402
import upgo_oracle as UP  # noqa: E402
import vtrace_oracle as VT  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
GAMMA = 0.98


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=16, epochs=1, min_seq=1, lr=5e-5, port=None, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="upgo", rmq_port=port if port is not None else uuid.uuid4().int % 100000,
                         epochs=epochs, min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=lr, checkpoint=False,
                         pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5,
                         run_local=True, hidden_size=hidden_size, cell=cell, **kw)


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(P.dev())


# ------------------------------------------------------------------------------------------------ kernel vs oracle
LENS = [1, 31, 32, 33, 97, 130, 517]


def _inputs(lens, seed, n_sub=10):
    g = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = int(off[-1])
    lt = np.where(g.random((n, 5)) < 0.6, -3.0 * g.random((n, 5)), 0.0).astype(np.float32)
    lb = (lt + np.where(lt != 0, g.uniform(-0.7, 0.7, (n, 5)), 0.0)).astype(np.float32)
    return dict(off=off, n=n, rewards=(g.standard_normal((n, n_sub)) * 0.3).astype(np.float32),
                values=g.standard_normal(n).astype(np.float32), base=g.standard_normal(n).astype(np.float32), lt=lt, lb=lb,
                boot=g.standard_normal(len(lens)).astype(np.float32),
                valid=np.array([g.integers(0, L + 1) for L in lens], np.int64))


def _oracle(x, vtrace, boot, valid, coef, rho_clip=1.0):
    """Per segment: prep's advantage fp32(base + c A^U) and the statistics over the first valid rows."""
    want = np.zeros(x["n"], np.float32)
    stats = []
    for s, (lo, hi) in enumerate(zip(x["off"][:-1], x["off"][1:])):
        lr = VT.log_rho(x["lt"][lo:hi], x["lb"][lo:hi]) if vtrace else None
        au, through = UP.upgo(x["rewards"][lo:hi], x["values"][lo:hi], GAMMA, 0.0 if boot is None else boot[s], lr,
                              rho_clip)
        want[lo:hi] = UP.advantages(x["base"][lo:hi], au, coef)
        k = hi - lo if valid is None else valid[s]
        stats.append(UP.stats(au[:k], through[:k]))
    return want, np.array(stats)


def _run(x, vtrace, boot, valid, coef, rho_clip=1.0, stats=True):
    from dotaclient_b200 import ops
    adv = T(x["base"])
    out = ops.upgo_scan(T(x["rewards"]), T(x["values"]), T(x["off"]), adv, GAMMA, coef,
                        boot_value=None if boot is None else T(boot), logp_target=T(x["lt"]) if vtrace else None,
                        logp_behaviour=T(x["lb"]) if vtrace else None, rho_clip=rho_clip,
                        valid_len=None if valid is None else T(valid), stats=stats)
    return out


@pytest.mark.parametrize("vtrace", [False, True])
@pytest.mark.parametrize("extras", [False, True])
def test_kernel_vs_oracle(vtrace, extras):
    """Segments of 1, 31, 32, 33 and >= 3 tiles, with and without bootstraps and [real | padding] valid lengths: the
    outputs within fp32 rounding of float64, the row and through counts exact, the sum of A^U to 1e-12."""
    x = _inputs(LENS, 3 + vtrace + 2 * extras)
    boot, valid = (x["boot"], x["valid"]) if extras else (None, None)
    rho_clip = 1.5 if vtrace else 1.0
    adv, st = _run(x, vtrace, boot, valid, 0.5, rho_clip)
    adv2, st2 = _run(x, vtrace, boot, valid, 0.5, rho_clip)
    assert torch.equal(adv, adv2) and torch.equal(st, st2)              # deterministic, bitwise
    want, want_st = _oracle(x, vtrace, boot, valid, 0.5, rho_clip)
    V._close(adv.cpu().numpy(), want, 1e-6)
    st = st.cpu().numpy()
    assert np.array_equal(st[:, :2], want_st[:, :2])
    assert 0 < st[:, 1].sum() < st[:, 0].sum()                           # both kinds of step occur
    assert np.all(np.abs(st[:, 2] - want_st[:, 2]) <= 1e-12 * (1 + st[:, 0] * 10))
    assert torch.equal(_run(x, vtrace, boot, valid, 0.5, rho_clip, stats=False), adv)    # the statistics change nothing


def test_benchmark_scale_vs_oracle():
    """256 rollouts x 512 rows (the C2 batch's 131,072 tokens), GAE and V-trace: 24 sampled segments against float64."""
    x = _inputs([512] * 256, 17)
    pick = np.random.default_rng(0).choice(256, 24, replace=False)
    for vtrace in (False, True):
        adv, st = _run(x, vtrace, x["boot"], None, 0.75)
        adv, st = adv.cpu().numpy(), st.cpu().numpy()
        want, want_st = _oracle(x, vtrace, x["boot"], None, 0.75)
        for s in pick:
            lo, hi = x["off"][s], x["off"][s + 1]
            V._close(adv[lo:hi], want[lo:hi], 1e-6)
            assert np.array_equal(st[s, :2], want_st[s, :2])


def _signed(lens, seed, sign):
    """Values for which every TD error has ``sign`` (by a margin), from the end of each segment backwards."""
    x = _inputs(lens, seed)
    r = VT.reward_sum(x["rewards"]).astype(np.float64)
    g = np.random.default_rng(seed + 1)
    for s, (lo, hi) in enumerate(zip(x["off"][:-1], x["off"][1:])):
        v_next = float(x["boot"][s])
        for t in range(hi - 1, lo - 1, -1):
            x["values"][t] = np.float32(r[t] + GAMMA * v_next - sign * (0.05 + g.random()))
            v_next = float(x["values"][t])
    return x


@pytest.mark.parametrize("sign", [+1, -1])
def test_identities_against_gae_scan(sign):
    """All through (every delta >= 0): A^U = ret - V with dc_gae_scan's ret.  None through: A^U = dc_gae_scan's
    advantage at lambda = 0."""
    from dotaclient_b200 import ops
    x = _signed(LENS, 40, sign)
    x["base"][:] = 0
    adv, st = _run(x, False, x["boot"], None, 1.0)
    st = st.cpu().numpy()
    assert st[:, 1].sum() == (st[:, 0].sum() - len(LENS) if sign > 0 else 0)
    r, v, seg, boot = T(x["rewards"]), T(x["values"]), T(x["off"]), T(x["boot"])
    adv = adv.cpu().numpy()
    if sign > 0:
        _, ret = ops.gae_scan(r, v, seg, GAMMA, 0.97, boot_value=boot, boot_reward=boot)
        V._close(adv, (ret.double() - v.double()).cpu().numpy(), 2e-6)
        return
    want, _ = ops.gae_scan(r, v, seg, GAMMA, 0.0, boot_value=boot, boot_reward=boot)
    # dc_gae_scan forms the TD error in fp32 (gamma rounded to fp32, three roundings): its error is a few fp32 ulps of
    # the operands, not of the difference; the float64 oracle's delta pins the UPGO side to its own rounding
    rs = VT.reward_sum(x["rewards"]).astype(np.float64)
    vs = x["values"].astype(np.float64)
    v_next = np.concatenate([np.append(vs[lo + 1:hi], x["boot"][s]) for s, (lo, hi) in
                             enumerate(zip(x["off"][:-1], x["off"][1:]))])
    delta = (rs + GAMMA * v_next) - vs
    V._close(adv, delta, 1e-7)
    scale = np.abs(rs) + GAMMA * np.abs(v_next) + np.abs(vs)
    assert (np.abs(adv - want.cpu().numpy()) <= 4 * np.finfo(np.float32).eps * scale + 1e-7).all()


@pytest.mark.parametrize("vtrace", [False, True])
def test_indexed_equals_plain_bitwise(vtrace):
    """Rows scattered over a larger token array, some rows held by no token (value 0, nothing written): the indexed form
    adds exactly what the plain form adds, and every other token keeps its contents."""
    from dotaclient_b200 import ops
    x = _inputs(LENS, 8)
    n = x["n"]
    g = np.random.default_rng(9)
    n_tok = n + 300
    perm = g.permutation(n_tok)[:n]
    tok = np.where(g.random(n) < 0.1, -1, perm).astype(np.int64)
    x["values"][tok < 0] = 0.0
    if vtrace:
        x["lt"][tok < 0] = 0.0
    adv, _ = _run(x, vtrace, x["boot"], x["valid"], 0.5)
    store = np.zeros((n_tok, 8), np.float32)                           # the values as a column at a stride of 8
    store[tok[tok >= 0], 3] = x["values"][tok >= 0]
    lt_tok = np.zeros((n_tok, 5), np.float32)
    lt_tok[tok[tok >= 0]] = x["lt"][tok >= 0]
    fill = np.full(n_tok, 2.5, np.float32)
    fill[tok[tok >= 0]] = x["base"][tok >= 0]
    got = T(fill)
    ops.upgo_scan_indexed(T(x["rewards"]), T(store)[:, 3], T(tok), T(x["off"]), got, GAMMA, 0.5, boot_value=T(x["boot"]),
                          logp_target=T(lt_tok) if vtrace else None, logp_behaviour=T(x["lb"]) if vtrace else None)
    got, adv = got.cpu().numpy(), adv.cpu().numpy()
    held = tok >= 0
    assert np.array_equal(got[tok[held]], adv[held])
    free = np.ones(n_tok, bool)
    free[tok[held]] = False
    assert free.sum() >= 300 and (got[free] == 2.5).all()


# ------------------------------------------------------------------------------------------------ experience prep
PREP_CONFIGS = {
    "gae": dict(),
    "gae_masked": dict(mask_padding=True),
    "gae_packed_popart": dict(mask_padding=True, pack_sequences=True, value_norm=True),
    "vtrace": dict(advantage_estimator="vtrace"),
    "vtrace_packed": dict(advantage_estimator="vtrace", mask_padding=True, pack_sequences=True),
}


def _oracle_batch(batch0, coef, vtrace, rho_clip=1.0):
    """From the batch of an optimizer without UPGO, with its refresh record (prep's rollout-major rewards, segments,
    bootstraps, behaviour log-probs and the token of every row): the expected advantages fp32(A_base + c A^U) of every
    token, the tokens that hold a row, and the per-segment A^U and through flags."""
    r = batch0.refresh
    tok = r.tok.cpu().numpy()
    held = tok >= 0

    def at(t):                       # a [S, B, ...] batch tensor at prep's rollout-major rows, 0 where no token holds one
        rows = t.reshape((-1,) + tuple(t.shape[2:])).cpu().numpy()[np.maximum(tok, 0)]
        return np.where(held.reshape((-1,) + (1,) * (rows.ndim - 1)), rows, 0)
    values = at(batch0.old_values).astype(np.float32)
    base = at(batch0.advantages).astype(np.float32)
    lt = at(batch0.old_logp).astype(np.float32) if vtrace else None
    lb = r.behaviour_logp.cpu().numpy() if vtrace else None
    rewards = r.rewards.cpu().numpy()
    off = r.seg_off.cpu().numpy()
    boot = np.zeros(len(off) - 1, np.float32) if r.boot is None else r.boot.cpu().numpy()
    want = batch0.advantages.reshape(-1).cpu().numpy().copy()
    per_seg = []
    for s, (lo, hi) in enumerate(zip(off[:-1], off[1:])):
        if hi <= lo:
            per_seg.append((np.zeros(0), np.zeros(0, bool)))
            continue
        lr = VT.log_rho(lt[lo:hi], lb[lo:hi]) if vtrace else None
        au, through = UP.upgo(rewards[lo:hi], values[lo:hi], GAMMA, boot[s], lr, rho_clip)
        a = UP.advantages(base[lo:hi], au, coef)
        h = held[lo:hi]
        want[tok[lo:hi][h]] = a[h]
        per_seg.append((au, through))
    return want, held, per_seg


def _fields_equal(a, b, skip=()):
    for f in a.FIELDS:
        x, y = getattr(a, f), getattr(b, f)
        if f in skip:
            continue
        assert (x is None) == (y is None), f
        if x is not None:
            assert torch.equal(x, y), f
    for d in ("observations", "masks", "actions"):
        for k in getattr(a, d):
            assert torch.equal(getattr(a, d)[k], getattr(b, d)[k]), (d, k)


@pytest.mark.parametrize("name", sorted(PREP_CONFIGS))
def test_prep_matches_the_oracle(name, tmp_path):
    """Ragged rollouts, some cut from a longer game (bootstrapped from V(s_L)), all from non-zero initial states: prep's
    advantages equal fp32(A_base + c A^U) of the float64 oracle over prep's own values, rewards, segments and bootstraps;
    everything else in the batch is the batch without UPGO, bit for bit; upgo_coef = 0 is the default, bit for bit; the
    statistics match the oracle's over the real steps."""
    from dotaclient_b200.optimizer import rollout_segments
    kw = PREP_CONFIGS[name]
    vtrace = kw.get("advantage_estimator") == "vtrace"
    default = make_optimizer(tmp_path, recompute_advantages=True, **kw)
    off = make_optimizer(tmp_path, recompute_advantages=True, upgo_coef=0.0, **kw)
    on = make_optimizer(tmp_path, recompute_advantages=True, upgo_coef=0.5, **kw)
    rollouts = C._mixed(default, 3, behaviour=vtrace)
    b_def, b_off, b_on = (o.batch_from_rollouts(copy.deepcopy(rollouts)) for o in (default, off, on))
    _fields_equal(b_def, b_off)
    assert default.last_upgo_stats is None and off.last_upgo_stats is None
    _fields_equal(b_off, b_on, skip=("advantages",))
    want, held, per_seg = _oracle_batch(b_off, 0.5, vtrace)
    got = b_on.advantages.reshape(-1).cpu().numpy()
    V._close(got, want, 1e-6)
    assert not np.array_equal(got, b_off.advantages.reshape(-1).cpu().numpy())
    if "mask_padding" in kw:
        assert (b_on.advantages[~b_on.valid] == 0).all()
    # statistics over the real steps
    Ls = [r["rewards"].shape[0] for r in rollouts]
    terminal = [bool(r.get("terminal", True)) for r in rollouts]
    _, _, valid_len = rollout_segments(Ls, terminal, 16, on.mask_padding)
    n = thr = s = 0.0
    for (au, through), k in zip(per_seg, valid_len):
        n, thr, s = n + k, thr + through[:k].sum(), s + au[:k].sum()
    st = on.last_upgo_stats
    assert abs(st["through_fraction"] - thr / n) < 1e-12 and abs(st["mean_advantage"] - s / n) < 1e-9
    assert 0 < st["through_fraction"] < 1


@pytest.mark.parametrize("name", ["gae", "gae_masked", "vtrace_packed"])
def test_refresh_at_unchanged_weights_is_prep(name, tmp_path):
    """The refresh's scans fed prep's own values (and target log-probs) rewrite prep's advantages and returns bit for
    bit.  Then learning_rate = 0, epochs = 2: the refresh forward runs at another batch shape than prep's, so its values
    may differ in the last bits, and the refreshed advantages agree with prep's to fp32 rounding, as without UPGO."""
    kw = dict(PREP_CONFIGS[name])
    vtrace = kw.get("advantage_estimator") == "vtrace"
    opt = make_optimizer(tmp_path, epochs=2, lr=0.0, recompute_advantages=True, upgo_coef=0.5, **kw)
    batch = opt.batch_from_rollouts(C._mixed(opt, 1, behaviour=vtrace))
    adv0, ret0 = batch.advantages.clone(), batch.returns.clone()
    batch.advantages.fill_(11.0)
    batch.returns.fill_(-11.0)
    if batch.valid is not None:                         # rows no token of the refresh holds keep prep's zeros
        batch.advantages[~batch.valid] = 0
        batch.returns[~batch.valid] = 0
    opt._rescan(batch, batch.old_values, batch.old_logp.reshape(-1, 5) if vtrace else None, batch.refresh.boot)
    assert torch.equal(batch.advantages, adv0) and torch.equal(batch.returns, ret0)
    opt.train_epochs(batch)
    V._close(batch.advantages.cpu(), adv0.cpu(), 2e-5)
    V._close(batch.returns.cpu(), ret0.cpu(), 2e-5)


def test_prep_reads_the_coefficient_every_time(tmp_path):
    """upgo_coef assigned between preps takes effect at the next one, 0 gives back the batch without UPGO, and a
    coefficient outside its domain, or set with value heads, is refused by prep."""
    from dotaclient_b200.optimizer import REWARD_KEYS
    opt = make_optimizer(tmp_path)
    rollouts = C._mixed(opt, 2)
    b0 = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    opt.upgo_coef = 0.25
    b1 = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    assert opt.last_upgo_stats is not None and not torch.equal(b0.advantages, b1.advantages)
    opt.upgo_coef = 0.0
    b2 = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    assert opt.last_upgo_stats is None
    _fields_equal(b0, b2)
    for bad in (-1.0, float("nan"), True):
        opt.upgo_coef = bad
        with pytest.raises(ValueError, match="upgo_coef"):
            opt.batch_from_rollouts(copy.deepcopy(rollouts))
    heads = make_optimizer(tmp_path, value_heads={"win": [REWARD_KEYS[0]], "rest": list(REWARD_KEYS[1:])})
    heads.upgo_coef = 0.5
    with pytest.raises(ValueError, match="value_heads"):
        heads.batch_from_rollouts(copy.deepcopy(rollouts))


def _snapshot(opt):
    return (opt.flat.param.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.adam_steps.clone())


def test_replays_as_it_runs_eagerly_and_reports_its_metrics(tmp_path):
    """V-trace, joint ratio, the KL penalty, mask_padding + pack_sequences, 2 minibatches and both refreshes with UPGO:
    the epochs replayed from captured graphs equal the eager ones bit for bit.  Then run_iteration reports the upgo/*
    metrics of its prep, and none once the coefficient is 0."""
    from dotaclient_b200.optimizer import MessageQueue
    port = uuid.uuid4().int % 100000
    kw = dict(mask_padding=True, pack_sequences=True, policy_ratio="joint", kl_coef=0.3, num_minibatches=2,
              recompute_advantages=True, recompute_states=True, epochs=3, min_seq=4, upgo_coef=0.5,
              advantage_estimator="vtrace")
    a = make_optimizer(tmp_path, port=port, hidden_size=256, cell="gru", lr=1e-3, **kw)
    b = make_optimizer(tmp_path, hidden_size=256, cell="gru", lr=1e-3, **kw)
    b.use_cuda_graph = False
    rollouts = PK.ragged_rollouts(a.policy_base, 9, True, True)
    ba, bb = a.batch_from_rollouts(copy.deepcopy(rollouts)), b.batch_from_rollouts(copy.deepcopy(rollouts))
    assert torch.equal(ba.advantages, bb.advantages)
    for rep in range(2):                             # the second pass replays every minibatch shape
        ra, rb = a.train_epochs(ba), b.train_epochs(bb)
        assert [dict(s) for s in ra[3]] == [dict(s) for s in rb[3]], rep
        assert all(torch.equal(x, y) for x, y in zip(_snapshot(a), _snapshot(b))), rep
        assert torch.equal(ba.advantages, bb.advantages)
    assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"
    # run_iteration on GAE rollouts from the queue
    c = make_optimizer(tmp_path, port=port + 1, upgo_coef=0.5, min_seq=4)
    actor = MessageQueue(host="upgo", port=port + 1, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for it in range(2):
        for i, L in enumerate((40, 23, 57)):
            actor.publish_experience(pickle.dumps(make_rollout(L, 870 + 10 * it + i, game_id=i, weight_version=1)))
    m = c.run_iteration(1)
    assert m["upgo/coef"] == 0.5 and 0 < m["upgo/through_fraction"] < 1 and np.isfinite(m["upgo/mean_advantage"])
    c.upgo_coef = 0.0
    m = c.run_iteration(2)
    assert not any(k.startswith("upgo/") for k in m)
