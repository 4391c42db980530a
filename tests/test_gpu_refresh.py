"""GPU tests of the advantage refresh between PPO epochs (``DotaOptimizer(recompute_advantages=True)``): the indexed scans
bitwise against the existing ones on the identity layout and against float64 numpy on a shuffled packed layout at 131,072
tokens; the refresh at unchanged weights; the refresh against the float64 oracle (``refresh_oracle.py``) with cut
rollouts, padding masks, packing, PopArt and V-trace; whole iterations against the oracle; packed against unpacked, eager
against replayed, the KL early stop, and two ranks."""
import copy
import os
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refresh_oracle as RF  # noqa: E402
import test_gpu_continuation as C  # noqa: E402
import test_gpu_parity as P  # noqa: E402
import test_gpu_vtrace as V  # noqa: E402
from stacked_oracle import StackedRefPolicy  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
N_C2 = 131072


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=16, epochs=3, min_seq=1, lr=5e-5, port=None, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="refresh", rmq_port=port if port is not None else uuid.uuid4().int % 100000,
                         epochs=epochs, min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=lr, checkpoint=False,
                         pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5,
                         run_local=True, hidden_size=hidden_size, cell=cell, **kw)


# ------------------------------------------------------------------------------------------------ kernels
def _scan_inputs(lengths, seed, terminal=None):
    from dotaclient_b200.optimizer import rollout_segments
    g = np.random.default_rng(seed)
    S = 16
    terminal = [True] * len(lengths) if terminal is None else terminal
    seg, boot_src, valid_len = rollout_segments(lengths, terminal, S, True)
    n = int(seg[-1])
    n_cut = sum(not t for t in terminal)
    boot_cut = g.standard_normal(n_cut).astype(np.float32)
    boot = np.where(boot_src >= 0, boot_cut[np.maximum(boot_src, 0)], 0.0).astype(np.float32)
    return dict(seg=seg, boot=boot, valid_len=valid_len, n=n,
                rewards=(g.standard_normal((n, 10)) * 0.1).astype(np.float32),
                values=g.standard_normal(n).astype(np.float32),
                lt=(-np.abs(g.standard_normal((n, 5))) * 0.5).astype(np.float32),
                lb=(-np.abs(g.standard_normal((n, 5))) * 0.5).astype(np.float32))


@pytest.mark.parametrize("ld", [1, 128])
def test_identity_layout_equals_the_existing_scans_bitwise(ld):
    from dotaclient_b200 import ops
    d = P.dev()
    lengths = [1, 15, 16, 17, 31, 33, 64, 517, 1380, 2, 7]
    x = _scan_inputs(lengths, 3, terminal=[i % 3 != 0 for i in range(len(lengths))])
    n = x["n"]
    T = lambda a: torch.from_numpy(a).to(d)             # noqa: E731
    rew, seg, boot, vl = T(x["rewards"]), T(x["seg"]), T(x["boot"]), T(x["valid_len"])
    store = torch.zeros(n, ld, device=d)
    store[:, 0] = T(x["values"])
    values = store[:, 0]                                 # a column at a stride of ld
    tok = torch.arange(n, device=d)
    a0, r0 = ops.gae_scan(rew, T(x["values"]), seg, 0.98, 0.97, boot_value=boot, boot_reward=boot)
    a1, r1 = torch.full((n,), 7.0, device=d), torch.full((n,), 7.0, device=d)
    ops.gae_scan_indexed(rew, values, tok, seg, a1, r1, 0.98, 0.97, boot_value=boot, boot_reward=boot)
    assert torch.equal(a0, a1) and torch.equal(r0, r1)
    for clips in ((1.0, 1.0), (2.0, 0.5)):
        p0, v0 = ops.vtrace_scan(rew, T(x["values"]), T(x["lt"]), T(x["lb"]), seg, 0.98, 0.97, *clips, boot_value=boot,
                                 valid_len=vl)
        p1, v1 = torch.full((n,), 7.0, device=d), torch.full((n,), 7.0, device=d)
        ops.vtrace_scan_indexed(rew, values, T(x["lt"]), T(x["lb"]), tok, seg, p1, v1, 0.98, 0.97, *clips, boot_value=boot,
                                valid_len=vl)
        assert torch.equal(p0, p1) and torch.equal(v0, v1)


def _float64_scans(x, tok_np, values_tok, lt_tok, estimator):
    """Per segment, in float64, reading values and target log-probs at each row's token (0 where tok < 0)."""
    held = tok_np >= 0
    v = np.where(held, values_tok[np.maximum(tok_np, 0)], 0.0)
    lt = np.where(held[:, None], lt_tok[np.maximum(tok_np, 0)], 0.0)
    adv, ret = np.zeros(x["n"]), np.zeros(x["n"])
    for s in range(len(x["seg"]) - 1):
        lo, hi = int(x["seg"][s]), int(x["seg"][s + 1])
        if hi <= lo:
            continue
        if estimator == "gae":
            adv[lo:hi], ret[lo:hi] = RF.gae(x["rewards"][lo:hi], v[lo:hi], 0.98, 0.97, x["boot"][s])
        else:
            logrho = RF.VT.log_rho(lt[lo:hi], x["lb"][lo:hi])
            adv[lo:hi], ret[lo:hi] = RF.VT.vtrace(x["rewards"][lo:hi], v[lo:hi], logrho, 0.98, 0.97, 1.0, 1.0, x["boot"][s])
    return adv, ret


@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
def test_shuffled_packed_layout_vs_float64(estimator):
    """Ragged rollouts (some cut) packed at S = 16, the tokens then shuffled: 131,072 tokens.  Rows of tokens that hold
    no row are left untouched."""
    from dotaclient_b200 import ops
    from dotaclient_b200.optimizer import refresh_token_map, sequence_count
    g = np.random.default_rng(5)
    S, lengths = 16, []
    while sequence_count(lengths, S, pack=True) * S < N_C2 - 300:
        lengths.append(int(g.integers(1, 300)))
    B = N_C2 // S
    terminal = [bool(g.random() < 0.7) for _ in lengths]
    x = _scan_inputs(lengths, 6, terminal)
    perm = g.permutation(N_C2)
    tok_np = refresh_token_map(lengths, S, True, True)
    assert sequence_count(lengths, S, pack=True) <= B
    tok_np = np.where(tok_np >= 0, perm[np.maximum(tok_np, 0)], -1)
    values_tok = g.standard_normal(N_C2).astype(np.float32)
    lt_tok = (-np.abs(g.standard_normal((N_C2, 5))) * 0.5).astype(np.float32)
    d = P.dev()
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(d)     # noqa: E731
    adv = torch.full((S, B), 3.25, device=d)
    ret = torch.full((S, B), -3.25, device=d)
    packed = torch.zeros(S, B, 128, device=d)
    packed[..., 25] = T(values_tok).view(S, B)
    if estimator == "gae":
        ops.gae_scan_indexed(T(x["rewards"]), packed[..., 25], T(tok_np), T(x["seg"]), adv, ret, 0.98, 0.97,
                             boot_value=T(x["boot"]), boot_reward=T(x["boot"]))
    else:
        ops.vtrace_scan_indexed(T(x["rewards"]), packed[..., 25], T(lt_tok), T(x["lb"]), T(tok_np), T(x["seg"]), adv, ret,
                                0.98, 0.97, 1.0, 1.0, boot_value=T(x["boot"]), valid_len=T(x["valid_len"]))
    a, r = adv.reshape(-1).cpu().numpy(), ret.reshape(-1).cpu().numpy()
    want_a, want_r = _float64_scans(x, tok_np, values_tok, lt_tok, estimator)
    held = tok_np >= 0
    V._close(a[tok_np[held]], want_a[held], 1e-5)
    V._close(r[tok_np[held]], want_r[held], 1e-5)
    free = np.ones(N_C2, bool)
    free[tok_np[held]] = False
    assert free.sum() == N_C2 - held.sum() > 0
    assert (a[free] == 3.25).all() and (r[free] == -3.25).all()


# ------------------------------------------------------------------------------------------------ the refresh
def _rows(batch, values):
    """A [S, B] batch tensor at prep's rollout-major rows (0 where no token holds the row)."""
    tok = batch.refresh.tok
    flat = values.reshape(-1)
    return torch.where(tok >= 0, flat[tok.clamp(min=0)], torch.zeros_like(flat[:1])).cpu().numpy()


def _mixed(opt, seed, vtrace):
    return C._mixed(opt, seed, behaviour=vtrace)


@pytest.mark.parametrize("estimator,pack", [("gae", False), ("gae", True), ("vtrace", False), ("vtrace", True)])
def test_refresh_at_unchanged_weights_is_prep(estimator, pack, tmp_path):
    """learning_rate = 0, epochs = 2: the refresh forward runs at another batch shape than prep's, so the bits may differ;
    the values agree to fp32 rounding."""
    opt = make_optimizer(tmp_path, epochs=2, lr=0.0, recompute_advantages=True, mask_padding=True, pack_sequences=pack,
                         advantage_estimator=estimator)
    batch = opt.batch_from_rollouts(_mixed(opt, 1, estimator == "vtrace"))
    adv0, ret0 = batch.advantages.clone(), batch.returns.clone()
    calls = []
    real = opt._refresh_advantages
    opt._refresh_advantages = lambda b: (calls.append(1), real(b))
    opt.train_epochs(batch)
    assert len(calls) == 1
    da = float((batch.advantages - adv0).abs().max())
    dr = float((batch.returns - ret0).abs().max())
    print("largest difference at unchanged weights: advantages %.3g, returns %.3g" % (da, dr))
    V._close(batch.advantages.cpu(), adv0.cpu(), 2e-5)
    V._close(batch.returns.cpu(), ret0.cpu(), 2e-5)
    assert (batch.advantages[~batch.valid] == 0).all() and (batch.returns[~batch.valid] == 0).all()


REFRESH_CONFIGS = {
    "gae": dict(),
    "gae_masked": dict(mask_padding=True),
    "gae_packed_popart": dict(mask_padding=True, pack_sequences=True, value_norm=True),
    "vtrace": dict(advantage_estimator="vtrace"),
    "vtrace_packed": dict(advantage_estimator="vtrace", mask_padding=True, pack_sequences=True),
    "vtrace_masked_popart_gru": dict(advantage_estimator="vtrace", mask_padding=True, value_norm=True, hidden_size=256,
                                     cell="gru"),
}


@pytest.mark.parametrize("name", sorted(REFRESH_CONFIGS))
def test_refresh_vs_float64_oracle(name, tmp_path):
    """After two steps at a large learning rate, the refresh against the oracle run from the same weights, chunk by chunk
    from the batch's stored states, with prep's bootstraps of the cut rollouts."""
    from dotaclient_b200.optimizer import rollout_segments
    torch.set_num_threads(8)
    kw = dict(REFRESH_CONFIGS[name])
    H, cell = kw.pop("hidden_size", 128), kw.pop("cell", "lstm")
    S = 16
    opt = make_optimizer(tmp_path, hidden_size=H, cell=cell, epochs=2, lr=2e-3, recompute_advantages=True, **kw)
    vtrace = kw.get("advantage_estimator") == "vtrace"
    rollouts = _mixed(opt, 2, vtrace)
    if kw.get("value_norm"):
        rollouts = [dict(r, rewards=(np.asarray(r["rewards"]) * 25.0 + 4.0).astype(np.float32)) for r in rollouts]
    batch = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    prep_adv = _rows(batch, batch.advantages)
    prep_pol = copy.deepcopy(opt.policy_base)          # the weights the batch's chunk states were computed with
    for _ in range(2):
        opt.train(batch)
    opt._refresh_advantages(batch)
    got_a, got_r = _rows(batch, batch.advantages), _rows(batch, batch.returns)
    # the oracle: the same weights in float64, the unpacked chunks of each rollout from prep's states
    ref = StackedRefPolicy(H, cell, 1)
    ref.load_state_dict({k: v.detach().cpu() for k, v in opt.policy_base.state_dict().items()})
    pol64 = ref.double()
    mu, sigma = opt._value_norm_moments() if opt.value_norm else (0.0, 1.0)
    Ls = [int(r["rewards"].shape[0]) for r in rollouts]
    terminal = [bool(r.get("terminal", True)) for r in rollouts]
    seg, _, _ = rollout_segments(Ls, terminal, S, opt.mask_padding)
    boot = batch.refresh.boot.cpu().numpy() if batch.refresh.boot is not None else np.zeros(len(seg) - 1, np.float32)
    seg_boot = dict(zip(seg[:-1].tolist(), boot.tolist()))
    want_a, want_r, base = [], [], 0
    for i, r in enumerate(rollouts):
        L = Ls[i]
        Lp = (L + S - 1) // S * S
        chunks = []
        for j in range(Lp // S):
            sl = slice(j * S, min((j + 1) * S, L))
            pad = S - (sl.stop - sl.start)
            padt = lambda t: torch.cat([t[sl], torch.zeros((pad,) + tuple(t.shape[1:]), dtype=t.dtype)])  # noqa: E731
            st = opt.policy_base.init_hidden()
            if j == 0 and "initial_hidden" in r:
                st = r["initial_hidden"]
            elif j > 0:
                st = C._learner_state(prep_pol, r, j * S, r.get("initial_hidden"))[0]
            chunks.append(({k: padt(torch.as_tensor(v)[:L]) for k, v in r["observations"].items()},
                           {k: padt(torch.as_tensor(v)) for k, v in r["masks"].items()},
                           {k: padt(torch.as_tensor(v)) for k, v in r["actions"].items()}, st))
        a, q = RF.refresh_rollout(pol64, chunks, r["rewards"], L, estimator="vtrace" if vtrace else "gae", gamma=0.98,
                                  lam=0.97, mask_padding=opt.mask_padding, terminal=terminal[i],
                                  boot=seg_boot.get(base, 0.0), behaviour=r.get("behaviour_logp"), mu=mu, sigma=sigma)
        want_a.append(a)
        want_r.append(q)
        base += Lp
    want_a, want_r = np.concatenate(want_a), np.concatenate(want_r)
    held = batch.refresh.tok.cpu().numpy() >= 0
    scale = max(1.0, float(np.abs(want_r).max()))
    V._close(got_a[held] / scale, want_a[held] / scale, 3e-4)
    V._close(got_r[held] / scale, want_r[held] / scale, 3e-4)
    # the refresh is not prep: two large steps moved the critic well past the tolerance
    assert np.abs(prep_adv[held] - want_a[held]).max() / scale > 1e-3


ITER_CONFIGS = {
    "gae_m1_lstm": dict(M=1),
    "gae_m2_lstm_masked": dict(M=2, mask_padding=True),
    "vtrace_m2_gru_masked": dict(M=2, mask_padding=True, advantage_estimator="vtrace", hidden_size=256, cell="gru"),
    "vtrace_m1_lstm_popart": dict(M=1, advantage_estimator="vtrace", value_norm=True),
    "gae_m1_gru_masked_popart": dict(M=1, mask_padding=True, value_norm=True, hidden_size=256, cell="gru"),
    # rollouts cut from a longer game: non-zero initial states, and prep's V(s_L) bootstraps kept by every refresh
    "gae_m2_lstm_cut": dict(M=2, cut=True),
    "gae_m1_gru_cut_masked": dict(M=1, cut=True, mask_padding=True, hidden_size=256, cell="gru"),
    # kl_stop ends the iteration at its third step, after two refreshes, and no refresh follows
    "gae_m1_lstm_masked_kl_stop": dict(M=1, mask_padding=True, kl_stop=True, epochs=4),
}


def _kl_limit(tmp_path, H, cell, rollouts, epochs, **kw):
    """A limit between the all-ranks KL of the second and the third step of an iteration run without a stop, so that the
    third step is the one the limit stops."""
    probe = make_optimizer(tmp_path, hidden_size=H, cell=cell, epochs=epochs, min_seq=2, recompute_advantages=True,
                           kl_stop=1e9, **kw)
    stats = probe.train_epochs(probe.batch_from_rollouts(copy.deepcopy(rollouts)))[3]
    kl = [st["kl_all_ranks"] for st in stats]
    assert 0 < 2 * kl[1] < kl[2], kl
    return float(np.sqrt(kl[1] * kl[2]))


@pytest.mark.parametrize("name", sorted(ITER_CONFIGS))
def test_iteration_vs_oracle(name, tmp_path):
    """One iteration of 3 epochs (4 under kl_stop): per-step losses and gradient norms, the final advantages, weights and
    Adam moments, at the whole-step tests' tolerances."""
    torch.set_num_threads(8)
    kw = dict(ITER_CONFIGS[name])
    M, H, cell = kw.pop("M"), kw.pop("hidden_size", 128), kw.pop("cell", "lstm")
    cut, kl_stop, epochs = kw.pop("cut", False), kw.pop("kl_stop", False), kw.pop("epochs", 3)
    S = 16
    probe = make_optimizer(tmp_path, hidden_size=H, cell=cell)          # the same seeded weights, for the rollouts only
    if cut:
        rollouts = C._mixed(probe, 5)
    else:
        rollouts = [make_rollout(L, 700 + i) for i, L in enumerate((40, 23, 48, 7))]
    if kw.get("value_norm"):
        rollouts = [dict(r, rewards=(np.asarray(r["rewards"]) * 25.0 + 4.0).astype(np.float32)) for r in rollouts]
    if kw.get("advantage_estimator") == "vtrace":
        rollouts = V._stale_behaviour(probe, rollouts, 30)
    limit = _kl_limit(tmp_path, H, cell, rollouts, epochs, **kw) if kl_stop else None
    mine = make_optimizer(tmp_path, hidden_size=H, cell=cell, epochs=epochs, min_seq=2, num_minibatches=M,
                          recompute_advantages=True, value_norm_decay=0.9, kl_stop=limit, **kw)
    refreshes = []
    real = mine._refresh_advantages
    mine._refresh_advantages = lambda b: (refreshes.append(1), real(b))
    torch.manual_seed(7)
    oracle = RF.RefreshRefOptimizer(StackedRefPolicy(H, cell, 1), seq_len=S, decay=0.9,
                                    estimator=kw.get("advantage_estimator", "gae"),
                                    mask_padding=kw.get("mask_padding", False), value_norm=kw.get("value_norm", False),
                                    kl_stop=limit)
    batch = mine.batch_from_rollouts(copy.deepcopy(rollouts))
    xs_o = oracle.prepare(copy.deepcopy(rollouts))
    rng = copy.deepcopy(mine.minibatch_rng)
    lm, em, gm, _ = mine.train_epochs(batch)
    res = oracle.train_epochs(xs_o, rollouts, epochs, M, rng)
    if kl_stop:
        assert len(lm) == len(res) == 3 and res[-1][2] is None and mine.last_kl_updates == (2, 2)
        assert len(refreshes) == 2
    else:
        assert len(lm) == len(res) == epochs * M and len(refreshes) == epochs - 1
    for step, (lo, eo, go) in enumerate(res):
        for k in lo:
            np.testing.assert_allclose(float(lm[step][k]), float(lo[k]), rtol=2e-4, atol=2e-6, err_msg="%s %d" % (k, step))
        if go is not None:
            np.testing.assert_allclose(float(gm[step]["unclipped"]), float(go["unclipped"]), rtol=2e-3)
    adv_o = np.concatenate([s.advantages.numpy() for s in xs_o])
    ret_o = np.concatenate([s.returns.numpy() for s in xs_o])
    V._close(batch.advantages.t().reshape(-1).cpu(), adv_o, 2e-4)
    V._close(batch.returns.t().reshape(-1).cpu(), ret_o, 2e-4)
    # Adam steps of lr 5e-5: a parameter can differ by up to one step's size per step where its gradient is ~0
    for name_, p in oracle.policy_base.named_parameters():
        mp = dict(mine.policy_base.named_parameters())[name_].detach().cpu()
        torch.testing.assert_close(mp, p.detach(), rtol=1e-4, atol=1e-4 + 5e-5 * len(res), msg=name_)
    sd = mine.optimizer.state_dict()["state"]
    want = P._adam_state_by_name(oracle)
    names = [n for n, _ in oracle.policy_base.named_parameters()]
    for i, st in sd.items():
        w = want[names[i]]
        assert float(st["step"]) == float(w["step"])
        torch.testing.assert_close(st["exp_avg"], w["exp_avg"], rtol=2e-3,
                                   atol=2e-3 * float(w["exp_avg"].abs().max()) + 1e-12)
        torch.testing.assert_close(st["exp_avg_sq"], w["exp_avg_sq"], rtol=4e-3,
                                   atol=4e-3 * float(w["exp_avg_sq"].abs().max()) + 1e-20)


# ------------------------------------------------------------------------------------------------ equivalences
def test_packed_equals_unpacked(tmp_path):
    from dotaclient_b200.optimizer import refresh_token_map  # noqa: F401
    out = []
    for pack in (False, True):
        opt = make_optimizer(tmp_path, epochs=3, recompute_advantages=True, mask_padding=True, pack_sequences=pack)
        batch = opt.batch_from_rollouts(_mixed(opt, 3, False))
        opt.train_epochs(batch)
        out.append((_rows(batch, batch.advantages), _rows(batch, batch.returns), opt.flat.param.detach().cpu()))
    (a0, r0, p0), (a1, r1, p1) = out
    V._close(a1, a0, 1e-5)
    V._close(r1, r0, 1e-5)
    torch.testing.assert_close(p1, p0, rtol=1e-5, atol=1e-6)


def test_eager_equals_replayed(tmp_path):
    out = []
    for graphs in (False, True):
        opt = make_optimizer(tmp_path, epochs=4, recompute_advantages=True, mask_padding=True)
        opt.use_cuda_graph = graphs
        batch = opt.batch_from_rollouts(_mixed(opt, 4, False))
        losses = opt.train_epochs(batch)[0]
        out.append(([[float(v) for v in l.values()] for l in losses], batch.advantages.clone(),
                    opt.flat.param.detach().clone()))
        if graphs:
            assert any(isinstance(v, tuple) for v in opt._graphs.values())
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][2], out[1][2])


@pytest.mark.parametrize("kl_stop", [1e-30, 1e9])
def test_no_refresh_after_a_kl_stop(kl_stop, tmp_path):
    """One refresh before every epoch that starts after the first: none after the step that stopped the iteration."""
    opt = make_optimizer(tmp_path, epochs=3, lr=1e-3, recompute_advantages=True, kl_stop=kl_stop)
    batch = opt.batch_from_rollouts([make_rollout(L, 90 + i) for i, L in enumerate((40, 23))])
    calls = []
    real = opt._refresh_advantages
    opt._refresh_advantages = lambda b: (calls.append(1), real(b))
    losses = opt.train_epochs(batch)[0]
    assert len(calls) == len(losses) - 1
    run, skipped = opt.last_kl_updates
    assert (skipped > 0 and len(losses) < 3) if kl_stop < 1 else (skipped == 0 and len(losses) == 3)


def test_feature_off_attaches_nothing_and_epoch_one_does_nothing(tmp_path):
    off = make_optimizer(tmp_path)
    assert off.batch_from_rollouts([make_rollout(40, 1)]).refresh is None
    one = make_optimizer(tmp_path, epochs=1, recompute_advantages=True)
    batch = one.batch_from_rollouts([make_rollout(40, 1)])
    adv = batch.advantages.clone()
    one.train_epochs(batch)
    assert torch.equal(batch.advantages, adv)


@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
def test_refresh_in_time_blocks_equals_one_block(estimator, tmp_path):
    """The refresh forward over blocks of 3 time steps (the state carried across blocks, resets of a packed batch inside
    them) gives the advantages of one forward over the whole batch, at a fraction of its transient memory."""
    opt = make_optimizer(tmp_path, epochs=2, lr=1e-3, recompute_advantages=True, mask_padding=True, pack_sequences=True,
                         advantage_estimator=estimator)
    extra = [make_rollout(L, 60 + L) for L in (5, 9, 3)]
    if estimator == "vtrace":
        extra = V._stale_behaviour(opt, extra, 7)
    batch = opt.batch_from_rollouts(_mixed(opt, 6, estimator == "vtrace") + extra)
    assert batch.reset_slot is not None and int((batch.reset_slot >= 0).sum()) > 0
    opt.train(batch)
    out = {}
    for tokens in (10 ** 9, 3 * batch.batch_size):
        opt.REFRESH_CHUNK_TOKENS = tokens
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        opt._refresh_advantages(batch)
        torch.cuda.synchronize()
        out[tokens] = (batch.advantages.clone(), batch.returns.clone(), torch.cuda.max_memory_allocated() - base)
    (a0, r0, m0), (a1, r1, m1) = out[10 ** 9], out[3 * batch.batch_size]
    V._close(a1.cpu(), a0.cpu(), 1e-6)
    V._close(r1.cpu(), r0.cpu(), 1e-6)
    assert m1 < m0, (m1, m0)


def test_refresh_keeps_peak_memory_below_a_step(tmp_path):
    """The refresh forward keeps no activations: its peak is below that of a training step on the same batch."""
    opt = make_optimizer(tmp_path, epochs=2, recompute_advantages=True)
    batch = opt.batch_from_rollouts([make_rollout(L, 40 + i) for i, L in enumerate((512, 300, 211))])
    opt.train(batch)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    opt._refresh_advantages(batch)
    torch.cuda.synchronize()
    refresh_peak = torch.cuda.max_memory_allocated() - base
    torch.cuda.reset_peak_memory_stats()
    opt.use_cuda_graph = False
    opt.train(batch)
    torch.cuda.synchronize()
    step_peak = torch.cuda.max_memory_allocated() - base
    print("peak above the resident state: refresh %.1f MB, step %.1f MB" % (refresh_peak / 2**20, step_peak / 2**20))
    assert refresh_peak < step_peak


# ------------------------------------------------------------------------------------------------ two ranks
def _check_two_ranks(got):
    import refresh_multi_rank as RM
    a, b = got
    assert a["sizes"] != b["sizes"]                                       # different batches on the two ranks
    for rec in got:                                                       # every rank refreshed its own batch
        assert rec["refreshes"] == [s for s in rec["sizes"] for _ in range(RM.EPOCHS - 1)]
    assert int(a["steps"].max()) == RM.ITERATIONS * RM.EPOCHS * 2
    assert torch.equal(a["steps"], b["steps"])
    assert torch.equal(a["param"], b["param"]) and torch.equal(a["exp_avg"], b["exp_avg"])    # replicas bit-identical


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_nccl_stay_in_sync(tmp_path):
    import refresh_multi_rank as RM
    _check_two_ranks(RM.run(tmp_path, "nccl"))


def test_two_ranks_gloo_one_gpu_stay_in_sync(tmp_path):
    import refresh_multi_rank as RM
    _check_two_ranks(RM.run(tmp_path, "gloo"))
