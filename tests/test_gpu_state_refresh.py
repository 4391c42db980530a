"""GPU tests of the state refresh between PPO epochs (``DotaOptimizer(recompute_states=True)``): the refresh at unchanged
weights against prep, bitwise, in one time block and in blocks of 3 steps; the refreshed states (and, with
``recompute_advantages``, advantages and returns) after two large steps against the float64 oracle
(``state_refresh_oracle.py``); the drift against float64 torch; ``dc_refresh_states`` and the fill gather at the
benchmark's shapes against torch indexing; packed against unpacked, eager against replayed, the KL early stop, peak memory,
and two ranks."""
import copy
import os
import sys
import types
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import state_refresh_oracle as SO  # noqa: E402
import test_gpu_continuation as C  # noqa: E402
import test_gpu_parity as P  # noqa: E402
import test_gpu_vtrace as V  # noqa: E402
from stacked_oracle import StackedRefPolicy  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=16, epochs=3, min_seq=1, lr=5e-5, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="staterefresh", rmq_port=uuid.uuid4().int % 100000, epochs=epochs,
                         min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=lr, checkpoint=False,
                         pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5,
                         run_local=True, hidden_size=hidden_size, cell=cell, **kw)


def _states(batch):
    return [t.clone() for t in (batch.h0, batch.c0, batch.reset_h, batch.reset_c) if t is not None]


def _snapshot(batch):
    """A copy of the batch's recurrent start states, in a form ``_dest_state`` reads."""
    clone = lambda t: None if t is None else t.clone()          # noqa: E731
    return types.SimpleNamespace(batch_size=batch.batch_size, h0=clone(batch.h0), c0=clone(batch.c0),
                                 reset_h=clone(batch.reset_h), reset_c=clone(batch.reset_c))


def _rollouts(opt, seed, vtrace=False, extra=True):
    """Cut and terminal rollouts with initial states, plus short ones whose tails share packed columns."""
    rs = C._mixed(opt, seed, behaviour=vtrace, lengths=(40, 23, 48, 7, 37), terminal=(False, True, False, True, False))
    if extra:
        more = [make_rollout(L, 60 + L + seed) for L in (5, 9, 3, 21)]
        rs += V._stale_behaviour(opt, more, 7) if vtrace else more
    return rs


def _dest_state(batch, layer, H, slot):
    """Layer ``layer``'s (h, c) at destination ``slot`` of the batch (h0 column, or reset-table row)."""
    B = batch.batch_size
    if slot < B:
        return batch.h0[layer, slot], (None if batch.c0 is None else batch.c0[layer, slot])
    row = slot - B
    h = batch.reset_h.view(-1, batch.reset_h.shape[2])[row, layer * H:(layer + 1) * H]
    c = None if batch.reset_c is None else batch.reset_c.view(-1, batch.reset_c.shape[2])[row, layer * H:(layer + 1) * H]
    return h, c


CELLS = [("lstm", 128, 1, False), ("lstm", 128, 1, True), ("gru", 256, 1, True), ("lstm", 128, 2, True),
         ("gru", 256, 2, False)]


@pytest.mark.parametrize("cell,H,layers,pack", CELLS)
def test_unchanged_weights_reproduce_prep_bitwise(cell, H, layers, pack, tmp_path):
    """learning_rate = 0: the refresh forward is prep's, at prep's shape in one time block, so every state it writes is
    prep's bit for bit and the drift is exactly 0, and so are they in blocks of 3 steps."""
    opt = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers, epochs=2, lr=0.0, recompute_states=True,
                         mask_padding=True, pack_sequences=pack)
    batch = opt.batch_from_rollouts(_rollouts(opt, 1))
    before = _states(batch)
    assert batch.state_refresh.layout.step.size > 0
    opt.train_epochs(batch)
    st = opt.last_state_refresh_stats
    assert st["drift"] == 0.0 and st["states"] == batch.state_refresh.layout.step.size
    for a, b in zip(_states(batch), before):
        assert torch.equal(a, b)
    opt.REFRESH_CHUNK_TOKENS = 3 * batch.state_refresh.layout.R
    opt._refresh_states(batch)
    for a, b in zip(_states(batch), before):
        assert torch.equal(a, b)
    assert opt.last_state_refresh_stats["drift"] == 0.0


STATE_CONFIGS = {
    "lstm128_unpacked": dict(),
    "lstm128_packed_masked": dict(mask_padding=True, pack_sequences=True),
    "gru256_packed_masked": dict(mask_padding=True, pack_sequences=True, hidden_size=256, cell="gru"),
    "lstm128_2layer_packed": dict(mask_padding=True, pack_sequences=True, num_layers=2),
    "gae_adv_lstm_unpacked": dict(recompute_advantages=True),
    "gae_adv_packed_popart": dict(recompute_advantages=True, mask_padding=True, pack_sequences=True, value_norm=True),
    "vtrace_adv_masked_gru": dict(recompute_advantages=True, advantage_estimator="vtrace", mask_padding=True,
                                  hidden_size=256, cell="gru"),
    "vtrace_adv_packed_popart_2layer": dict(recompute_advantages=True, advantage_estimator="vtrace", mask_padding=True,
                                            pack_sequences=True, value_norm=True, num_layers=2),
}


@pytest.mark.parametrize("name", sorted(STATE_CONFIGS))
def test_refresh_vs_float64_oracle(name, tmp_path):
    """After two steps at a large learning rate: every refreshed state against the oracle's whole-rollout rerun, the drift
    against float64 torch on the states it replaced, and with recompute_advantages the advantages and returns against the
    oracle's scan from its refreshed states and bootstraps."""
    torch.set_num_threads(8)
    kw = dict(STATE_CONFIGS[name])
    H, cell, layers = kw.pop("hidden_size", 128), kw.pop("cell", "lstm"), kw.pop("num_layers", 1)
    S = 16
    opt = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers, epochs=2, lr=2e-3, recompute_states=True,
                         **kw)
    vtrace = kw.get("advantage_estimator") == "vtrace"
    rollouts = _rollouts(opt, 2, vtrace)
    if kw.get("value_norm"):
        rollouts = [dict(r, rewards=(np.asarray(r["rewards"]) * 25.0 + 4.0).astype(np.float32)) for r in rollouts]
    batch = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    for _ in range(2):
        opt.train(batch)
    old = _snapshot(batch)
    opt._refresh_states(batch)
    ref = StackedRefPolicy(H, cell, layers)
    ref.load_state_dict({k: v.detach().cpu() for k, v in opt.policy_base.state_dict().items()})
    pol64 = ref.double()
    lay = batch.state_refresh.layout
    worst, moved = 0.0, 0.0
    per_rollout = {}
    for i, r in enumerate(rollouts):
        start = r.get("initial_hidden", opt.policy_base.init_hidden())
        per_rollout[i] = SO.rollout_states(pol64, r, S, start)[0]
    for step, i, slot in zip(lay.step, lay.rollout, lay.slot):
        want = per_rollout[int(i)][int(step) // S]
        want_h, want_c = (want if cell == "lstm" else (want, None))
        for layer in range(layers):
            h, c = _dest_state(batch, layer, H, int(slot))
            pairs = [(h, want_h[layer, 0])] + ([(c, want_c[layer, 0])] if cell == "lstm" else [])
            for g, w in pairs:
                err = float((g.double().cpu() - w).abs().max()) / max(1.0, float(w.abs().max()))
                worst = max(worst, err)
    print("largest state error against float64: %.3g" % worst)
    assert worst <= 3e-4
    # the drift: float64 torch over the states the refresh replaced (every element it wrote)
    d = opt.last_state_refresh_stats["drift"]
    new_v, old_v = [], []
    for slot in lay.slot:
        for layer in range(layers):
            new_v += [t for t in _dest_state(batch, layer, H, int(slot)) if t is not None]
            old_v += [t for t in _dest_state(old, layer, H, int(slot)) if t is not None]
    want_d = SO.drift(new_v, old_v)
    moved = want_d
    assert abs(d - want_d) <= 1e-9 * max(want_d, 1e-30) + 1e-15, (d, want_d)
    assert moved > 1e-4                                          # two large steps moved the states
    if not kw.get("recompute_advantages"):
        return
    mu, sigma = opt._value_norm_moments() if opt.value_norm else (0.0, 1.0)
    want_a, want_r = [], []
    for i, r in enumerate(rollouts):
        a, q = SO.refreshed_advantages(pol64, r, S, r.get("initial_hidden", opt.policy_base.init_hidden()),
                                       estimator="vtrace" if vtrace else "gae", mask_padding=opt.mask_padding, mu=mu,
                                       sigma=sigma)
        want_a.append(a)
        want_r.append(q)
    want_a, want_r = np.concatenate(want_a), np.concatenate(want_r)
    tok = batch.refresh.tok.cpu().numpy()
    held = tok >= 0
    got_a = batch.advantages.reshape(-1).cpu().numpy()[tok[held]]
    got_r = batch.returns.reshape(-1).cpu().numpy()[tok[held]]
    scale = max(1.0, float(np.abs(want_r).max()))
    V._close(got_a / scale, want_a[held] / scale, 3e-4)
    V._close(got_r / scale, want_r[held] / scale, 3e-4)


# ------------------------------------------------------------------------------------------------ kernels at bench shapes
# name -> (cell, H, R rollouts, padded length): C2 is bench's 256 rollouts of 512 steps (LSTM-128), the stream shape 64
# rollouts of 256 steps cut into 1024 sequences of 16 (GRU-256)
KERNEL_SHAPES = {"c2": ("lstm", 128, 256, 512, 512), "stream": ("gru", 256, 64, 256, 16)}


@pytest.mark.parametrize("shape", sorted(KERNEL_SHAPES))
def test_kernels_bitwise_against_torch_indexing(shape):
    """``dc_refresh_states`` writes exactly the state-buffer rows torch indexing reads (h0 columns and reset rows), leaves
    every other element alone, and sums the drift as float64 torch does up to reordering; the fill gather equals torch
    indexing with zeros at -1."""
    from dotaclient_b200 import ops
    from dotaclient_b200.optimizer import DotaOptimizer
    d = P.dev()
    cell, H, R, Lp, S = KERNEL_SHAPES[shape]
    g = torch.Generator().manual_seed(5)
    T = min(Lp, max(1, DotaOptimizer.REFRESH_CHUNK_TOKENS // R))
    L = 2
    ybufs = [torch.randn((T + 1, R, H), generator=g).to(d) for _ in range(L)]
    cbufs = [torch.randn((T + 1, R, H), generator=g).to(d) for _ in range(L)] if cell == "lstm" else None
    B, K = R * Lp // S, 2
    h0 = torch.randn((L, B, H), generator=g).to(d)
    c0 = torch.randn((L, B, H), generator=g).to(d) if cell == "lstm" else None
    rh = torch.randn((K, B, L * H), generator=g).to(d)
    rc = torch.randn((K, B, L * H), generator=g).to(d) if cell == "lstm" else None
    n = min(B + K * B, 3000)
    slot = torch.randperm(B + K * B, generator=g)[:n]
    step = torch.randint(0, T + 1, (n,), generator=g)
    rollout = torch.randint(0, R, (n,), generator=g)
    want = [t.clone() for t in (h0, c0, rh, rc) if t is not None]
    acc = torch.zeros(2, dtype=torch.float64, device=d)
    ops.refresh_states(ybufs, cbufs, 0, step.to(d), rollout.to(d), slot.to(d), h0, c0, rh, rc, acc)
    w_h0, w_c0 = want[0], (want[1] if cell == "lstm" else None)
    w_rh, w_rc = (want[2], want[3]) if cell == "lstm" else (want[1], None)
    num = den = 0.0
    for k in range(n):
        s, t, i = int(slot[k]), int(step[k]), int(rollout[k])
        for layer in range(L):
            for bufs, tab0, tabr in ((ybufs, w_h0, w_rh), (cbufs, w_c0, w_rc)):
                if bufs is None:
                    continue
                dst = tab0[layer, s] if s < B else tabr.view(-1, L * H)[s - B, layer * H:(layer + 1) * H]
                new = bufs[layer][t, i]
                num += float(((new.double() - dst.double()) ** 2).sum())
                den += float((dst.double() ** 2).sum())
                dst.copy_(new)
    got = [t for t in (h0, c0, rh, rc) if t is not None]
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    s2, o2 = acc.tolist()
    assert abs(s2 - num) <= 1e-12 * num and abs(o2 - den) <= 1e-12 * den
    # the fill gather: [S, B, 40, 32]-like rows of the batch into [T, R] with -1 -> zeros
    src = torch.randn((S, B, 40, 8), generator=g).to(d)
    idx = torch.randint(-1, S * B, (T * R,), generator=g)
    out = ops.gather_rows_fill([src.view(S * B, 40, 8)], idx.to(d))[0]
    ref = torch.where((idx >= 0).to(d)[:, None, None], src.view(S * B, 40, 8)[idx.clamp(min=0).to(d)],
                      torch.zeros((), device=d))
    assert torch.equal(out, ref)
    mask = torch.rand((S, B, 9), generator=g).to(d) > 0.5
    outm = ops.gather_rows_fill([mask.view(S * B, 9)], idx.to(d))[0]
    refm = torch.where((idx >= 0).to(d)[:, None], mask.view(S * B, 9)[idx.clamp(min=0).to(d)], False)
    assert torch.equal(outm, refm)


# the benchmark's own rollouts: C2 is bench.py's 256 rollouts of 512 steps at seq_len 512 (one chunk each, so its layout
# has no chunk start after the first and the refresh replaces nothing), the stream shape tools/state_refresh_bench.py's
# 64 rollouts of 256 steps at seq_len 16
BENCH_LAYOUTS = {"c2": ("lstm", 128, 512, 512, 256), "stream": ("gru", 256, 16, 256, 64)}


@pytest.mark.parametrize("shape", sorted(BENCH_LAYOUTS))
def test_kernels_with_the_benchmark_layouts(shape, tmp_path):
    """Every time block of a refresh over the benchmark's own batch, with the layout tables ``batch_from_rollouts``
    made: the fill gather of every input equals torch indexing with zeros at -1, and ``dc_refresh_states`` writes exactly
    the state-buffer rows torch indexing reads into the h0 columns (bitwise)."""
    from dotaclient_b200 import ops
    from dotaclient_b200.policy import Policy
    from dotaclient_b200.synthetic import rollout_seed
    cell, H, S, L, R = BENCH_LAYOUTS[shape]
    opt = make_optimizer(tmp_path, hidden_size=H, cell=cell, seq_len=S, epochs=2, recompute_states=True)
    if shape == "c2":
        rollouts = [make_rollout(L, rollout_seed(0, i)) for i in range(R)]
    else:
        rollouts = [make_rollout(L, 1000 + i) for i in range(R)]
    batch = opt.batch_from_rollouts(rollouts)
    del rollouts
    st = batch.state_refresh
    lay = st.layout
    assert lay.R == R and lay.L_max == L
    assert lay.step.size == (0 if shape == "c2" else R * (L // S - 1))
    lstm = cell == "lstm"
    T = max(1, opt.REFRESH_CHUNK_TOKENS // R)
    h = torch.zeros((1, R, H), device=batch.h0.device)
    c = torch.zeros_like(h) if lstm else None
    want_h0 = batch.h0.clone()
    want_c0 = batch.c0.clone() if lstm else None
    with torch.no_grad():
        for t0 in range(0, L, T):
            t1 = min(L, t0 + T)
            n = t1 - t0
            idx = st.obs_token[t0 * R:t1 * R]
            ins = {}
            for k in Policy.INPUT_KEYS:
                src = batch.observations[k]
                flat = src.reshape((-1,) + tuple(src.shape[2:]))
                ins[k] = ops.gather_rows_fill([flat], idx)[0].view((n, R) + tuple(src.shape[2:]))
                ref = flat[idx.clamp(min=0)] * (idx >= 0).view((-1,) + (1,) * (src.dim() - 2)).float()
                assert torch.equal(ins[k].reshape(ref.shape), ref), k
            ybufs, cbufs, _, _ = opt._rollout_forward(ins, h, c)
            lo, hi = np.searchsorted(lay.step, [t0, t1])
            if hi > lo:
                acc = torch.zeros(2, dtype=torch.float64, device=h.device)
                ops.refresh_states(ybufs, cbufs if lstm else None, t0, st.step[lo:hi], st.rollout[lo:hi],
                                   st.slot[lo:hi], batch.h0, batch.c0, None, None, acc)
                src_t = st.step[lo:hi] - t0
                want_h0[0, st.slot[lo:hi]] = ybufs[0][src_t, st.rollout[lo:hi]]
                if lstm:
                    want_c0[0, st.slot[lo:hi]] = cbufs[0][src_t, st.rollout[lo:hi]]
            h = ybufs[0][n].unsqueeze(0)
            c = cbufs[0][n].unsqueeze(0) if lstm else None
    assert torch.equal(batch.h0, want_h0)
    if lstm:
        assert torch.equal(batch.c0, want_c0)


# ------------------------------------------------------------------------------------------------ equivalences
def test_packed_equals_unpacked(tmp_path):
    out = []
    for pack in (False, True):
        opt = make_optimizer(tmp_path, epochs=3, recompute_states=True, recompute_advantages=True, mask_padding=True,
                             pack_sequences=pack)
        batch = opt.batch_from_rollouts(_rollouts(opt, 3))
        opt.train_epochs(batch)
        out.append((opt.last_state_refresh_stats["drift"], opt.flat.param.detach().cpu()))
    (d0, p0), (d1, p1) = out
    assert abs(d1 - d0) <= 1e-4 * d0
    torch.testing.assert_close(p1, p0, rtol=1e-5, atol=1e-6)


def test_eager_equals_replayed(tmp_path):
    """The replayed step reads the refreshed h0 in place: losses, states and weights are bit-identical."""
    out = []
    for graphs in (False, True):
        opt = make_optimizer(tmp_path, epochs=4, lr=1e-3, recompute_states=True, mask_padding=True)
        opt.use_cuda_graph = graphs
        batch = opt.batch_from_rollouts(_rollouts(opt, 4))
        losses = opt.train_epochs(batch)[0]
        out.append(([[float(v) for v in l.values()] for l in losses], _states(batch), opt.flat.param.detach().clone()))
        if graphs:
            assert any(isinstance(v, tuple) for v in opt._graphs.values())
    assert out[0][0] == out[1][0]
    assert all(torch.equal(a, b) for a, b in zip(out[0][1], out[1][1])) and torch.equal(out[0][2], out[1][2])


ITER_CONFIGS = {
    "m1_lstm": dict(M=1),
    "m2_lstm_masked": dict(M=2, mask_padding=True),
    "m2_gru_masked_adv": dict(M=2, mask_padding=True, recompute_advantages=True, hidden_size=256, cell="gru"),
    "m1_lstm_popart_adv": dict(M=1, value_norm=True, recompute_advantages=True),
    "m2_gru_vtrace_masked_adv": dict(M=2, mask_padding=True, recompute_advantages=True, advantage_estimator="vtrace",
                                     hidden_size=256, cell="gru"),
    # rollouts cut from a longer game: non-zero start states, and with the advantages V(s_L) from the refreshed state
    "m2_lstm_cut": dict(M=2, cut=True),
    "m1_lstm_cut_masked_adv": dict(M=1, cut=True, mask_padding=True, recompute_advantages=True),
    "m2_lstm_cut_adv": dict(M=2, cut=True, recompute_advantages=True),
    "m1_gru_cut_masked_adv": dict(M=1, cut=True, mask_padding=True, recompute_advantages=True, hidden_size=256,
                                  cell="gru"),
    # kl_stop ends the iteration at its third step, after two refreshes, and no refresh follows
    "m1_lstm_masked_kl_stop": dict(M=1, mask_padding=True, kl_stop=True, epochs=4),
}


def _kl_limit(tmp_path, H, cell, rollouts, epochs, **kw):
    """A limit between the all-ranks KL of the second and the third step of an iteration run without a stop, so that the
    third step is the one the limit stops."""
    probe = make_optimizer(tmp_path, hidden_size=H, cell=cell, epochs=epochs, min_seq=2, recompute_states=True,
                           kl_stop=1e9, **kw)
    stats = probe.train_epochs(probe.batch_from_rollouts(copy.deepcopy(rollouts)))[3]
    kl = [st["kl_all_ranks"] for st in stats]
    assert 0 < 2 * kl[1] < kl[2], kl
    return float(np.sqrt(kl[1] * kl[2]))


@pytest.mark.parametrize("name", sorted(ITER_CONFIGS))
def test_iteration_vs_oracle(name, tmp_path):
    """One iteration of 3 epochs (4 under kl_stop) with the state refresh, against the reference optimizer extended with
    it (``state_refresh_oracle.StateRefreshRefOptimizer``): per-step losses and gradient norms, the final advantages,
    weights and Adam moments, at the whole-step tests' tolerances."""
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
                          recompute_states=True, value_norm_decay=0.9, kl_stop=limit, **kw)
    refreshes = []
    real = mine._refresh_states
    mine._refresh_states = lambda b: (refreshes.append(1), real(b))
    torch.manual_seed(7)
    oracle = SO.StateRefreshRefOptimizer(StackedRefPolicy(H, cell, 1), seq_len=S, decay=0.9,
                                         recompute_advantages=kw.get("recompute_advantages", False),
                                         estimator=kw.get("advantage_estimator", "gae"),
                                         mask_padding=kw.get("mask_padding", False),
                                         value_norm=kw.get("value_norm", False), kl_stop=limit)
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
    # the refreshed start states the last epoch trained from
    h_o = [s.hidden[0] if isinstance(s.hidden, tuple) else s.hidden for s in xs_o]
    torch.testing.assert_close(batch.h0.cpu(), torch.cat(h_o, dim=1).float(), rtol=1e-4, atol=1e-4)
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


@pytest.mark.parametrize("M", [1, 2])
def test_iteration_refreshes_before_every_later_epoch(M, tmp_path):
    """3 epochs: two refreshes, none before epoch 0; the minibatch shuffles are those of an optimizer without the refresh;
    with kl_stop, none after the step that stopped the iteration."""
    opt = make_optimizer(tmp_path, epochs=3, min_seq=2, lr=1e-3, num_minibatches=M, recompute_states=True,
                         mask_padding=True)
    off = make_optimizer(tmp_path, epochs=3, min_seq=2, lr=1e-3, num_minibatches=M, mask_padding=True)
    calls = []
    real = opt._refresh_states
    opt._refresh_states = lambda b: (calls.append(1), real(b))
    rollouts = _rollouts(opt, 5, extra=False)
    opt.train_epochs(opt.batch_from_rollouts(copy.deepcopy(rollouts)))
    off.train_epochs(off.batch_from_rollouts(copy.deepcopy(rollouts)))
    assert len(calls) == 2
    assert opt.minibatch_rng.bit_generator.state == off.minibatch_rng.bit_generator.state
    for kl_stop in (1e-30, 1e9):
        stop = make_optimizer(tmp_path, epochs=3, lr=1e-3, recompute_states=True, kl_stop=kl_stop)
        n = []
        real_s = stop._refresh_states
        stop._refresh_states = lambda b: (n.append(1), real_s(b))
        losses = stop.train_epochs(stop.batch_from_rollouts(copy.deepcopy(rollouts)))[0]
        assert len(n) == len(losses) - 1 if kl_stop < 1 else len(n) == 2


def test_peak_memory_is_bounded_by_the_block(tmp_path):
    opt = make_optimizer(tmp_path, epochs=2, lr=1e-3, recompute_states=True, recompute_advantages=True)
    batch = opt.batch_from_rollouts([make_rollout(L, 40 + i) for i, L in enumerate((512, 300, 211))])
    opt.train(batch)
    peaks = {}
    for tokens in (10 ** 9, 3 * 3):
        opt.REFRESH_CHUNK_TOKENS = tokens
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        opt._refresh_states(batch)
        torch.cuda.synchronize()
        peaks[tokens] = torch.cuda.max_memory_allocated() - base
    print("peak above the resident state: one block %.1f MB, blocks of 3 steps %.1f MB"
          % (peaks[10 ** 9] / 2**20, peaks[9] / 2**20))
    assert peaks[9] < peaks[10 ** 9] / 4


def test_feature_off_attaches_nothing(tmp_path):
    off = make_optimizer(tmp_path)
    batch = off.batch_from_rollouts([make_rollout(40, 1)])
    assert batch.state_refresh is None and off.last_state_refresh_stats is None
    one = make_optimizer(tmp_path, epochs=1, recompute_states=True)
    batch = one.batch_from_rollouts([make_rollout(40, 1)])
    h0 = batch.h0.clone()
    one.train_epochs(batch)
    assert torch.equal(batch.h0, h0) and one.last_state_refresh_stats is None


# ------------------------------------------------------------------------------------------------ two ranks
def _check_two_ranks(got):
    import state_refresh_multi_rank as RM
    a, b = got
    assert a["sizes"] != b["sizes"]
    for rec in got:
        assert rec["refreshes"] == [s for s in rec["sizes"] for _ in range(RM.EPOCHS - 1)]
        assert all(np.isfinite(x) and x > 0 for x in rec["drifts"])
    assert int(a["steps"].max()) == RM.ITERATIONS * RM.EPOCHS * 2
    assert torch.equal(a["steps"], b["steps"])
    assert torch.equal(a["param"], b["param"]) and torch.equal(a["exp_avg"], b["exp_avg"])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_nccl_stay_in_sync(tmp_path):
    import state_refresh_multi_rank as RM
    _check_two_ranks(RM.run(tmp_path, "nccl"))


def test_two_ranks_gloo_one_gpu_stay_in_sync(tmp_path):
    import state_refresh_multi_rank as RM
    _check_two_ranks(RM.run(tmp_path, "gloo"))
