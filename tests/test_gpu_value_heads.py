"""GPU tests of the value heads (``DotaOptimizer(value_heads=...)``): the multi-head scan against the float64 oracle
(``value_heads_oracle.py``) on ragged rollouts with terminal and cut bootstraps, with and without the padding segments, and
at the benchmark's 131,072 rows; the indexed scan against the plain one; one group of all ten keys bitwise against
``dc_gae_scan``; the value-heads loss against float64; a training step of one all-keys head against the default
optimizer; the affine_value gradient rows of three heads against float64; a three-head iteration with every option,
eager against replayed; and the checkpoints."""
import os
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_continuation as C  # noqa: E402
import test_gpu_parity as P  # noqa: E402
import value_heads_oracle as VH  # noqa: E402
from dotaclient_b200.policy import REWARD_KEYS  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
N_C2 = 131072
THREE = {'win': ['win'], 'fight': ['enemy', 'kills', 'death', 'hp'], 'farm': ['xp', 'lh', 'denies', 'tower_hp', 'mana']}
GAMMAS3 = {'win': 0.999, 'farm': 0.95}


def make_optimizer(log_dir, hidden_size=128, cell="lstm", seq_len=16, epochs=1, min_seq=1, lr=5e-5, checkpoint=False,
                   pretrained_model=None, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="value-heads", rmq_port=uuid.uuid4().int % 100000, epochs=epochs,
                         min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=lr, checkpoint=checkpoint,
                         pretrained_model=pretrained_model, mq_prefetch_count=1, log_dir=str(log_dir), entropy_coef=5e-4,
                         vf_coef=0.5, run_local=True, hidden_size=hidden_size, cell=cell, **kw)


def _groups(K, g):
    if K == 1:
        return np.zeros(10, np.int32), np.array([0.98])
    if K == 2:
        return np.array([1, 0, 1, 1, 1, 1, 1, 1, 1, 1], np.int32), np.array([0.999, 0.95])
    return g.permutation(np.arange(10) % K).astype(np.int32), np.linspace(0.9, 1.0, K)


def _scan_case(lengths, terminal, mask, K, seed):
    from dotaclient_b200.optimizer import rollout_segments
    g = np.random.default_rng(seed)
    seg, boot_src, _ = rollout_segments(lengths, terminal, 16, mask)
    n = int(seg[-1])
    n_cut = sum(not t for t in terminal)
    cut_v = g.standard_normal((n_cut, K)).astype(np.float32)
    boot = np.where(boot_src[:, None] >= 0, cut_v[np.maximum(boot_src, 0)], 0.0).astype(np.float32)
    group, gammas = _groups(K, g)
    return dict(seg=seg, boot=boot, group=group, gammas=gammas,
                rewards=(g.standard_normal((n, 10)) * 0.1).astype(np.float32),
                values=g.standard_normal((n, K)).astype(np.float32))


def _T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(P.dev())


def _within_rounding(got, want64):
    """fp32 results of float64 recursions: within one fp32 ulp of the float64 value."""
    got = np.asarray(got, np.float32)
    tol = np.spacing(np.abs(got)).astype(np.float64) + 1e-12
    bad = np.abs(got.astype(np.float64) - want64) > tol
    assert not bad.any(), (np.flatnonzero(bad.reshape(-1))[:5], got.reshape(-1)[bad.reshape(-1)][:5],
                           want64.reshape(-1)[bad.reshape(-1)][:5])


LENGTHS = [1, 15, 16, 17, 31, 33, 64, 517, 1380, 2, 7]
TERMINAL = [i % 3 != 0 for i in range(len(LENGTHS))]


@pytest.mark.parametrize("K", [1, 2, 10])
@pytest.mark.parametrize("mask", [False, True])
def test_scan_vs_float64(K, mask):
    from dotaclient_b200 import ops
    x = _scan_case(LENGTHS, TERMINAL, mask, K, 10 + K)
    boot = _T(x["boot"])
    adv, ret = ops.gae_scan_heads(_T(x["rewards"]), _T(x["values"]), _T(x["seg"]), x["group"], x["gammas"], 0.97,
                                  boot_value=boot, boot_reward=boot)
    _, _, a64, r64 = VH.scan_heads(x["rewards"], x["values"], x["seg"], x["group"], x["gammas"], 0.97, x["boot"],
                                   x["boot"])
    assert tuple(adv.shape) == (len(a64),) and tuple(ret.shape) == r64.shape
    _within_rounding(adv.cpu().numpy(), a64)
    _within_rounding(ret.cpu().numpy(), r64)


def test_scan_at_the_benchmark_rows_sampled():
    """131,072 rows of ragged, partly cut rollouts at K = 10; the oracle runs on a sample of the segments."""
    from dotaclient_b200 import ops
    g = np.random.default_rng(21)
    lengths = []
    while sum((L + 15) // 16 * 16 for L in lengths) < N_C2 - 1400:
        lengths.append(int(g.integers(1000, 1400)))
    rest = N_C2 - sum((L + 15) // 16 * 16 for L in lengths)
    if rest:
        lengths.append(rest)
    terminal = [bool(g.random() < 0.6) for _ in lengths]
    x = _scan_case(lengths, terminal, True, 10, 22)
    assert int(x["seg"][-1]) == N_C2
    boot = _T(x["boot"])
    adv, ret = ops.gae_scan_heads(_T(x["rewards"]), _T(x["values"]), _T(x["seg"]), x["group"], x["gammas"], 0.97,
                                  boot_value=boot, boot_reward=boot)
    adv, ret = adv.cpu().numpy(), ret.cpu().numpy()
    for s in g.choice(len(x["seg"]) - 1, 12, replace=False):
        lo, hi = int(x["seg"][s]), int(x["seg"][s + 1])
        if hi <= lo:
            continue
        _, _, a64, r64 = VH.scan_heads(x["rewards"][lo:hi], x["values"][lo:hi], [0, hi - lo], x["group"], x["gammas"],
                                       0.97, x["boot"][s:s + 1], x["boot"][s:s + 1])
        _within_rounding(adv[lo:hi], a64)
        _within_rounding(ret[lo:hi], r64)


@pytest.mark.parametrize("K", [1, 3])
def test_indexed_equals_plain_scan_scattered(K):
    """A packed-like layout: more tokens than rows, the rows' tokens shuffled, some rows without a token.  Values are read
    from the K value columns of a [n_tok, 128] head output."""
    from dotaclient_b200 import ops
    x = _scan_case(LENGTHS, TERMINAL, True, K, 30 + K)
    n = len(x["rewards"])
    g = np.random.default_rng(31)
    n_tok = n + 77
    tok = g.permutation(n_tok)[:n].astype(np.int64)
    tok[g.random(n) < 0.05] = -1
    store = g.standard_normal((n_tok, 128)).astype(np.float32)
    rows_v = np.where(tok[:, None] >= 0, store[np.maximum(tok, 0), 25:25 + K], 0.0).astype(np.float32)
    boot = _T(x["boot"])
    a0, r0 = ops.gae_scan_heads(_T(x["rewards"]), _T(rows_v), _T(x["seg"]), x["group"], x["gammas"], 0.97,
                                boot_value=boot, boot_reward=boot)
    packed = _T(store)
    a1 = torch.full((n_tok,), 7.0, device=P.dev())
    r1 = torch.full((n_tok, K), -7.0, device=P.dev())
    ops.gae_scan_heads_indexed(_T(x["rewards"]), packed[:, 25:25 + K], _T(tok), _T(x["seg"]), a1, r1, x["group"],
                               x["gammas"], 0.97, boot_value=boot, boot_reward=boot)
    held = torch.from_numpy(tok >= 0).to(P.dev())
    t = _T(tok)[held]
    assert torch.equal(a1[t], a0[held]) and torch.equal(r1[t], r0[held])
    untouched = torch.ones(n_tok, dtype=torch.bool, device=P.dev())
    untouched[t] = False
    assert bool((a1[untouched] == 7.0).all()) and bool((r1[untouched] == -7.0).all())


def test_one_group_of_all_keys_is_dc_gae_scan_bitwise():
    from dotaclient_b200 import ops
    x = _scan_case(LENGTHS, TERMINAL, True, 1, 41)
    rew, seg, boot = _T(x["rewards"]), _T(x["seg"]), _T(x["boot"])
    v = _T(x["values"])
    for gamma in (0.98, 0.999):
        a0, r0 = ops.gae_scan(rew, v[:, 0], seg, gamma, 0.97, boot_value=boot[:, 0], boot_reward=boot[:, 0])
        a1, r1 = ops.gae_scan_heads(rew, v, seg, np.zeros(10, np.int32), [gamma], 0.97, boot_value=boot,
                                    boot_reward=boot)
        assert torch.equal(a0, a1) and torch.equal(r0, r1[:, 0])
        n = len(x["rewards"])
        store = torch.zeros(n, 128, device=P.dev())
        store[:, 25] = v[:, 0]
        tok = torch.arange(n, device=P.dev())
        a2, r2 = torch.empty(n, device=P.dev()), torch.empty(n, device=P.dev())
        ops.gae_scan_indexed(rew, store[:, 25], tok, seg, a2, r2, gamma, 0.97, boot_value=boot[:, 0],
                             boot_reward=boot[:, 0])
        a3, r3 = torch.empty(n, device=P.dev()), torch.empty(n, 1, device=P.dev())
        ops.gae_scan_heads_indexed(rew, store[:, 25:26], tok, seg, a3, r3, np.zeros(10, np.int32), [gamma], 0.97,
                                   boot_value=boot, boot_reward=boot)
        assert torch.equal(a2, a3) and torch.equal(r2, r3[:, 0]) and torch.equal(a0, a2)


@pytest.mark.parametrize("K", [1, 3, 10])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("clip", [0.0, 0.2])
def test_loss_kernel_vs_float64(K, masked, clip):
    from dotaclient_b200 import _lib, ops
    g = np.random.default_rng(50 + K)
    N = 5000
    packed = g.standard_normal((N, 128)).astype(np.float32)
    ret = (packed[:, 25:25 + K] + g.standard_normal((N, K)) * 0.5).astype(np.float32)
    old = (packed[:, 25:25 + K] + g.standard_normal((N, K)) * 0.3).astype(np.float32)
    valid = g.random(N) < 0.8 if masked else None
    dev = P.dev()
    hp = ops.hparam_block(dev, vf_coef=0.5, value_clip=clip)
    out = torch.zeros(_lib.LOSS_SLOTS, device=dev)
    out[0] = 1.25
    d_packed = torch.zeros(N, 128, device=dev)
    stats = torch.zeros(_lib.PPO_STATS_SLOTS, device=dev)
    hs = torch.full((_lib.VALUE_HEADS_STATS_SLOTS,), 9.0, device=dev)
    ops.value_heads_loss(_T(packed), d_packed, _T(ret), hp, out, hs, old_value=_T(old),
                         valid=None if valid is None else _T(valid), stats=stats)
    loss, dv, heads, ev_h, ev_t = VH.value_heads_loss(packed[:, 25:25 + K], ret, 0.5, old, clip, valid)
    out, d_packed, hs = out.cpu().numpy(), d_packed.cpu().numpy(), hs.cpu().numpy()
    np.testing.assert_allclose(out[3], loss, rtol=1e-5)
    assert out[0] == np.float32(np.float32(1.25) + out[3])
    np.testing.assert_allclose(d_packed[:, 25:25 + K], dv, rtol=1e-5, atol=1e-12)
    assert not d_packed[:, :25].any() and not d_packed[:, 25 + K:].any()
    np.testing.assert_allclose(hs[:K], heads, rtol=1e-5)
    np.testing.assert_allclose(hs[_lib.VALUE_HEADS_MAX:_lib.VALUE_HEADS_MAX + K], ev_h, rtol=1e-4, atol=1e-5)
    assert not hs[K:_lib.VALUE_HEADS_MAX].any() and not hs[_lib.VALUE_HEADS_MAX + K:].any()
    np.testing.assert_allclose(stats.cpu().numpy()[_lib.STAT_EXPLAINED_VAR], ev_t, rtol=1e-4, atol=1e-5)


def test_one_all_keys_head_trains_as_the_default(tmp_path):
    rollouts = [make_rollout(L, 200 + i) for i, L in enumerate((40, 23, 48))]
    res = []
    for kw in ({}, {'value_heads': {'all': list(REWARD_KEYS)}}):
        opt = make_optimizer(tmp_path, value_clip=0.2, **kw)
        opt.use_cuda_graph = False
        batch = opt.batch_from_rollouts(rollouts)
        losses = opt.train(batch)[0]
        res.append((batch, {k: float(v) for k, v in losses.items()}, dict(opt.last_ppo_stats), opt.flat.param.clone(),
                    opt.exp_avg.clone(), opt.exp_avg_sq.clone()))
    (b0, l0, s0, p0, m0, v0), (b1, l1, s1, p1, m1, v1) = res
    assert torch.equal(b0.advantages, b1.advantages) and torch.equal(b0.returns, b1.returns)
    assert torch.equal(b0.old_values, b1.old_values)
    for k in l0:
        np.testing.assert_allclose(l1[k], l0[k], rtol=1e-5, atol=1e-7, err_msg=k)
    np.testing.assert_allclose(s1['explained_variance'], s0['explained_variance'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(s1['loss/value/all'], l0['value_loss'], rtol=1e-5)
    torch.testing.assert_close(p1, p0, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m1, m0, rtol=1e-4, atol=1e-9)
    torch.testing.assert_close(v1, v0, rtol=1e-4, atol=1e-12)


def test_three_head_value_gradient_rows_vs_float64(tmp_path):
    from dotaclient_b200 import _lib, ops
    opt = make_optimizer(tmp_path, value_heads=THREE, value_gammas=GAMMAS3, mask_padding=True)
    batch = opt.batch_from_rollouts([make_rollout(L, 300 + i) for i, L in enumerate((40, 23, 48))])
    pol = opt.policy_base
    x, ue = pol._encode(batch.observations['env'], [batch.observations[k] for k in pol.INPUT_KEYS[1:]])
    y, _ = pol._recur(x.contiguous(), (batch.h0, batch.c0))
    y = y.detach().requires_grad_(False)
    packed, _ = pol._head_outputs(y, ue)
    dev = P.dev()
    d_packed = torch.zeros_like(packed)
    out = torch.zeros(_lib.LOSS_SLOTS, device=dev)
    hs = torch.zeros(_lib.VALUE_HEADS_STATS_SLOTS, device=dev)
    ops.value_heads_loss(packed, d_packed, batch.returns, ops.hparam_block(dev, vf_coef=0.5), out, hs, valid=batch.valid)
    pol.zero_grad(set_to_none=True)
    torch.autograd.backward([packed], [d_packed])
    N = packed.numel() // 128
    v = packed.detach().reshape(N, 128)[:, 25:28].cpu().numpy()
    _, dv, _, _, _ = VH.value_heads_loss(v, batch.returns.reshape(N, 3).cpu().numpy(), 0.5,
                                         valid=batch.valid.reshape(N).cpu().numpy())
    y64 = y.reshape(N, -1).double().cpu().numpy()
    gw, gb = dv.T @ y64, dv.sum(axis=0)
    w, b = pol.affine_value.weight.grad.double().cpu().numpy(), pol.affine_value.bias.grad.double().cpu().numpy()
    np.testing.assert_allclose(w, gw, rtol=1e-4, atol=1e-5 * np.abs(gw).max())
    np.testing.assert_allclose(b, gb, rtol=1e-4, atol=1e-5 * np.abs(gb).max())


def test_three_heads_every_option_eager_equals_replayed(tmp_path):
    out = []
    for graphs in (False, True):
        opt = make_optimizer(tmp_path, epochs=3, min_seq=2, value_heads=THREE, value_gammas=GAMMAS3, mask_padding=True,
                             pack_sequences=True, num_minibatches=2, recompute_advantages=True, recompute_states=True)
        opt.use_cuda_graph = graphs
        batch = opt.batch_from_rollouts(C._mixed(opt, 4, False))
        assert tuple(batch.returns.shape) == tuple(batch.advantages.shape) + (3,)
        losses, _, _, stats = opt.train_epochs(batch)
        out.append(([[float(v) for v in l.values()] for l in losses], batch.advantages.clone(), batch.returns.clone(),
                    opt.flat.param.detach().clone(), [s['loss/value/win'] for s in stats]))
        if graphs:
            assert any(isinstance(v, tuple) for v in opt._graphs.values())
    assert out[0][0] == out[1][0] and out[0][4] == out[1][4]
    for a, b in zip(out[0][1:4], out[1][1:4]):
        assert torch.equal(a, b)


def test_checkpoints(tmp_path):
    from dotaclient_b200.policy import Policy, fold_value_heads
    run = tmp_path / "run"
    opt = make_optimizer(run, checkpoint=True, value_heads=THREE, value_gammas=GAMMAS3)
    opt.use_cuda_graph = False
    opt.train(opt.batch_from_rollouts([make_rollout(L, 400 + i) for i, L in enumerate((40, 23))]))
    opt.upload_model(version=2)
    heads = {k: v.detach().cpu().clone() for k, v in opt.policy_base.state_dict().items()}
    published = torch.load(str(run / "model_000000002.pt"), map_location="cpu")
    Policy(hidden_size=128, cell="lstm").load_state_dict(published, strict=True)      # the reference's shape
    for k, v in fold_value_heads(heads).items():
        assert torch.equal(published[k], v), k
    assert (run / "value_heads_000000002.state").exists()
    # resume restores the three heads
    opt2 = make_optimizer(run, checkpoint=True, value_heads=THREE, value_gammas=GAMMAS3)
    assert opt2.iteration_start == 3
    assert torch.equal(opt2.policy_base.affine_value.weight.detach().cpu(), heads['affine_value.weight'])
    assert torch.equal(opt2.policy_base.affine_value.bias.detach().cpu(), heads['affine_value.bias'])
    # other groups: refused
    with pytest.raises(ValueError, match="reinterpreted"):
        make_optimizer(run, checkpoint=True, value_heads={'all': list(REWARD_KEYS)})
    # a one-row model without the side file is split
    plain = tmp_path / "plain"
    base = make_optimizer(plain, checkpoint=True)
    one = {k: v.cpu() for k, v in base.policy_base.state_dict().items()}
    opt3 = make_optimizer(tmp_path / "new", pretrained_model=str(plain / "model_000000001.pt"), value_heads=THREE)
    w = opt3.policy_base.affine_value.weight.detach().cpu()
    assert torch.equal(w, (one['affine_value.weight'] / 3).expand(3, -1))
    assert torch.equal(opt3.policy_base.affine_value.bias.detach().cpu(), (one['affine_value.bias'] / 3).expand(3))
