"""GPU tests of experience prep on rollouts cut from a longer game (``'initial_hidden'``, ``'terminal': False``): explicit
defaults change no bit, a game sent in pieces preps like the whole game, the bootstrap against the float64 oracle under
GAE and V-trace with and without ``mask_padding``, the padded rows and the extra observation row, the whole step against
the CPU oracle, and ``run_iteration`` on ``split_rollout`` pieces."""
import copy
import os
import pickle
import sys
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import continuation_oracle as CO  # noqa: E402
import test_gpu_parity as P  # noqa: E402
import test_gpu_vtrace as V  # noqa: E402
import vtrace_oracle as VT  # noqa: E402
from stacked_oracle import StackedRefPolicy  # noqa: E402
from dotaclient_b200.synthetic import make_rollout, split_rollout  # noqa: E402

pytestmark = pytest.mark.gpu
HEADS = P.HEADS
G, LAM = 0.98, 0.97


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", num_layers=1, seq_len=16, min_seq=1, port=None, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="continuation", rmq_port=port if port is not None else uuid.uuid4().int % 100000,
                         epochs=1, min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=5e-5, checkpoint=False,
                         pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5,
                         run_local=True, hidden_size=hidden_size, cell=cell, num_layers=num_layers, **kw)


def _random_state(pol, seed, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    h = scale * torch.randn(pol.num_layers, 1, pol.hidden_size, generator=g)
    return (h, scale * torch.randn(h.shape, generator=g)) if pol.cell == "lstm" else h


def _learner_state(pol, data, steps, hidden=None):
    """The learner's recurrent state after ``steps`` steps of ``data`` (Policy.forward from ``hidden``, default zero)."""
    d = P.dev()
    h = pol.init_hidden() if hidden is None else hidden
    h = tuple(x.to(d) for x in h) if isinstance(h, tuple) else h.to(d)
    with torch.no_grad():
        _, value, h = pol.forward(**{k: v[:steps].unsqueeze(0).to(d) for k, v in data["observations"].items()}, hidden=h)
    return (tuple(x.cpu() for x in h) if isinstance(h, tuple) else h.cpu()), value


def _state_parts(h):
    return h if isinstance(h, tuple) else (h,)


def _mixed(opt, seed, behaviour=False, lengths=(40, 23, 48, 7, 33), terminal=(False, True, False, True, False)):
    """Ragged rollouts, the non-terminal ones with their extra observation row, all with non-zero initial states, and
    with ``behaviour`` the behaviour log-probabilities of a stale policy."""
    out = []
    for i, (L, term) in enumerate(zip(lengths, terminal)):
        r = make_rollout(L + (0 if term else 1), 500 + 10 * seed + i, game_id=i)
        if behaviour:
            r = V._stale_behaviour(opt, [r], 20 + i)[0]
        if not term:
            r = split_rollout(r, [L])[0]
        r["initial_hidden"] = _random_state(opt.policy_base, 50 + 10 * seed + i)
        out.append(r)
    return out


def _tensors_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, dict):
            _tensors_equal(x, y)
        elif isinstance(x, (list, tuple)) and x and isinstance(x[0], torch.Tensor):
            assert len(x) == len(y) and all(torch.equal(u, v) for u, v in zip(x, y)), k
        elif isinstance(x, torch.Tensor):
            assert torch.equal(x, y), k
        elif isinstance(x, np.ndarray):
            assert np.array_equal(x, y), k
        else:
            assert x == y, k


# ------------------------------------------------------------------------------------------------ explicit defaults
@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
@pytest.mark.parametrize("mask_padding", [False, True])
def test_explicit_defaults_change_no_bit(estimator, mask_padding, tmp_path):
    opt = make_optimizer(tmp_path, num_layers=2, advantage_estimator=estimator, mask_padding=mask_padding)
    rollouts = [make_rollout(L, 300 + i, game_id=i) for i, L in enumerate((40, 23, 48))]
    if estimator == "vtrace":
        rollouts = V._stale_behaviour(opt, rollouts, 4)
    explicit = copy.deepcopy(rollouts)
    for r in explicit:
        r["initial_hidden"] = opt.policy_base.init_hidden()
        r["terminal"] = True
    p0, p1 = opt._prepare_rollouts(copy.deepcopy(rollouts)), opt._prepare_rollouts(copy.deepcopy(explicit))
    assert p0["bootstrap"] is None and p1["bootstrap"] is None
    _tensors_equal(p0, p1)
    b0, b1 = opt.batch_from_rollouts(copy.deepcopy(rollouts)), opt.batch_from_rollouts(copy.deepcopy(explicit))
    for (_, k, x), (_, _, y) in zip(b0.tensors(), b1.tensors()):
        assert torch.equal(x, y), k


# ------------------------------------------------------------------------------------------------ a game in pieces
def _behaviour(opt, game):
    return V._stale_behaviour(opt, [game], 9)[0]


@pytest.mark.parametrize("H,cell,layers", [(256, "gru", 1), (128, "lstm", 2)])
def test_pieces_prep_like_the_whole_game(H, cell, layers, tmp_path):
    """A 53-step game (3 S + 5) cut at 21 (not a multiple of S) and 32 (a multiple), the pieces starting from the
    learner's own state at the cut: values, old log-probs and every chunk's entering state match the whole game's at the
    same steps, and advantages, returns and V-trace targets satisfy the whole-game identities (continuation_oracle)."""
    S = 16
    gae = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers)
    vt = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers, advantage_estimator="vtrace")
    pol = gae.policy_base
    game = _behaviour(gae, make_rollout(53, 77, game_id=5))
    cuts = [21, 32]
    states = [None] + [_learner_state(pol, game, c)[0] for c in cuts]
    pieces = split_rollout(game, cuts, initial_hiddens=states)
    bounds = [(0, 21), (21, 32), (32, 53)]
    w, p = gae._prepare_rollouts([copy.deepcopy(game)]), gae._prepare_rollouts(copy.deepcopy(pieces))
    wv, pv = vt._prepare_rollouts([copy.deepcopy(game)]), vt._prepare_rollouts(copy.deepcopy(pieces))
    assert p["bootstrap"].shape == (2,)
    V_w = w["values_lr"][:, 0].double().cpu().numpy()
    A_w, ret_w = w["adv_c"].double().cpu().numpy(), w["ret_c"].double().cpu().numpy()
    vs_w = wv["ret_c"].double().cpu().numpy()
    old_w = w["old_logp"][:53, 0].cpu().numpy()
    acted = np.stack([np.asarray(game["actions"][k]).any(axis=1) for k in HEADS], axis=1)
    c = LAM * np.minimum(1.0, np.exp(VT.log_rho(old_w, np.where(acted, game["behaviour_logp"], 0.0))))
    base = 0
    for i, (a, b) in enumerate(bounds):
        n, last = b - a, b == 53
        torch.testing.assert_close(p["values_lr"][:n, i], w["values_lr"][a:b, 0], rtol=1e-4, atol=2e-5)
        torch.testing.assert_close(p["old_logp"][:n, i], w["old_logp"][a:b, 0], rtol=1e-4, atol=2e-5)
        for j in range((n + S - 1) // S):                      # the state entering each chunk
            for bufs in (("ybufs",) + (("cbufs",) if cell == "lstm" else ())):
                for k in range(layers):
                    torch.testing.assert_close(p[bufs][k][j * S, i], w[bufs][k][a + j * S, 0], rtol=1e-4, atol=2e-5)
        if not last:                                           # the bootstrap is the critic's value at the cut
            torch.testing.assert_close(p["bootstrap"][i], w["values_lr"][b, 0], rtol=1e-4, atol=2e-5)
        t = np.arange(n)
        A_p, ret_p = p["adv_c"][base:base + n].double().cpu().numpy(), p["ret_c"][base:base + n].double().cpu().numpy()
        vs_p = pv["ret_c"][base:base + n].double().cpu().numpy()
        if last:
            want_A, want_ret, want_vs = A_w[a:b], ret_w[a:b], vs_w[a:b]
        else:
            want_A = A_w[a:b] - (G * LAM) ** (n - t) * A_w[b]
            want_ret = ret_w[a:b] - G ** (n - t) * (ret_w[b] - V_w[b])
            prod = np.array([np.prod(c[a + s:b]) for s in range(n)])
            want_vs = vs_w[a:b] - G ** (n - t) * prod * (vs_w[b] - V_w[b])
        np.testing.assert_allclose(A_p, want_A, rtol=1e-4, atol=2e-5, err_msg="advantages of piece %d" % i)
        np.testing.assert_allclose(ret_p, want_ret, rtol=1e-5, atol=1e-5, err_msg="returns of piece %d" % i)
        np.testing.assert_allclose(vs_p, want_vs, rtol=1e-4, atol=2e-5, err_msg="V-trace targets of piece %d" % i)
        base += p["Lps"][i]


# ------------------------------------------------------------------------------------------------ bootstrap vs oracle
@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
@pytest.mark.parametrize("mask_padding", [False, True])
def test_bootstrap_vs_oracle(estimator, mask_padding, tmp_path):
    """Ragged mixed batches against the float64 oracle fed prep's own values and bootstrap: the real steps end on V(s_L)
    (0 when terminal), the padding on 0 (zeroed under mask_padding), and V-trace statistics cover the real steps only."""
    opt = make_optimizer(tmp_path, advantage_estimator=estimator, mask_padding=mask_padding)
    S = opt.seq_len
    rollouts = _mixed(opt, 1, behaviour=estimator == "vtrace")
    batch = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    p = opt._prepare_rollouts(copy.deepcopy(rollouts))
    boots = p["bootstrap"].cpu().numpy()
    assert boots.shape == (3,)
    base, n_cut, col, want_stats = 0, 0, 0, []
    for i, r in enumerate(rollouts):
        L, Lp, term = int(r["rewards"].shape[0]), p["Lps"][i], r.get("terminal", True)
        v = p["values_lr"][:Lp, i].cpu().numpy()
        rew = np.concatenate([VT.reward_sum(r["rewards"]), np.zeros(Lp - L, np.float32)])
        b = 0.0 if term else boots[n_cut]
        if estimator == "vtrace":
            old = p["old_logp"][:Lp, i].cpu().numpy()
            acted = np.stack([np.asarray(r["actions"][k]).any(axis=1) for k in HEADS], axis=1)
            lr = np.concatenate([VT.log_rho(old[:L], np.where(acted, r["behaviour_logp"], 0.0)),
                                 VT.log_rho(old[L:], np.zeros((Lp - L, 5)))])
            scan = lambda lo, hi, boot: VT.vtrace(rew[lo:hi], v[lo:hi], lr[lo:hi], G, LAM, boot=boot)  # noqa: E731
            want_stats.append(VT.stats(lr[:L]))
        else:
            scan = lambda lo, hi, boot: CO.gae(rew[lo:hi], v[lo:hi], G, LAM, boot, boot)  # noqa: E731
        if term and not mask_padding:
            want_a, want_r = scan(0, Lp, 0.0)
        else:
            (a1, r1), (a2, r2) = scan(0, L, b), scan(L, Lp, 0.0)
            if mask_padding:
                a2, r2 = np.zeros(Lp - L), np.zeros(Lp - L)
            want_a, want_r = np.concatenate([a1, a2]), np.concatenate([r1, r2])
        V._close(p["adv_c"][base:base + Lp].cpu().numpy(), want_a)
        V._close(p["ret_c"][base:base + Lp].cpu().numpy(), want_r)
        n = Lp // S
        V._close(batch.advantages[:, col:col + n].t().reshape(-1).cpu().numpy(), want_a)
        V._close(batch.returns[:, col:col + n].t().reshape(-1).cpu().numpy(), want_r)
        if mask_padding:
            assert batch.valid[:, col:col + n].t().reshape(-1).tolist() == [True] * L + [False] * (Lp - L)
        base, col, n_cut = base + Lp, col + n, n_cut + (not term)
    if estimator == "vtrace":
        got, want = opt.last_vtrace_stats, VT.summary(np.stack(want_stats))
        for k in want:
            assert got[k] == pytest.approx(want[k], rel=1e-9, abs=1e-12), k


# ------------------------------------------------------------------------------------------------ padded rows, extra row
@pytest.mark.parametrize("H,cell,layers", [(256, "gru", 1), (128, "lstm", 2)])
def test_padded_rows_and_the_extra_row(H, cell, layers, tmp_path):
    """Sent non-terminal rather than terminal (same steps, same initial state), a rollout's padded rows keep their
    advantages and returns bit for bit, the training batch is bit-identical but for the real steps' advantages and
    returns, and its bootstrap is Policy.forward on the extra row from the learner's state after the last step."""
    opt = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers)
    pol = opt.policy_base
    other = make_rollout(29, 11, game_id=1) | {"initial_hidden": _random_state(pol, 12)}
    cut = split_rollout(make_rollout(41, 13, game_id=2), [40])[0] | {"initial_hidden": _random_state(pol, 14)}
    whole = cut | {"terminal": True, "observations": {k: v[:40] for k, v in cut["observations"].items()}}
    pc, pw = opt._prepare_rollouts(copy.deepcopy([other, cut])), opt._prepare_rollouts(copy.deepcopy([other, whole]))
    base = pc["Lps"][0]
    assert torch.equal(pc["adv_c"][:base], pw["adv_c"][:base]) and torch.equal(pc["ret_c"][:base], pw["ret_c"][:base])
    pad = slice(base + 40, base + 48)
    assert torch.equal(pc["adv_c"][pad], pw["adv_c"][pad]) and torch.equal(pc["ret_c"][pad], pw["ret_c"][pad])
    assert not torch.equal(pc["adv_c"][base:base + 40], pw["adv_c"][base:base + 40])
    bc, bw = opt.batch_from_rollouts(copy.deepcopy([other, cut])), opt.batch_from_rollouts(copy.deepcopy([other, whole]))
    for (_, k, x), (_, _, y) in zip(bc.tensors(), bw.tensors()):
        if k not in ("advantages", "returns"):
            assert torch.equal(x, y), k
    # the bootstrap: Policy.forward on row 40 from the state after step 39 (state buffer slot 40 of every layer)
    d = P.dev()
    h = torch.stack([yb[40, 1] for yb in pc["ybufs"]]).unsqueeze(1)
    hidden = (h, torch.stack([cb[40, 1] for cb in pc["cbufs"]]).unsqueeze(1)) if cell == "lstm" else h
    with torch.no_grad():
        _, value, _ = pol.forward(**{k: v[40:41].unsqueeze(0).to(d) for k, v in cut["observations"].items()}, hidden=hidden)
    torch.testing.assert_close(pc["bootstrap"], value.reshape(1), rtol=1e-5, atol=1e-6)
    # ... and from the learner's state after the last step, run by Policy.forward over the rollout
    state, _ = _learner_state(pol, cut, 40, hidden=cut["initial_hidden"])
    for x, y in zip(_state_parts(state), _state_parts(hidden)):
        torch.testing.assert_close(x, y.cpu(), rtol=1e-4, atol=2e-5)
    _, value2 = _learner_state(pol, cut, 41, hidden=cut["initial_hidden"])
    torch.testing.assert_close(pc["bootstrap"], value2[0, 40].reshape(1), rtol=1e-4, atol=2e-5)


# ------------------------------------------------------------------------------------------------ the step vs the oracle
@pytest.mark.parametrize("H,cell,layers,mask_padding", [(256, "gru", 1, False), (128, "lstm", 2, True)])
def test_step_vs_oracle(H, cell, layers, mask_padding, tmp_path):
    """Prep of a batch mixing terminal and non-terminal rollouts with non-zero initial states, then two train() steps,
    against the reference prep started from the same states and bootstrapped from the reference policy on the extra row,
    at the tolerances of test_masked_step_vs_oracle."""
    torch.set_num_threads(8)
    S = 16
    mine = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=layers, mask_padding=mask_padding)
    torch.manual_seed(7)
    oracle = CO.ContinuationRefOptimizer(StackedRefPolicy(H, cell, layers), seq_len=S, mask_padding=mask_padding)
    rollouts = _mixed(mine, 2)
    xs_m = [s for grp in mine.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in grp]
    xs_o = [s for r in rollouts for s in oracle.experiences_from_rollout(copy.deepcopy(r))]
    P._compare_sequences(xs_m, xs_o, cell)
    if mask_padding:
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


# ------------------------------------------------------------------------------------------------ run_iteration
def test_run_iteration_on_split_pieces(tmp_path):
    """Two games published in 5 pieces (3 of them non-terminal) through the in-process MessageQueue train, and the
    iteration reports non_terminal_fraction; whole games report no such key."""
    from dotaclient_b200.optimizer import MessageQueue
    games = [make_rollout(L, 900 + i, game_id=i, weight_version=1, with_canvas=True) for i, L in enumerate((40, 57))]

    def run(rollouts, port, min_seq):
        opt = make_optimizer(tmp_path, min_seq=min_seq, port=port, num_minibatches=2)
        actor = MessageQueue(host="continuation", port=port, prefetch_count=1, use_model_exchange=False)
        actor.connect()
        for r in rollouts:
            actor.publish_experience(pickle.dumps(r))
        before = opt.flat.param.clone()
        metrics = opt.run_iteration(1)
        assert int(opt.adam_steps.max()) == 2 and not torch.equal(opt.flat.param, before)
        assert np.isfinite(float(metrics["loss/sum"]))
        return metrics

    pol = make_optimizer(tmp_path).policy_base
    pieces = split_rollout(games[0], [20], [None, _learner_state(pol, games[0], 20)[0]])
    pieces += split_rollout(games[1], [16, 30], [None] + [_learner_state(pol, games[1], c)[0] for c in (16, 30)])
    assert [len(p["rewards"]) for p in pieces] == [20, 20, 16, 14, 27]
    base = uuid.uuid4().int % 100000
    met = run(pieces, base, 8)             # 2 + 2 + 1 + 1 + 2 sequences: every piece
    assert met["non_terminal_fraction"] == pytest.approx(3 / 5, rel=1e-12)
    met0 = run(games, base + 1, 7)         # 3 + 4
    assert set(met) - set(met0) == {"non_terminal_fraction"} and set(met0) <= set(met)
