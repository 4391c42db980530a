"""Host-side checks of rollouts cut from a longer game: the validation of ``'initial_hidden'`` / ``'terminal'`` before
anything is uploaded, the scan segments and bootstrap sources of experience prep (``rollout_segments``),
``synthetic.split_rollout``, and the float64 oracle of bootstrapped GAE / returns / V-trace (``continuation_oracle.py``)
against hand-computed values and against the identities that tie a cut game to the whole one."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import continuation_oracle as CO  # noqa: E402
import vtrace_oracle as VT  # noqa: E402
from dotaclient_b200.optimizer import (check_continuation, chunk_valid_lengths, padded_segment_offsets,  # noqa: E402
                                       rollout_segments)
from dotaclient_b200.synthetic import make_rollout, split_rollout  # noqa: E402

G, LAM = 0.98, 0.97


# ------------------------------------------------------------------------------------------------ validation
def _piece(L=20, terminal=None, hidden=None, extra_rows=None, game_id=3):
    d = make_rollout(L + (1 if extra_rows is None and terminal is False else (extra_rows or 0)), 5, game_id=game_id)
    d = dict(d, rewards=d["rewards"][:L], masks={k: v[:L] for k, v in d["masks"].items()},
             actions={k: v[:L] for k, v in d["actions"].items()})
    d["player_id"] = 4
    if terminal is not None:
        d["terminal"] = terminal
    if hidden is not None:
        d["initial_hidden"] = hidden
    return d


GRU = ("gru", 2, 64)
LSTM = ("lstm", 1, 32)


def test_valid_rollouts_pass():
    h = torch.randn(2, 1, 64)
    check_continuation([_piece(), _piece(terminal=True), _piece(terminal=False, hidden=h),
                        _piece(hidden=h.numpy(), terminal=np.bool_(True))], *GRU)
    hc = (torch.randn(1, 1, 32), np.zeros((1, 1, 32), np.float32))
    check_continuation([_piece(terminal=False, hidden=hc), _piece(hidden=list(hc))], *LSTM)


@pytest.mark.parametrize("d, cfg, match", [
    (_piece(hidden=torch.zeros(1, 1, 64)), GRU, r"float \[2, 1, 64\]"),
    (_piece(hidden=torch.zeros(2, 64)), GRU, r"float \[2, 1, 64\]"),
    (_piece(hidden=torch.zeros(2, 1, 32)), GRU, r"float \[2, 1, 64\]"),
    (_piece(hidden=torch.zeros(2, 1, 64, dtype=torch.int32)), GRU, r"float \[2, 1, 64\]"),
    (_piece(hidden=(torch.zeros(2, 1, 64), torch.zeros(2, 1, 64))), GRU, "one \\[2, 1, 64\\] array"),
    (_piece() | {"initial_hidden": None}, GRU, "not a tensor"),
    (_piece(hidden=torch.zeros(1, 1, 32)), LSTM, r"\(h, c\) pair"),
    (_piece(hidden=(torch.zeros(1, 1, 32),)), LSTM, r"\(h, c\) pair"),
    (_piece(hidden=(torch.zeros(1, 1, 32), torch.zeros(1, 1, 16))), LSTM, r"float \[1, 1, 32\]"),
    (_piece(hidden=(torch.zeros(1, 1, 32), [[0.0] * 32])), LSTM, "not a tensor"),
    (_piece(hidden=torch.full((2, 1, 64), float("nan"))), GRU, "not finite"),
    (_piece(hidden=(torch.zeros(1, 1, 32), torch.full((1, 1, 32), float("inf")))), LSTM, "not finite"),
    (_piece(terminal=1), GRU, "'terminal' must be True or False"),
    (_piece(terminal="no"), GRU, "'terminal' must be True or False"),
    (_piece(terminal=None) | {"terminal": None}, GRU, "'terminal' must be True or False"),
    (_piece(terminal=False, extra_rows=0), GRU, r"has 20 rows; a non-terminal rollout of 20 steps carries 21"),
    (_piece(terminal=False, extra_rows=2), GRU, r"has 22 rows; a non-terminal rollout of 20 steps carries 21"),
    (_piece(extra_rows=1), GRU, r"has 21 rows; a terminal rollout of 20 steps carries 20"),
    (_piece(L=0, terminal=False), GRU, "at least one step"),
])
def test_malformed_rollouts_are_named(d, cfg, match):
    with pytest.raises(ValueError, match=match) as e:
        check_continuation([_piece(game_id=1), d], *cfg)
    assert "game_id=3 player_id=4" in str(e.value)


def test_observation_rows_checked_per_key():
    d = _piece(terminal=False)
    d["observations"] = dict(d["observations"], enemy_towers=d["observations"]["enemy_towers"][:20])
    with pytest.raises(ValueError, match="observations\\['enemy_towers'\\] has 20 rows"):
        check_continuation([d], *GRU)


def test_prep_refuses_before_any_upload(monkeypatch):
    """``_prepare_rollouts`` raises the ValueError before it touches a device or pins memory (no GPU needed)."""
    from dotaclient_b200.optimizer import DotaOptimizer
    from dotaclient_b200.policy import Policy

    def no_device(*a, **k):
        raise AssertionError("device or pinned-memory work before the rollouts were checked")
    opt = DotaOptimizer.__new__(DotaOptimizer)
    opt.seq_len, opt.device, opt.mask_padding = 16, torch.device("cuda", 0), False
    opt.advantage_estimator, opt._staging, opt._staging_event = "gae", {}, None
    opt.policy_base = Policy(hidden_size=64, cell="gru", num_layers=2)
    monkeypatch.setattr(torch.Tensor, "pin_memory", no_device)
    monkeypatch.setattr(torch.Tensor, "to", no_device)
    monkeypatch.setattr(torch.cuda, "Event", no_device)
    for bad in (_piece(hidden=torch.zeros(1, 1, 64)), _piece(terminal=False, extra_rows=0), _piece(terminal=0)):
        with pytest.raises(ValueError, match="game_id=3 player_id=4"):
            opt._prepare_rollouts([_piece(game_id=1), bad])


# ------------------------------------------------------------------------------------------------ segment layout
def _today(lengths, S, mask_padding):
    if mask_padding:
        return padded_segment_offsets(lengths, S)
    return np.concatenate([[0], np.cumsum([(L + S - 1) // S * S for L in lengths])]).astype(np.int64)


@pytest.mark.parametrize("mask_padding", [False, True])
@pytest.mark.parametrize("lengths", [[40, 23, 48, 7, 33], [16], [1, 32], [5]])
def test_all_terminal_layout_is_todays(lengths, mask_padding):
    off, boot, valid = rollout_segments(lengths, [True] * len(lengths), 16, mask_padding)
    assert off.dtype == boot.dtype == valid.dtype == np.int64
    assert off.tolist() == _today(lengths, 16, mask_padding).tolist()
    assert (boot == -1).all()
    assert valid.tolist() == ([n for L in lengths for n in (L, 0)] if mask_padding else lengths)


def test_mixed_layout_by_hand():
    """Lengths 40 (cut), 23 (terminal), 48 (cut, a multiple of 16), 7 (terminal), 33 (cut), S = 16."""
    lengths, terminal = [40, 23, 48, 7, 33], [False, True, False, True, False]
    off, boot, valid = rollout_segments(lengths, terminal, 16, False)
    assert off.tolist() == [0, 40, 48, 80, 128, 128, 144, 177, 192]
    assert boot.tolist() == [0, -1, -1, 1, -1, -1, 2, -1]
    assert valid.tolist() == [40, 0, 23, 48, 0, 7, 33, 0]
    off, boot, valid = rollout_segments(lengths, terminal, 16, True)
    assert off.tolist() == [0, 40, 48, 71, 80, 128, 128, 135, 144, 177, 192]
    assert boot.tolist() == [0, -1, -1, -1, 1, -1, -1, -1, 2, -1]
    assert valid.tolist() == [40, 0, 23, 0, 48, 0, 7, 0, 33, 0]


@pytest.mark.parametrize("mask_padding", [False, True])
@pytest.mark.parametrize("seed", range(4))
def test_layout_properties(seed, mask_padding):
    """Random mixes: segments tile every rollout's padded rows in order, a cut rollout is [real | padding] whatever the
    mode, its real segment names it (in order of the cut rollouts), and the real steps add up to the lengths."""
    rng = np.random.RandomState(seed)
    S = int(rng.choice([4, 16, 32]))
    lengths = [int(v) for v in rng.randint(1, 4 * S, size=9)] + [2 * S]
    terminal = [bool(v) for v in rng.rand(9) < 0.5] + [False]
    off, boot, valid = rollout_segments(lengths, terminal, S, mask_padding)
    assert (np.diff(off) >= 0).all() and off[-1] == sum((L + S - 1) // S * S for L in lengths)
    assert valid.sum() == sum(lengths) and len(boot) == len(valid) == len(off) - 1
    s, base, n_cut = 0, 0, 0
    for L, term in zip(lengths, terminal):
        Lp = (L + S - 1) // S * S
        if term and not mask_padding:
            assert (off[s], off[s + 1], boot[s]) == (base, base + Lp, -1)
            s += 1
        else:
            assert (off[s], off[s + 1], off[s + 2]) == (base, base + L, base + Lp)
            assert boot[s] == (-1 if term else n_cut) and boot[s + 1] == -1 and valid[s + 1] == 0
            s += 2
        n_cut += not term
        base += Lp
    assert s == len(boot) and sorted(b for b in boot if b >= 0) == list(range(n_cut))
    assert chunk_valid_lengths(lengths, S)[-2:] == [S, S]


# ------------------------------------------------------------------------------------------------ split_rollout
def test_split_rollout_rows_boundaries_and_flags():
    data = make_rollout(53, 9, game_id=7)
    data["behaviour_logp"] = np.arange(53 * 5, dtype=np.float32).reshape(53, 5)
    hs = [None, torch.ones(1, 1, 8), torch.full((1, 1, 8), 2.0)]
    pieces = split_rollout(data, [21, 32], initial_hiddens=hs)
    assert [p["terminal"] for p in pieces] == [False, False, True]
    assert [p["rewards"].shape[0] for p in pieces] == [21, 11, 21]
    for p, (a, b) in zip(pieces, [(0, 21), (21, 32), (32, 53)]):
        extra = 0 if p["terminal"] else 1
        for k, v in p["observations"].items():
            assert v.shape[0] == b - a + extra
            assert torch.equal(v, data["observations"][k][a:b + extra])
        for group in ("masks", "actions"):
            for k, v in p[group].items():
                assert torch.equal(v, data[group][k][a:b])
        assert np.array_equal(p["rewards"], data["rewards"][a:b])
        assert np.array_equal(p["behaviour_logp"], data["behaviour_logp"][a:b])
        assert p["game_id"] == 7 and p["weight_version"] == data["weight_version"]
    for p, q in zip(pieces, pieces[1:]):                    # row L of a piece is the next piece's row 0
        for k in p["observations"]:
            assert torch.equal(p["observations"][k][-1], q["observations"][k][0])
    assert "initial_hidden" not in pieces[0] and pieces[1]["initial_hidden"] is hs[1] and pieces[2]["initial_hidden"] is hs[2]
    check_continuation(pieces, "gru", 1, 8)
    assert "terminal" not in data and data["observations"]["env"].shape[0] == 53


def test_split_rollout_without_cuts_and_bad_cuts():
    data = make_rollout(10, 1)
    (whole,) = split_rollout(data, [])
    assert whole["terminal"] is True and torch.equal(whole["observations"]["env"], data["observations"]["env"])
    for cuts in ([0], [10], [5, 5], [6, 3]):
        with pytest.raises(ValueError, match="cuts"):
            split_rollout(data, cuts)
    with pytest.raises(ValueError, match="initial_hiddens"):
        split_rollout(data, [4], initial_hiddens=[None])


# ------------------------------------------------------------------------------------------------ the float64 oracle
def test_gae_oracle_by_hand():
    """Two steps, r = (1, 2), V = (0.5, 0.25), bootstrap b = 4."""
    adv, ret = CO.gae([1.0, 2.0], [0.5, 0.25], G, LAM, boot_value=4.0, boot_reward=4.0)
    d1 = 2.0 + G * 4.0 - 0.25
    d0 = 1.0 + G * 0.25 - 0.5
    np.testing.assert_allclose(adv, [d0 + G * LAM * d1, d1], rtol=1e-15)
    np.testing.assert_allclose(ret, [1.0 + G * 2.0 + G * G * 4.0, 2.0 + G * 4.0], rtol=1e-15)
    adv0, ret0 = CO.gae([1.0, 2.0], [0.5, 0.25], G, LAM)                    # terminal: bootstrap 0
    np.testing.assert_allclose(adv0, [d0 + G * LAM * (2.0 - 0.25), 2.0 - 0.25], rtol=1e-15)
    np.testing.assert_allclose(ret0, [1.0 + G * 2.0, 2.0], rtol=1e-15)


def test_gae_oracle_matches_the_reference_scan():
    """With its trailing element the reference's advantage_returns is this oracle (fp32 deltas vs float64: 1e-5)."""
    from oracle import ref_optimizer as RO
    rng = np.random.RandomState(3)
    r, v = rng.randn(70).astype(np.float32), rng.randn(70).astype(np.float32)
    b = np.float32(0.7)
    ra, rr = RO.advantage_returns(np.append(r, b), np.append(v, b))
    adv, ret = CO.gae(r, v, RO.GAMMA, RO.LAMBDA, boot_value=b, boot_reward=b)
    np.testing.assert_allclose(ra, adv, rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(rr, ret, rtol=1e-5, atol=1e-5)


def test_vtrace_oracle_bootstrap_by_hand():
    """One step, rho = 0.5 (both clips 1): vs = V + rho (r + gamma b - V), pg = rho (r + gamma b - V)."""
    pg, vs = VT.vtrace(np.array([1.0], np.float32), np.array([0.5], np.float32), [np.log(0.5)], G, LAM, boot=4.0)
    np.testing.assert_allclose(vs, [0.5 + 0.5 * (1.0 + G * 4.0 - 0.5)], rtol=1e-14)
    np.testing.assert_allclose(pg, [0.5 * (1.0 + G * 4.0 - 0.5)], rtol=1e-14)


def _game(n, seed):
    rng = np.random.RandomState(seed)
    return (rng.randn(n).astype(np.float32), rng.randn(n).astype(np.float32),
            rng.randn(n) * 0.7)                                         # rewards, values, log rho


@pytest.mark.parametrize("cut", [1, 16, 21, 52])
def test_whole_game_identities(cut):
    """With V the whole game's values and the cut at L: A_whole[t] = A_cut[t] + (gl)^(L-t) A_whole[L],
    ret_cut[t] = ret_whole[t] - g^(L-t) (ret_whole[L] - V[L]), vs_whole[t] - vs_cut[t] = g^(L-t) prod c_k (vs_whole[L] - V[L])
    for t < L; and the second piece, from L on, is the same scan as the whole game's tail."""
    r, v, lr = _game(53, cut)
    L = cut
    A, ret = CO.gae(r, v, G, LAM)
    a_cut, ret_cut = CO.gae(r[:L], v[:L], G, LAM, boot_value=v[L], boot_reward=v[L])
    t = np.arange(L)
    np.testing.assert_allclose(A[:L], a_cut + (G * LAM) ** (L - t) * A[L], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ret_cut, ret[:L] - G ** (L - t) * (ret[L] - v[L]), rtol=1e-12, atol=1e-12)
    a_tail, ret_tail = CO.gae(r[L:], v[L:], G, LAM)
    np.testing.assert_allclose(a_tail, A[L:], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ret_tail, ret[L:], rtol=1e-12, atol=1e-12)
    for rho_clip, c_clip in ((1.0, 1.0), (2.0, 0.8)):
        pg, vs = VT.vtrace(r, v, lr, G, LAM, rho_clip, c_clip)
        pg_cut, vs_cut = VT.vtrace(r[:L], v[:L], lr[:L], G, LAM, rho_clip, c_clip, boot=v[L])
        c = LAM * np.minimum(c_clip, np.exp(lr))
        prod = np.array([np.prod(c[s:L]) for s in range(L)])
        np.testing.assert_allclose(vs[:L] - vs_cut, G ** (L - t) * prod * (vs[L] - v[L]), rtol=1e-10, atol=1e-12)
        rhob = np.minimum(rho_clip, np.exp(lr[:L]))                       # pg_t = rhob (r + g vs_{t+1} - V)
        vs_next = np.append(vs_cut[1:], np.float64(v[L]))
        np.testing.assert_allclose(pg_cut, rhob * (r[:L] + G * vs_next - v[:L]), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(VT.vtrace(r[L:], v[L:], lr[L:], G, LAM, rho_clip, c_clip)[1], vs[L:], rtol=1e-12)
