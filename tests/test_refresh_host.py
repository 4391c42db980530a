"""CPU tests of the advantage refresh between PPO epochs (``recompute_advantages``): the token map against brute-force maps
built from the batch's own layout, the setting and its CLI flag and plumbing, the header against ``_lib`` for the indexed
scans (arguments refused before any CUDA call), and the refusal of a batch without refresh data."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
NEW_SYMBOLS = ("dc_gae_scan_indexed", "dc_vtrace_scan_indexed")

# ragged, exact multiples of seq_len, length 1, one long rollout, and a mix that packs several tails into one column
LENGTHS = [[1], [16], [1, 1, 1], [16, 32, 48], [5, 16, 37, 1, 64, 11, 3], [130, 7, 7, 9, 15, 2, 31, 17],
           [100], [12, 12, 12, 12, 4, 4]]


def _padded(lengths, S):
    return [(int(L) + S - 1) // S * S for L in lengths]


def _brute_unpacked(lengths, S, mask_padding):
    """Where ``batch_from_rollouts`` puts rollout-major row r: its advantages are ``adv_c.view(B, S).t()``."""
    Lps = _padded(lengths, S)
    n = sum(Lps)
    B = n // S
    held = torch.arange(n).view(B, S).t().contiguous().numpy()          # [S, B]: the row each token holds
    tok = np.full(n, -1, dtype=np.int64)
    for t in range(S):
        for c in range(B):
            tok[held[t, c]] = t * B + c
    if mask_padding:
        base = 0
        for L, Lp in zip(lengths, Lps):
            tok[base + L:base + Lp] = -1
            base += Lp
    return tok


def _brute_packed(lengths, S):
    """Where the packed batch puts rollout-major row r: token (t, c) holds step ``lay.step[t, c]`` of rollout
    ``lay.rollout[t, c]``."""
    from dotaclient_b200.optimizer import pack_layout
    Lps = _padded(lengths, S)
    lay = pack_layout(lengths, S)
    tok = np.full(sum(Lps), -1, dtype=np.int64)
    for t in range(S):
        for c in range(lay.B):
            i = int(lay.rollout[t, c])
            if i >= 0:
                tok[sum(Lps[:i]) + int(lay.step[t, c])] = t * lay.B + c
    return tok


@pytest.mark.parametrize("lengths", LENGTHS)
@pytest.mark.parametrize("S", [16, 4])
@pytest.mark.parametrize("mask_padding", [False, True])
def test_token_map_unpacked(lengths, S, mask_padding):
    from dotaclient_b200.optimizer import refresh_token_map
    tok = refresh_token_map(lengths, S, False, mask_padding)
    want = _brute_unpacked(lengths, S, mask_padding)
    assert tok.dtype == np.int64 and np.array_equal(tok, want)
    real = tok[tok >= 0]
    assert np.unique(real).size == real.size
    assert (tok >= 0).sum() == (sum(lengths) if mask_padding else sum(_padded(lengths, S)))


@pytest.mark.parametrize("lengths", LENGTHS)
@pytest.mark.parametrize("S", [16, 4])
def test_token_map_packed(lengths, S):
    """Packing needs mask_padding: exactly the real steps map to tokens, each to its own."""
    from dotaclient_b200.optimizer import refresh_token_map, sequence_count
    tok = refresh_token_map(lengths, S, True, True)
    assert np.array_equal(tok, _brute_packed(lengths, S))
    real = tok[tok >= 0]
    assert real.size == sum(lengths) and np.unique(real).size == real.size
    assert real.max() < S * sequence_count(lengths, S, pack=True)


def test_token_map_matches_the_observation_layout():
    """The unpacked observations are ``chunk_columns`` of the [L_max, R] tensors: a token holds the observation of the
    row the map sends to it."""
    from dotaclient_b200.optimizer import chunk_columns, refresh_token_map
    lengths, S = [5, 16, 37, 1, 64], 16
    Lps = _padded(lengths, S)
    Lmax, R = max(Lps), len(lengths)
    obs = torch.full((Lmax, R), -1, dtype=torch.int64)
    base = np.concatenate([[0], np.cumsum(Lps)[:-1]])
    for i, Lp in enumerate(Lps):
        obs[:Lp, i] = torch.arange(Lp) + int(base[i])
    flat = chunk_columns(obs, Lps, S).reshape(-1).numpy()
    tok = refresh_token_map(lengths, S, False, False)
    assert np.array_equal(flat[tok], np.arange(sum(Lps)))


def test_packed_rows_is_the_packed_batch_gather():
    """``_packed_batch`` gathers the advantages of prep's rows with ``packed_rows``; its inverse is the token map."""
    from dotaclient_b200.optimizer import pack_layout, packed_rows, refresh_token_map
    lengths, S = [130, 7, 7, 9, 15, 2, 31, 17], 16
    rows = packed_rows(pack_layout(lengths, S), _padded(lengths, S)).reshape(-1)
    tok = refresh_token_map(lengths, S, True, True)
    assert np.array_equal(rows[tok[tok >= 0]], np.flatnonzero(tok >= 0))


# ------------------------------------------------------------------------------------------------ settings and CLI
def test_settings_validation():
    from dotaclient_b200.optimizer import check_ppo_settings
    base = (0.98, 0.97, 0.1, 0.5)
    check_ppo_settings(*base, recompute_advantages=True)
    check_ppo_settings(*base, recompute_advantages=False)
    for bad in (1, 0, "yes", None):
        with pytest.raises(ValueError, match="recompute_advantages"):
            check_ppo_settings(*base, recompute_advantages=bad)


def test_constructor_and_main_refuse_bad_settings_up_front():
    from dotaclient_b200.optimizer import DotaOptimizer, main
    with pytest.raises(ValueError, match="recompute_advantages"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, recompute_advantages=1)
    with pytest.raises(ValueError, match="recompute_advantages"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, recompute_advantages="on")


def test_cli_flag():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).recompute_advantages is False
    assert p.parse_args(["--recompute-advantages"]).recompute_advantages is True
    assert "--recompute-advantages" in p.format_help()


@pytest.mark.parametrize("kw", [{}, {"recompute_advantages": True}])
def test_main_passes_the_flag_to_the_optimizer(kw, monkeypatch):
    from dotaclient_b200 import optimizer as O
    seen = {}

    class Fake:
        mq = None

        def __init__(self, **k):
            seen.update(k)

        def run(self):
            seen["ran"] = True

    monkeypatch.setattr(O, "DotaOptimizer", Fake)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    O.main("x", 0, 3, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, **kw)
    assert seen["recompute_advantages"] is kw.get("recompute_advantages", False) and seen["ran"]


# ------------------------------------------------------------------------------------------------ C ABI
def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(dc_\w+)\s*\(([^;{]*?)\)\s*;", text):
        args = m.group(2).strip()
        protos[m.group(1)] = 0 if args in ("", "void") else args.count(",") + 1
    return protos


def test_header_and_lib_table_agree():
    from dotaclient_b200 import _lib
    protos = _declared()
    for name in NEW_SYMBOLS:
        assert name in protos and name in _lib.SIGNATURES, name
        assert len(_lib.SIGNATURES[name][1]) == protos[name], name
    # the indexed entry points take the existing ones' arguments plus the value stride and the token map
    assert protos["dc_gae_scan_indexed"] == protos["dc_gae_scan"] + 2
    assert protos["dc_vtrace_scan_indexed"] == protos["dc_vtrace_scan"] + 2


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_new_symbols_are_exported_and_check_their_arguments(lib):
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name), name
    assert lib.dc_version() >= 111
    p = 4096
    # (rewards, n_sub, values, ld, tok, seg_off, n_seg, boot_value, boot_reward, gamma, lam, adv, ret, stream)
    gae = lib.dc_gae_scan_indexed
    assert gae(p, 10, p, 128, p, p, 0, None, None, 0.98, 0.97, p, p, None) == 0          # nothing to do
    rc = gae(p, 10, p, 0, p, p, 4, None, None, 0.98, 0.97, p, p, None)
    assert rc == -1 and b"ld_values" in lib.dc_last_error()
    rc = gae(p, 10, p, 128, None, p, 4, None, None, 0.98, 0.97, p, p, None)
    assert rc == -1 and b"null pointer" in lib.dc_last_error()
    rc = gae(p, 0, p, 128, p, p, 4, None, None, 0.98, 0.97, p, p, None)
    assert rc == -1 and b"n_sub" in lib.dc_last_error()
    assert gae(p, 10, p, 128, p, p, -1, None, None, 0.98, 0.97, p, p, None) == -1
    # (rewards, n_sub, values, ld, logp_target, logp_behaviour, tok, seg_off, n_seg, valid_len, boot_value, gamma, lam,
    #  rho_clip, c_clip, pg_adv, vs, seg_stats, stream)
    vt = lib.dc_vtrace_scan_indexed
    assert vt(p, 10, p, 128, p, p, p, p, 0, None, None, 0.98, 0.97, 1.0, 1.0, p, p, None, None) == 0
    rc = vt(p, 10, p, 1, p, p, None, p, 4, None, None, 0.98, 0.97, 1.0, 1.0, p, p, None, None)
    assert rc == -1 and b"null pointer" in lib.dc_last_error()
    rc = vt(p, 10, p, 0, p, p, p, p, 4, None, None, 0.98, 0.97, 1.0, 1.0, p, p, None, None)
    assert rc == -1 and b"ld_values" in lib.dc_last_error()
    rc = vt(p, 10, p, 1, p, p, p, p, 4, None, None, 0.98, 0.97, 0.0, 1.0, p, p, None, None)
    assert rc == -1 and b"rho_clip" in lib.dc_last_error()


# ------------------------------------------------------------------------------------------------ the batch
def _batch(S=4, B=3):
    from dotaclient_b200.optimizer import ExperienceBatch
    from dotaclient_b200.policy import Policy
    from dotaclient_b200.synthetic import HEAD_SIZES
    obs = {k: torch.zeros(S, B, 2) for k in Policy.INPUT_KEYS}
    heads = {k: torch.zeros(S, B, n, dtype=torch.bool) for k, n in HEAD_SIZES.items()}
    return ExperienceBatch(obs, heads, dict(heads), torch.zeros(S, B, 5), torch.zeros(S, B), torch.zeros(S, B),
                           torch.zeros(1, B, 8))


def test_refresh_data_is_not_a_field():
    from dotaclient_b200.optimizer import AdvantageRefresh, ExperienceBatch
    b = _batch()
    assert b.refresh is None and "refresh" not in ExperienceBatch.FIELDS
    n = len(list(b.tensors()))
    b.refresh = AdvantageRefresh(torch.zeros(12, 10), torch.tensor([0, 12]), None, torch.arange(12), None, None)
    assert len(list(b.tensors())) == n and b.graph_key() == _batch().graph_key()
    assert b.map(lambda v: v.clone()).refresh is None


def _stub(epochs, on, M=1):
    from dotaclient_b200.optimizer import DotaOptimizer
    o = DotaOptimizer.__new__(DotaOptimizer)
    o.epochs, o.recompute_advantages, o.num_minibatches = epochs, on, M

    def launched(*a, **k):
        raise AssertionError("a step was launched")
    o.train = o._refresh_advantages = launched
    return o


def test_train_epochs_refuses_a_batch_without_refresh_data():
    with pytest.raises(ValueError, match="recompute_advantages"):
        _stub(3, True).train_epochs(_batch())
    with pytest.raises(ValueError, match="recompute_advantages"):
        _stub(2, True, M=3).train_epochs(_batch())


# ------------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("estimator", ["gae", "vtrace"])
@pytest.mark.parametrize("mask_padding", [False, True])
def test_oracle_refresh_at_the_prep_weights_is_prep(estimator, mask_padding):
    """At unchanged weights the float64 refresh reproduces the oracle's own fp32 prep."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import refresh_oracle as RF
    from stacked_oracle import StackedRefPolicy
    from dotaclient_b200.synthetic import make_rollout
    torch.manual_seed(7)
    S = 8
    o = RF.RefreshRefOptimizer(StackedRefPolicy(32, "lstm", 1), seq_len=S, estimator=estimator, mask_padding=mask_padding)
    rollouts = [make_rollout(L, 40 + i) for i, L in enumerate((13, 8, 1, 20))]
    g = np.random.default_rng(1)
    for r in rollouts:
        r["behaviour_logp"] = (g.standard_normal((r["rewards"].shape[0], 5)) * 0.1 - 1.0).astype(np.float32)
    seqs = o.prepare(rollouts)
    adv0 = torch.cat([s.advantages for s in seqs]).numpy()
    ret0 = torch.cat([s.returns for s in seqs]).numpy()
    o.refresh(seqs, rollouts)
    adv1 = torch.cat([s.advantages for s in seqs]).numpy()
    ret1 = torch.cat([s.returns for s in seqs]).numpy()
    np.testing.assert_allclose(adv1, adv0, rtol=1e-4, atol=2e-6)
    np.testing.assert_allclose(ret1, ret0, rtol=1e-4, atol=2e-6)
    assert np.abs(adv0).max() > 1e-2


def test_oracle_refresh_keeps_the_bootstraps_of_cut_rollouts():
    """Rollouts cut from a longer game: at unchanged weights the refresh, with prep's V(s_L), reproduces prep."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import refresh_oracle as RF
    from stacked_oracle import StackedRefPolicy
    from dotaclient_b200.synthetic import make_rollout, split_rollout
    torch.manual_seed(7)
    S, rollouts = 8, []
    for i, (L, terminal) in enumerate(((20, False), (13, True), (9, False))):
        r = make_rollout(L + (0 if terminal else 1), 50 + i)
        if not terminal:
            r = split_rollout(r, [L])[0]
        r["initial_hidden"] = tuple(0.3 * torch.randn(1, 1, 32) for _ in range(2))
        rollouts.append(r)
    for mask_padding in (False, True):
        o = RF.RefreshRefOptimizer(StackedRefPolicy(32, "lstm", 1), seq_len=S, mask_padding=mask_padding)
        seqs = o.prepare(rollouts)
        assert [t for t, _ in o._ends] == [False, True, False] and o._ends[0][1] != 0.0
        adv0 = torch.cat([s.advantages for s in seqs]).numpy()
        o.refresh(seqs, rollouts)
        np.testing.assert_allclose(torch.cat([s.advantages for s in seqs]).numpy(), adv0, rtol=1e-4, atol=2e-6)
