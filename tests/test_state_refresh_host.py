"""CPU tests of the state refresh between PPO epochs (``recompute_states``): ``state_refresh_layout`` against brute-force
maps read off the batch builders (the unpacked batch built on the host from rows that carry their own coordinates, the
packed batch from its pack layout), its host checks, the setting and its CLI flag and plumbing, the header against
``_lib`` for the new entry points (arguments refused before any CUDA call), and the refusal of a batch without the
record."""
import os
import re
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
NEW_SYMBOLS = ("dc_gather_columns_fill", "dc_refresh_states")

# length 1, exact multiples of seq_len, ragged, one long rollout, and mixes that pack several tails into one column
LENGTHS = [[1], [16], [1, 1, 1], [16, 32, 48], [5, 16, 37, 1, 64, 11, 3], [130, 7, 7, 9, 15, 2, 31, 17], [100],
           [12, 12, 12, 12, 4, 4]]


def _padded(lengths, S):
    return [(int(L) + S - 1) // S * S for L in lengths]


def _host_unpacked_batch(lengths, S, mask_padding=False):
    """``DotaOptimizer._unpacked_batch`` on the host, from prepared tensors whose observation and state-buffer entries at
    (step t, rollout i) hold the forward row ``t * R + i``: the batch then names the row of every token and of every
    column's initial state.  ``mask_padding``: with prep's ``valid [S, B]`` mask of the real steps."""
    from dotaclient_b200.optimizer import DotaOptimizer, chunk_valid_lengths
    Lps = _padded(lengths, S)
    R, Lmax = len(lengths), max(Lps)
    o = DotaOptimizer.__new__(DotaOptimizer)
    o.seq_len, o.device = S, torch.device("cpu")
    o.policy_base = types.SimpleNamespace(cell="gru", num_layers=1, hidden_size=1)
    grid = (torch.arange(Lmax + 1)[:, None] * R + torch.arange(R)[None, :]).double()
    p = dict(Ls=list(lengths), Lps=Lps, Lmax=Lmax, same=all(L == Lmax for L in lengths), obs={"env": grid[:Lmax, :, None]},
             masks={}, actions={}, old_logp=torch.zeros(Lmax, R, 5), adv_c=torch.zeros(sum(Lps)),
             ret_c=torch.zeros(sum(Lps)), ybufs=[grid[:, :, None]], cbufs=[grid[:, :, None]],
             values_lr=torch.zeros(Lmax, R), valid=None, old_log_probs=None)
    if mask_padding:                                  # as _prepare_rollouts builds it
        p['valid'] = torch.arange(S)[:, None] < torch.tensor(chunk_valid_lengths(lengths, S))[None, :]
    return o._unpacked_batch(p), R, Lmax


def _brute_unpacked(lengths, S, mask_padding=False):
    batch, R, Lmax = _host_unpacked_batch(lengths, S, mask_padding)
    token_row = batch.observations["env"][..., 0].reshape(-1).long().numpy()
    obs_token = np.full(Lmax * R, -1, dtype=np.int64)
    obs_token[token_row] = np.arange(token_row.size)
    start = batch.h0[0, :, 0].long().numpy()                 # the row of each column's initial state
    dst = sorted((int(r) // R, int(r) % R, b) for b, r in enumerate(start) if r // R > 0)
    if mask_padding:                                  # a masked token still holds its row's observation
        real = np.asarray([int(r) // R < lengths[int(r) % R] for r in token_row])
        assert np.array_equal(batch.valid.reshape(-1).numpy(), real)
    return obs_token, token_row, dst


def _brute_packed(lengths, S):
    """The packed batch's tokens hold step ``lay.step`` of rollout ``lay.rollout``; a column starts from the state at
    ``h0_step`` of ``h0_rollout``, a reset at its token's step (``_packed_batch``)."""
    from dotaclient_b200.optimizer import pack_layout
    lay = pack_layout(lengths, S)
    R, Lmax = len(lengths), max(_padded(lengths, S))
    token_row = np.where(lay.rollout >= 0, lay.step * R + lay.rollout, -1).reshape(-1)
    obs_token = np.full(Lmax * R, -1, dtype=np.int64)
    for tok, row in enumerate(token_row):
        if row >= 0:
            obs_token[row] = tok
    dst = [(int(lay.h0_step[c]), int(lay.h0_rollout[c]), c) for c in range(lay.B) if lay.h0_step[c] > 0]
    for t in range(S):
        for c in range(lay.B):
            k = int(lay.reset_slot[t, c])
            if k >= 0 and lay.step[t, c] > 0:
                dst.append((int(lay.step[t, c]), int(lay.rollout[t, c]), lay.B + k * lay.B + c))
    return obs_token, token_row, sorted(dst)


@pytest.mark.parametrize("lengths", LENGTHS)
@pytest.mark.parametrize("S", [16, 4])
@pytest.mark.parametrize("pack,mask_padding", [(False, False), (False, True), (True, True)])
def test_layout_against_the_batch(lengths, S, pack, mask_padding):
    """``mask_padding`` changes neither layout (a masked step's observation is still in the batch, and the unpacked batch
    built with prep's ``valid`` mask gives the same maps), so one map serves both; packing needs it."""
    from dotaclient_b200.optimizer import check_state_refresh_layout, pack_layout, state_refresh_layout
    lay = state_refresh_layout(lengths, S, pack)
    obs_token, token_row, dst = _brute_packed(lengths, S) if pack else _brute_unpacked(lengths, S, mask_padding)
    assert np.array_equal(lay.obs_token, obs_token) and np.array_equal(lay.token_row, token_row)
    got = sorted(zip(lay.step.tolist(), lay.rollout.tolist(), lay.slot.tolist()))
    assert got == dst
    assert np.all(np.diff(lay.step) >= 0) and np.all(lay.step % S == 0)
    # every chunk start after a rollout's first has exactly one destination
    assert lay.step.size == sum(-(-int(L) // S) - 1 for L in lengths)
    B = token_row.size // S
    check_state_refresh_layout(lay, B, pack_layout(lengths, S).K if pack else 0)


def test_layout_reuses_a_given_pack_layout():
    from dotaclient_b200.optimizer import pack_layout, state_refresh_layout
    lengths, S = [130, 7, 7, 9, 15, 2, 31, 17], 16
    a = state_refresh_layout(lengths, S, True, layout=pack_layout(lengths, S))
    b = state_refresh_layout(lengths, S, True)
    assert all(np.array_equal(x, y) for x, y in zip(a[2:], b[2:]))


def test_layout_check_rejects_bad_tables():
    from dotaclient_b200.optimizer import check_state_refresh_layout, pack_layout, state_refresh_layout
    lengths, S = [130, 7, 7, 9, 15, 2, 31, 17], 16
    lay = state_refresh_layout(lengths, S, True)
    B, K = pack_layout(lengths, S).B, pack_layout(lengths, S).K
    check_state_refresh_layout(lay, B, K)
    bad = [lay._replace(slot=np.concatenate([lay.slot[:-1], lay.slot[:1]])),          # a slot twice
           lay._replace(slot=lay.slot + B + K * B),                                    # outside the tables
           lay._replace(step=lay.step[::-1].copy()),                                   # not sorted
           lay._replace(step=lay.step * 0),                                            # step 0 is data
           lay._replace(rollout=lay.rollout + len(lengths)),
           lay._replace(obs_token=lay.obs_token + S * B),
           lay._replace(token_row=lay.token_row - 5),
           lay._replace(rollout=lay.rollout[1:])]
    for b in bad:
        with pytest.raises(ValueError, match="state refresh layout"):
            check_state_refresh_layout(b, B, K)


# ------------------------------------------------------------------------------------------------ settings and CLI
def test_settings_validation():
    from dotaclient_b200.optimizer import check_ppo_settings
    base = (0.98, 0.97, 0.1, 0.5)
    check_ppo_settings(*base, recompute_states=True)
    check_ppo_settings(*base, recompute_states=True, recompute_advantages=True)
    for bad in (1, 0, "yes", None):
        with pytest.raises(ValueError, match="recompute_states"):
            check_ppo_settings(*base, recompute_states=bad)


def test_constructor_and_main_refuse_bad_settings_up_front():
    from dotaclient_b200.optimizer import DotaOptimizer, main
    with pytest.raises(ValueError, match="recompute_states"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, recompute_states=1)
    with pytest.raises(ValueError, match="recompute_states"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, recompute_states="on")


def test_cli_flag():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).recompute_states is False
    assert p.parse_args(["--recompute-states"]).recompute_states is True
    assert "--recompute-states" in p.format_help()


@pytest.mark.parametrize("kw", [{}, {"recompute_states": True}, {"recompute_states": True, "recompute_advantages": True}])
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
    assert seen["recompute_states"] is kw.get("recompute_states", False) and seen["ran"]


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
    assert _lib.SIGNATURES["dc_gather_columns_fill"] == _lib.SIGNATURES["dc_gather_columns"]
    text = open(HEADER).read()
    assert re.search(r"#define DC_REFRESH_MAX_LAYERS %d\b" % _lib.REFRESH_MAX_LAYERS, text)
    from dotaclient_b200.optimizer import DotaOptimizer
    assert DotaOptimizer.MAX_LAYERS <= _lib.REFRESH_MAX_LAYERS


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_new_symbols_are_exported_and_check_their_arguments(lib):
    from dotaclient_b200 import _lib
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name), name
    assert lib.dc_version() >= 112
    p = 4096
    ptrs = (_lib._c.c_void_p * 2)(p, p)
    # (n_layers, H, h_bufs, c_bufs, R, t0, step, rollout, slot, n, B, K, h0, c0, reset_h, reset_c, partial, acc, stream)
    rs = lib.dc_refresh_states
    assert rs(1, 128, ptrs, None, 4, 0, p, p, p, 0, 4, 0, p, None, None, None, p, p, None) == 0      # nothing to do
    cases = [((0, 128, ptrs, None, 4, 0, p, p, p, 3, 4, 0, p, None, None, None, p, p, None), b"n_layers"),
             ((17, 128, ptrs, None, 4, 0, p, p, p, 3, 4, 0, p, None, None, None, p, p, None), b"n_layers"),
             ((1, 100, ptrs, None, 4, 0, p, p, p, 3, 4, 0, p, None, None, None, p, p, None), b"H=100"),
             ((1, 128, ptrs, None, 0, 0, p, p, p, 3, 4, 0, p, None, None, None, p, p, None), b"R=0"),
             ((1, 128, ptrs, None, 4, 0, p, p, p, -1, 4, 0, p, None, None, None, p, p, None), b"n=-1"),
             ((1, 128, ptrs, None, 4, 0, p, p, p, 3, 4, 0, p, None, None, None, p, None, None), b"null acc"),
             ((1, 128, ptrs, None, 4, 0, None, p, p, 3, 4, 0, p, None, None, None, p, p, None), b"null pointer"),
             ((1, 128, ptrs, ptrs, 4, 0, p, p, p, 3, 4, 0, p, None, None, None, p, p, None), b"c_bufs and c0"),
             ((1, 128, ptrs, None, 4, 0, p, p, p, 3, 4, 2, p, None, None, None, p, p, None), b"K=2"),
             ((1, 128, ptrs, None, 4, 0, p, p, p, 3, 4, 0, p + 4, None, None, None, p, p, None), b"16-byte"),
             ((1, 128, ptrs, None, 4, 0, p, p, p, 3, 4, 0, p, None, None, None, p + 8, p, None), b"16-byte")]
    for args, msg in cases:
        assert rs(*args) == -1 and msg in lib.dc_last_error(), (args, lib.dc_last_error())
    bad_ptrs = (_lib._c.c_void_p * 1)(p + 4)
    assert rs(1, 128, bad_ptrs, None, 4, 0, p, p, p, 3, 4, 0, p, None, None, None, p, p, None) == -1
    assert b"aligned" in lib.dc_last_error()
    # the fill gather checks as dc_gather_columns does, under its own name
    d = (_lib.GatherDesc * 1)(_lib.GatherDesc(p, p * 2, 1, 0, 16))
    assert lib.dc_gather_columns_fill(d, 1, p, 0, None) == 0
    rc = lib.dc_gather_columns_fill(d, 1, p, 4, None)
    assert rc == -1 and b"dc_gather_columns_fill" in lib.dc_last_error() and b"src_cols=0" in lib.dc_last_error()
    assert lib.dc_gather_columns_fill(d, 33, p, 4, None) == -1 and b"n_desc" in lib.dc_last_error()
    d = (_lib.GatherDesc * 1)(_lib.GatherDesc(p, p * 2, 1, 4, 0))
    assert lib.dc_gather_columns_fill(d, 1, p, 4, None) == -1 and b"row_bytes" in lib.dc_last_error()


def test_refresh_states_wrapper_checks_before_any_launch():
    from dotaclient_b200 import ops
    h = torch.zeros(1, 4, 32)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.refresh_states([torch.zeros(3, 2, 32)], None, 0, torch.zeros(1, dtype=torch.int64),
                           torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int64), h, None, None, None,
                           torch.zeros(2, dtype=torch.float64))
    with pytest.raises(ValueError, match="index"):
        ops.gather_columns_fill([], torch.zeros(3, dtype=torch.int32))


# ------------------------------------------------------------------------------------------------ the batch
def _batch(S=4, B=3):
    from dotaclient_b200.optimizer import ExperienceBatch
    from dotaclient_b200.policy import Policy
    from dotaclient_b200.synthetic import HEAD_SIZES
    obs = {k: torch.zeros(S, B, 2) for k in Policy.INPUT_KEYS}
    heads = {k: torch.zeros(S, B, n, dtype=torch.bool) for k, n in HEAD_SIZES.items()}
    return ExperienceBatch(obs, heads, dict(heads), torch.zeros(S, B, 5), torch.zeros(S, B), torch.zeros(S, B),
                           torch.zeros(1, B, 8))


def test_record_is_not_a_field():
    from dotaclient_b200.optimizer import ExperienceBatch, StateRefresh, state_refresh_layout
    b = _batch()
    assert b.state_refresh is None and "state_refresh" not in ExperienceBatch.FIELDS
    n = len(list(b.tensors()))
    lay = state_refresh_layout([4, 8], 4, False)
    z = torch.zeros(0, dtype=torch.int64)
    b.state_refresh = StateRefresh(lay, z, z, z, z, z, None, None, None, None, None, None)
    assert len(list(b.tensors())) == n and b.graph_key() == _batch().graph_key()
    assert b.map(lambda v: v.clone()).state_refresh is None


def _stub(epochs, states, advantages=False, M=1):
    from dotaclient_b200.optimizer import DotaOptimizer
    o = DotaOptimizer.__new__(DotaOptimizer)
    o.epochs, o.recompute_states, o.recompute_advantages, o.num_minibatches = epochs, states, advantages, M

    def launched(*a, **k):
        raise AssertionError("a step was launched")
    o.train = o._refresh_advantages = o._refresh_states = launched
    return o


def test_train_epochs_refuses_a_batch_without_the_record():
    with pytest.raises(ValueError, match="recompute_states"):
        _stub(3, True).train_epochs(_batch())
    b = _batch()
    b.refresh = object()                                   # the advantage refresh's data alone is not enough
    with pytest.raises(ValueError, match="recompute_states"):
        _stub(2, True, advantages=True).train_epochs(b)


def test_drift_of_the_sums():
    from dotaclient_b200.optimizer import _drift
    assert _drift(0.0, 0.0) == 0.0 and _drift(4.0, 16.0) == 0.5 and _drift(1.0, 0.0) == float("inf")


# ------------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("advantages", [False, True])
def test_oracle_refresh_at_the_prep_weights_is_prep(advantages):
    """At unchanged weights the float64 whole-rollout rerun gives the chunk start states the oracle's own prep stored
    (and, with the advantages, prep's advantages, V(s_L) of cut rollouts included)."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import state_refresh_oracle as SO
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
    o = SO.StateRefreshRefOptimizer(StackedRefPolicy(32, "lstm", 1), seq_len=S, recompute_advantages=advantages)
    seqs = o.prepare(rollouts)
    h0 = [tuple(x.clone() for x in s.hidden) for s in seqs]
    adv0 = torch.cat([s.advantages for s in seqs]).numpy()
    o.refresh(seqs, rollouts)
    for s, h in zip(seqs, h0):
        for a, b in zip(s.hidden, h):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(torch.cat([s.advantages for s in seqs]).numpy(), adv0, rtol=1e-4, atol=2e-6)
    assert len(seqs) > len(rollouts)                       # chunks after the first exist
