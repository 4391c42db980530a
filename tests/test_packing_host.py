"""CPU tests of sequence packing (``DotaOptimizer(pack_sequences=True)``): the packed layout, the settings and CLI flag, the
packed pull rule of ``run_iteration``, the batch fields, and the argument checks of ``dc_rnn_seq_fwd_reset`` /
``dc_rnn_seq_bwd_reset`` (which run before any CUDA call)."""
import os
import re
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")

CASES = [
    ([40, 23, 48, 7, 16], 16),
    ([5], 16),                       # R = 1, shorter than S: all tail
    ([64], 16),                      # R = 1, a multiple of S: no tail
    ([3, 3, 3, 3, 3, 3], 16),        # many tails share one column
    ([1000, 1111, 1234, 1399, 1400, 1024, 1025], 512),
    ([17, 31, 15, 1, 2, 14, 16, 32, 48], 16),
]


def _check_layout(lengths, S):
    from dotaclient_b200.optimizer import pack_layout
    lay = pack_layout(lengths, S)
    B, K = lay.B, lay.K
    for a in (lay.rollout, lay.step, lay.reset_slot):
        assert a.shape == (S, B)
    assert lay.reset_slot.dtype == np.int32
    # every real step appears exactly once
    real = lay.rollout >= 0
    seen = sorted(zip(lay.rollout[real].tolist(), lay.step[real].tolist()))
    assert seen == [(i, t) for i, L in enumerate(lengths) for t in range(L)]
    assert (lay.step[~real] == -1).all()
    # full chunks: columns 0 .. n_full-1, rollout by rollout, each one chunk from the state at its first step
    full = [(i, j) for i, L in enumerate(lengths) for j in range(L // S)]
    assert lay.n_full == len(full)
    for c, (i, j) in enumerate(full):
        assert (lay.rollout[:, c] == i).all() and lay.step[:, c].tolist() == list(range(j * S, (j + 1) * S))
        assert (lay.h0_rollout[c], lay.h0_step[c]) == (i, j * S)
        assert (lay.reset_slot[:, c] == -1).all()
    # tail columns: whole tails back to back from row 0, padding only at the end, resets at every later tail's first step
    n_mid = []
    for c in range(lay.n_full, B):
        col_r, col_t = lay.rollout[:, c], lay.step[:, c]
        used = int((col_r >= 0).sum())
        assert used > 0 and (col_r[:used] >= 0).all() and (col_r[used:] == -1).all()      # no column exceeds S
        starts = [0] + [t for t in range(1, used) if col_r[t] != col_r[t - 1]]
        assert (lay.h0_rollout[c], lay.h0_step[c]) == (col_r[0], col_t[0])
        for n, t0 in enumerate(starts):
            i = int(col_r[t0])
            L = lengths[i]
            t1 = starts[n + 1] if n + 1 < len(starts) else used
            assert col_t[t0:t1].tolist() == list(range(L - L % S, L))                  # the whole tail, never split
            assert lay.reset_slot[t0, c] == (-1 if n == 0 else n - 1)
        assert (lay.reset_slot[[t for t in range(S) if t not in starts[1:]], c] == -1).all()
        n_mid.append(len(starts) - 1)
    assert K == max(n_mid, default=0)
    return lay


@pytest.mark.parametrize("lengths,S", CASES)
def test_pack_layout_properties(lengths, S):
    lay = _check_layout(lengths, S)
    from dotaclient_b200.optimizer import pack_layout, sequence_count
    again = pack_layout(list(lengths), S)                                         # deterministic
    for f in lay._fields:
        assert np.array_equal(np.asarray(getattr(lay, f)), np.asarray(getattr(again, f)))
    assert sequence_count(lengths, S, pack=True) == lay.B <= sequence_count(lengths, S)
    assert sequence_count(lengths, S) == sum((L + S - 1) // S for L in lengths)


def test_pack_layout_small_cases():
    from dotaclient_b200.optimizer import pack_layout
    lay = pack_layout([5], 16)                          # shorter than S: one tail column from the rollout's initial state
    assert (lay.B, lay.K, lay.n_full) == (1, 0, 0) and (lay.h0_rollout[0], lay.h0_step[0]) == (0, 0)
    lay = pack_layout([32], 16)                         # a multiple of S: no tail, nothing to pack
    assert (lay.B, lay.K, lay.n_full) == (2, 0, 2) and (lay.rollout >= 0).all()
    lay = pack_layout([10, 6, 3, 3], 16)                # first-fit-decreasing: [10, 6] then [3, 3]
    assert (lay.B, lay.K) == (2, 1)
    assert lay.rollout[:, 0].tolist() == [0] * 10 + [1] * 6 and lay.reset_slot[10, 0] == 0
    assert lay.rollout[:6, 1].tolist() == [2] * 3 + [3] * 3 and lay.reset_slot[3, 1] == 0
    lay = pack_layout([4, 4, 4, 4], 16)                 # ties by rollout order; four tails in one column: K = 3
    assert (lay.B, lay.K) == (1, 3) and lay.rollout[:, 0].tolist() == sum([[i] * 4 for i in range(4)], [])
    assert lay.reset_slot[[0, 4, 8, 12], 0].tolist() == [-1, 0, 1, 2]


def test_pack_layout_random():
    rng = np.random.default_rng(3)
    for _ in range(20):
        S = int(rng.choice([4, 16, 64]))
        lengths = rng.integers(1, 5 * S, size=int(rng.integers(1, 30))).tolist()
        _check_layout(lengths, S)


def test_check_reset_slots():
    from dotaclient_b200.optimizer import check_reset_slots
    rs = np.full((4, 3), -1, dtype=np.int32)
    rs[2, 0], rs[1, 1] = 0, 1
    check_reset_slots(rs, 2)
    with pytest.raises(ValueError, match="outside"):
        check_reset_slots(rs, 1)
    rs[3, 0] = 0                                        # row (0, column 0) used twice
    with pytest.raises(ValueError, match="two tokens"):
        check_reset_slots(rs, 2)
    with pytest.raises(ValueError, match="outside"):
        check_reset_slots(np.full((2, 2), -2, dtype=np.int32), 1)


def test_cli_flag_and_default():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).pack_sequences is False
    a = p.parse_args(["--pack-sequences", "--mask-padding"])
    assert a.pack_sequences is True and a.mask_padding is True
    assert "--pack-sequences" in p.format_help()


def test_packing_needs_mask_padding():
    """Refused with ValueError before any device work, by check_ppo_settings, the constructor and main()."""
    from dotaclient_b200.optimizer import DotaOptimizer, check_ppo_settings, main
    with pytest.raises(ValueError, match="mask_padding"):
        check_ppo_settings(0.98, 0.97, 0.1, 0.5, pack_sequences=True)
    with pytest.raises(ValueError, match="pack_sequences"):
        check_ppo_settings(0.98, 0.97, 0.1, 0.5, mask_padding=True, pack_sequences=1)
    with pytest.raises(ValueError, match="mask_padding"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, pack_sequences=True)
    with pytest.raises(ValueError, match="mask_padding"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, pack_sequences=True)
    check_ppo_settings(0.98, 0.97, 0.1, 0.5, mask_padding=True, pack_sequences=True)


def test_packed_pull_rule():
    """run_iteration pulls rollouts until the PACKED layout holds min_seq_per_epoch sequences."""
    from dotaclient_b200.optimizer import DotaOptimizer, sequence_count

    def pulls(lengths, S, min_seq, pack):
        stub = types.SimpleNamespace(seq_len=S, min_seq_per_epoch=min_seq, pack_sequences=pack)
        lens, n = [], 0
        for L in lengths:
            if n >= min_seq:
                break
            lens.append(L)
            n = DotaOptimizer._pulled_sequences(stub, lens, n)
        return lens, n

    rng = np.random.default_rng(5)
    lengths = rng.integers(1000, 1401, size=400).tolist()
    for S, min_seq in ((512, 64), (1024, 40), (128, 300)):
        lens_u, n_u = pulls(lengths, S, min_seq, False)
        lens_p, n_p = pulls(lengths, S, min_seq, True)
        assert n_u == sequence_count(lens_u, S) >= min_seq
        assert n_p == sequence_count(lens_p, S, pack=True) >= min_seq
        assert sequence_count(lens_p[:-1], S, pack=True) < min_seq            # not one rollout more than needed
        assert len(lens_p) >= len(lens_u)


def test_experience_batch_reset_fields_are_optional_and_last():
    from dotaclient_b200.optimizer import ExperienceBatch
    S, B, K, LH = 4, 3, 2, 8
    kw = dict(observations={"env": torch.zeros(S, B, 3)}, masks={"enum": torch.ones(S, B, 4, dtype=torch.bool)},
              actions={"enum": torch.zeros(S, B, 4, dtype=torch.bool)}, old_logp=torch.zeros(S, B, 5),
              advantages=torch.zeros(S, B), returns=torch.zeros(S, B), h0=torch.zeros(1, B, LH),
              valid=torch.ones(S, B, dtype=torch.bool))
    plain = ExperienceBatch(**kw)
    packed = ExperienceBatch(**kw, reset_slot=torch.full((S, B), -1, dtype=torch.int32), reset_h=torch.zeros(K, B, LH))
    names_plain = [k for _, k, _ in plain.tensors()]
    names_packed = [k for _, k, _ in packed.tensors()]
    assert names_packed[:len(names_plain)] == names_plain and names_packed[len(names_plain):] == ["reset_slot", "reset_h"]
    assert plain.graph_key() == (S, B, False, 'valid') and packed.graph_key() == (S, B, False, 'valid', ('reset', K))
    assert plain.reset() is None and packed.reset()[0] is packed.reset_slot
    cloned = packed.map(lambda v: v.clone())
    assert cloned.reset_h.shape == (K, B, LH) and cloned.reset_c is None


def _params(name):
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\b%s\s*\(([^)]*)\)" % name, text)
    return [a.strip() for a in m.group(1).split(",")]


def test_header_and_lib_table_agree_on_the_reset_entry_points():
    from dotaclient_b200 import _lib
    for name, base, extra in (("dc_rnn_seq_fwd_reset", "dc_rnn_seq_fwd", 4), ("dc_rnn_seq_bwd_reset", "dc_rnn_seq_bwd", 3)):
        assert len(_params(name)) == len(_lib.SIGNATURES[name][1]) == len(_params(base)) + extra


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_reset_entry_points_check_their_arguments(lib):
    """Argument errors return before any CUDA call (this box may have no GPU)."""
    one = 4096                                   # never dereferenced: validation fails first
    fwd, bwd = lib.dc_rnn_seq_fwd_reset, lib.dc_rnn_seq_bwd_reset
    assert fwd(7, one, one, one, one, one, one, one, one, 1, 4, 4, 128, one, None) == -1
    assert b"unknown cell" in lib.dc_last_error()
    assert fwd(1, one, one, one, one, one, one, one, one, 1, 4, 4, 130, one, None) == -2
    assert fwd(1, one, one, one, one, one, None, one, one, 1, 4, 4, 128, one, None) == -1
    assert b"dc_rnn_seq_fwd_reset: null reset_slot" in lib.dc_last_error()
    assert fwd(1, one, one, one, one, one, one, one, None, 1, 4, 4, 128, one, None) == -1     # the forward needs pre
    assert b"null reset table" in lib.dc_last_error()
    assert fwd(1, one, one, one, one, one, one, one, one, -1, 4, 4, 128, one, None) == -1
    assert fwd(1, None, one, one, one, one, one, one, one, 1, 4, 4, 128, one, None) == -1
    assert bwd(1, one, one, one, one, one, None, None, one, one, one, None, 1, 4, 4, 128, one, None) == -1  # no prev table
    assert b"dc_rnn_seq_bwd_reset" in lib.dc_last_error()
    assert bwd(1, one, one, one, one, one, None, None, one, one, None, None, 0, 4, 4, 128, one, None) == -1  # no slots
    assert bwd(0, one, one, one, one, None, None, None, one, None, one, one, 1, 4, 4, 96, one, None) == -1   # no dy
