"""Host-side checks of minibatch PPO: the CLI flag, the validation of ``num_minibatches``, ``minibatch_indices``, the C-ABI
declaration and argument checks of ``dc_gather_columns``, and the host index check of ``ops.gather_columns``."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")


# ------------------------------------------------------------------------------------------------ CLI / validation
def test_cli_flag_and_default():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).num_minibatches == 1
    assert p.parse_args(["--num-minibatches", "4"]).num_minibatches == 4
    assert "--num-minibatches" in p.format_help()


@pytest.mark.parametrize("bad", [0, -1, 1.5, "2", True, float("nan")])
def test_bad_num_minibatches_refused_up_front(bad):
    """Refused with ValueError before any device work (so this runs without a GPU), by the constructor, main() and
    check_ppo_settings."""
    from dotaclient_b200.optimizer import DotaOptimizer, check_ppo_settings, main
    with pytest.raises(ValueError, match="num_minibatches"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, num_minibatches=bad)
    with pytest.raises(ValueError, match="num_minibatches"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, num_minibatches=bad)
    with pytest.raises(ValueError, match="num_minibatches"):
        check_ppo_settings(0.98, 0.97, 0.1, 0.5, None, num_minibatches=bad)


def test_more_minibatches_than_min_seq_per_epoch_refused_up_front():
    from dotaclient_b200.optimizer import DotaOptimizer, check_minibatch_count, main
    with pytest.raises(ValueError, match="min_seq_per_epoch"):
        DotaOptimizer("x", 0, 1, 3, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, num_minibatches=4)
    with pytest.raises(ValueError, match="min_seq_per_epoch"):
        main("x", 0, 1, 3, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, num_minibatches=4)
    check_minibatch_count(3, 3)
    with pytest.raises(ValueError, match="min_seq_per_epoch"):
        check_minibatch_count(4, 3)


def test_accepted_settings():
    from dotaclient_b200.optimizer import check_ppo_settings
    check_ppo_settings(0.98, 0.97, 0.1, 0.5)
    check_ppo_settings(0.98, 0.97, 0.1, 0.5, num_minibatches=1)
    check_ppo_settings(0.98, 0.97, 0.1, 0.5, num_minibatches=np.int64(4))


# ------------------------------------------------------------------------------------------------ minibatch_indices
@pytest.mark.parametrize("B,M", [(7, 3), (8, 3), (16, 4), (5, 5), (1024, 4), (3, 2)])
def test_minibatch_indices_partition_the_batch(B, M):
    from dotaclient_b200.optimizer import minibatch_indices
    rng = np.random.default_rng(11)
    want = np.array_split(np.random.default_rng(11).permutation(B), M)
    got = minibatch_indices(B, M, rng)
    assert len(got) == M
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)
    sizes = [len(g) for g in got]
    assert max(sizes) - min(sizes) <= 1 and sum(sizes) == B
    np.testing.assert_array_equal(np.sort(np.concatenate(got)), np.arange(B))
    if B == 7:
        assert sizes == [3, 2, 2]
    if M == B:
        assert all(len(g) == 1 for g in got)


def test_one_minibatch_draws_nothing():
    from dotaclient_b200.optimizer import minibatch_indices
    rng = np.random.default_rng(7)
    state = rng.bit_generator.state
    got = minibatch_indices(9, 1, rng)
    assert len(got) == 1
    np.testing.assert_array_equal(got[0], np.arange(9))
    assert rng.bit_generator.state == state


# ------------------------------------------------------------------------------------------------ C ABI
def test_header_and_lib_table_agree_on_dc_gather_columns():
    from dotaclient_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\bint\s+dc_gather_columns\s*\(([^;]*?)\)\s*;", text, flags=re.S)
    assert m
    params = [p.strip() for p in m.group(1).split(",")]
    _c = _lib._c
    args = _lib.SIGNATURES["dc_gather_columns"][1]
    assert len(params) == len(args) == 5
    assert params[0].startswith("const dc_gather_desc *") and args[0] is _c.POINTER(_lib.GatherDesc)
    assert params[1].startswith("int ") and args[1] is _c.c_int
    assert params[2].startswith("const int64_t *") and args[2] is _c.c_void_p
    assert params[3].startswith("int64_t ") and args[3] is _c.c_int64
    assert params[4].startswith("dc_stream_t") and args[4] is _c.c_void_p
    defines = {d.group(1): int(d.group(2)) for d in re.finditer(r"#define\s+(DC_[A-Z0-9_]+)\s+(-?\d+)", text)}
    assert defines["DC_GATHER_MAX_TENSORS"] == _lib.GATHER_MAX_TENSORS == 32
    fields = re.search(r"typedef struct \{([^}]*)\} dc_gather_desc;", text).group(1)
    assert [f.split()[-1].strip("*;") for f in fields.strip().split(";") if f.strip()] == \
        [n for n, _ in _lib.GatherDesc._fields_]
    assert _c.sizeof(_lib.GatherDesc) == 40


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_dc_gather_columns_is_exported_and_checks_its_arguments(lib):
    """Every argument error returns -1 with a message before any CUDA call (this box may have no GPU); the empty cases
    return 0 without touching a pointer."""
    from dotaclient_b200 import _lib
    assert lib.dc_version() >= 104
    D = _lib.GatherDesc
    one, far = 1 << 20, 1 << 30          # never dereferenced: validation fails (or there is no work) first

    def call(descs, n_desc=None, index=one, n_index=4):
        arr = (D * max(len(descs), 1))(*descs) if descs is not None else None
        return lib.dc_gather_columns(arr, len(descs) if n_desc is None else n_desc, index, n_index, None)

    good = D(one, far, 2, 8, 16)
    for n_desc in (-1, 33):
        assert call([good], n_desc=n_desc) == -1 and b"n_desc" in lib.dc_last_error()
    assert call([good], n_index=-1) == -1 and b"n_index" in lib.dc_last_error()
    assert lib.dc_gather_columns(None, 1, one, 4, None) == -1 and b"null" in lib.dc_last_error()
    for bad in (D(one, far, 2, 8, 0), D(one, far, 2, 8, -4), D(one, far, -1, 8, 16), D(one, far, 2, -8, 16)):
        assert call([good, bad]) == -1 and b"descriptor 1" in lib.dc_last_error()
    assert call([good], index=None) == -1 and b"null index" in lib.dc_last_error()
    for bad in (D(None, far, 2, 8, 16), D(one, None, 2, 8, 16)):
        assert call([good, bad]) == -1 and b"null pointer" in lib.dc_last_error()
    assert call([D(one, far, 2, 0, 16)]) == -1 and b"src_cols=0" in lib.dc_last_error()
    assert call([D(one, one + 64, 2, 8, 16)]) == -1 and b"overlaps" in lib.dc_last_error()
    # nothing to do: no descriptors, no indices, or only empty tensors
    assert lib.dc_gather_columns(None, 0, None, 4, None) == 0
    assert call([good], index=None, n_index=0) == 0
    assert call([D(None, None, 0, 8, 16)], index=one) == 0


def test_gather_columns_checks_the_index_on_the_host():
    """An out-of-range, negative or non-integer index is refused with ValueError before anything reaches the device."""
    from dotaclient_b200 import ops
    src = torch.zeros(4, 6, 3)
    dst = torch.zeros(4, 2, 3)
    for bad in ([0, 6], [-1, 2], np.array([1, 7], np.int32), torch.tensor([0, 9])):
        with pytest.raises(ValueError, match="outside"):
            ops.gather_columns([(src, dst)], bad)
    for bad in (np.array([0.0, 1.0]), np.array([[0, 1]]), np.array([True, False])):
        with pytest.raises(ValueError, match="index"):
            ops.gather_columns([(src, dst)], bad)
    with pytest.raises(ValueError, match="contiguous"):
        ops.gather_columns([(src.transpose(0, 1), dst)], [0, 1])
