"""Host-side checks of ``value_norm`` (PopArt): the statistics update and the POP rescale against hand-written float64, the
settings and CLI flags, the header against the ctypes table, and the argument checks of the new entry points."""
import math
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import value_norm_oracle as VO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")


# ------------------------------------------------------------------------------------------------ statistics
def _fns():
    from dotaclient_b200.optimizer import DotaOptimizer, value_norm_moments, value_norm_update
    return value_norm_moments, value_norm_update, DotaOptimizer.VALUE_NORM_MIN_STD


def test_min_std_is_the_class_constant():
    assert _fns()[2] == 1e-2 == VO.MIN_STD


def test_identity_before_the_first_update():
    moments, _, floor = _fns()
    assert moments((0.0, 0.0, 0.0), floor) == (0.0, 1.0)


@pytest.mark.parametrize("decay", [0.0, 0.5, 0.99])
def test_first_update_is_the_batch_statistics(decay):
    moments, upd, floor = _fns()
    x = np.random.default_rng(1).normal(7.0, 3.0, 1000)
    st = upd((0.0, 0.0, 0.0), x.size, float(x.sum()), float((x * x).sum()), decay)
    mu, sigma = moments(st, floor)
    assert mu == pytest.approx(x.mean(), rel=1e-13)
    assert sigma == pytest.approx(x.std(), rel=1e-11)
    assert st[2] == pytest.approx(1.0 - decay, rel=1e-15)


def test_decay_against_hand_written_float64():
    moments, upd, floor = _fns()
    rng = np.random.default_rng(2)
    d, st, m, q, w = 0.9, (0.0, 0.0, 0.0), 0.0, 0.0, 0.0
    for k in range(5):
        x = rng.normal(3.0 * k, 1.0 + k, 200 + k)
        st = upd(st, x.size, float(x.sum()), float((x * x).sum()), d)
        m = d * m + (1 - d) * x.mean()
        q = d * q + (1 - d) * (x * x).mean()
        w = d * w + (1 - d)
        assert st == pytest.approx((m, q, w), rel=1e-13)
        mu = m / w
        assert moments(st, floor) == pytest.approx((mu, math.sqrt(q / w - mu * mu)), rel=1e-10)
        assert moments(st, floor) == pytest.approx(VO.moments(st), rel=1e-15)


def test_std_floor():
    moments, upd, floor = _fns()
    st = upd((0.0, 0.0, 0.0), 4, 4 * 5.0, 4 * 25.0, 0.99)           # constant targets: variance 0 (or a rounding below)
    assert moments(st, floor) == pytest.approx((5.0, 1e-2), rel=1e-12)
    st = upd((0.0, 0.0, 0.0), 3, 3.0, 3.0 + 3e-6, 0.0)              # variance 1e-6 -> std 1e-3 < the floor
    assert moments(st, floor)[1] == 1e-2


def test_empty_batch_leaves_the_state_unchanged():
    _, upd, _ = _fns()
    st = (1.5, 4.0, 0.3)
    assert upd(st, 0, 0.0, 0.0, 0.9) is st
    assert upd((0.0, 0.0, 0.0), 0.0, 0.0, 0.0, 0.9) == (0.0, 0.0, 0.0)


def test_pooled_shards_equal_the_concatenated_batch():
    """Data-parallel: the ranks' (n, sum, sum of squares) summed give the statistics of the whole batch."""
    moments, upd, floor = _fns()
    rng = np.random.default_rng(3)
    a, b = rng.normal(-4.0, 2.0, 300), rng.normal(10.0, 0.5, 77)
    pooled = [sum(v) for v in zip(VO.batch_sums(a.astype(np.float32)), VO.batch_sums(b.astype(np.float32)))]
    whole = VO.batch_sums(np.concatenate([a, b]).astype(np.float32))
    st_p = upd((0.1, 0.2, 0.3), *pooled, 0.95)
    st_w = upd((0.1, 0.2, 0.3), *whole, 0.95)
    assert st_p == pytest.approx(st_w, rel=1e-14)
    assert moments(st_p, floor) == pytest.approx(moments(st_w, floor), rel=1e-12)


def test_batch_sums_respect_the_valid_mask():
    x = np.array([1.0, 2.0, 100.0, 3.0], np.float32)
    assert VO.batch_sums(x, np.array([1, 1, 0, 1], bool)) == (3.0, 6.0, 14.0)


@pytest.mark.parametrize("old,new", [((0.0, 1.0), (5.0, 3.0)), ((5.0, 3.0), (-2.0, 0.01)), ((12.0, 40.0), (12.5, 41.0))])
def test_pop_factors_preserve_the_unnormalised_output(old, new):
    rng = np.random.default_rng(4)
    w = rng.normal(0, 0.1, 256).astype(np.float32)
    b = np.float32(0.3)
    y = rng.normal(0, 1, (50, 256))
    w2, b2 = VO.rescale(w, np.array([b]), old, new)
    before = old[1] * (y @ w.astype(np.float64) + float(b)) + old[0]
    after = new[1] * (y @ w2.astype(np.float64) + float(b2[0])) + new[0]
    np.testing.assert_allclose(after, before, rtol=1e-6, atol=1e-6 * (abs(old[0]) + old[1]))
    # in float64 without the final rounding the preservation is exact up to float64 rounding
    wd = w.astype(np.float64) * old[1] / new[1]
    bd = (old[1] * float(b) + old[0] - new[0]) / new[1]
    np.testing.assert_allclose(new[1] * (y @ wd + bd) + new[0], before, rtol=1e-12, atol=1e-12)


def test_denorm_and_normalise_round_once():
    v = np.array([0.1, -2.5, 3e4], np.float32)
    np.testing.assert_array_equal(VO.denorm(v, 0.0, 1.0), v)
    np.testing.assert_array_equal(VO.normalise(v, 0.0, 1.0), v)
    assert VO.denorm(v, 1.0 / 3, 7.0)[0] == np.float32(1.0 / 3 + 7.0 * float(np.float32(0.1)))


# ------------------------------------------------------------------------------------------------ settings / CLI
def test_settings_validation():
    from dotaclient_b200.optimizer import check_ppo_settings
    check_ppo_settings(0.98, 0.97, 0.1, 0.5)
    for d in (0.0, 0.5, 0.999999):
        check_ppo_settings(0.98, 0.97, 0.1, 0.5, value_norm=True, value_norm_decay=d)
    for bad in (1.0, -0.1, 2, float("nan"), None, True, "0.9"):
        with pytest.raises(ValueError, match="value_norm_decay"):
            check_ppo_settings(0.98, 0.97, 0.1, 0.5, value_norm=True, value_norm_decay=bad)
    for bad in (1, "yes", None):
        with pytest.raises(ValueError, match="value_norm="):
            check_ppo_settings(0.98, 0.97, 0.1, 0.5, value_norm=bad)


def test_constructor_and_main_refuse_a_bad_decay_up_front():
    from dotaclient_b200.optimizer import DotaOptimizer, main
    with pytest.raises(ValueError, match="value_norm_decay"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, value_norm=True,
                      value_norm_decay=1.0)
    with pytest.raises(ValueError, match="value_norm_decay"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, value_norm=True, value_norm_decay=-1)


def test_cli_flags():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    a = p.parse_args([])
    assert a.value_norm is False and a.value_norm_decay == 0.99
    a = p.parse_args(["--value-norm", "--value-norm-decay", "0.9"])
    assert a.value_norm is True and a.value_norm_decay == 0.9
    assert "--value-norm" in p.format_help() and "--value-norm-decay" in p.format_help()


@pytest.mark.parametrize("kw", [{}, {"value_norm": True}, {"value_norm": True, "value_norm_decay": 0.5}])
def test_main_passes_the_flags_to_the_optimizer(kw, monkeypatch):
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
    O.main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, **kw)
    assert seen["value_norm"] == kw.get("value_norm", False)
    assert seen["value_norm_decay"] == kw.get("value_norm_decay", 0.99) and seen["ran"]


# ------------------------------------------------------------------------------------------------ C ABI
def test_header_defines_the_hparam_slots_and_entry_points():
    from dotaclient_b200 import _lib
    text = open(HEADER).read()
    d = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (DC_HP_\w+) (\d+)", text)}
    assert d["DC_HP_VALUE_NORM_MEAN"] == _lib.HP_VALUE_NORM_MEAN == 6
    assert d["DC_HP_VALUE_NORM_STD"] == _lib.HP_VALUE_NORM_STD == 7
    assert max(d.values()) < _lib.HPARAM_SLOTS
    body = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    for name in ("dc_value_norm_stats", "dc_value_denorm", "dc_value_head_rescale"):
        m = re.search(r"\bint\s+%s\s*\(([^;]*?)\)\s*;" % name, body, flags=re.S)
        assert m, name
        assert len(m.group(1).split(",")) == len(_lib.SIGNATURES[name][1]), name


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_points_check_their_arguments(lib):
    """Argument errors return -1 with the entry point's name before any CUDA call (this box may have no GPU)."""
    assert lib.dc_version() >= 109
    one = 4096                                   # never dereferenced: validation fails first

    def err(rc, name, what):
        msg = lib.dc_last_error()
        assert rc == -1 and name.encode() in msg and what.encode() in msg, (rc, msg)
    err(lib.dc_value_norm_stats(one, None, -1, one, None), "dc_value_norm_stats", "N=-1")
    err(lib.dc_value_norm_stats(None, None, 8, one, None), "dc_value_norm_stats", "null pointer")
    err(lib.dc_value_norm_stats(one, one, 8, None, None), "dc_value_norm_stats", "null pointer")
    err(lib.dc_value_denorm(one, 1, -5, 0.0, 1.0, one, None), "dc_value_denorm", "N=-5")
    err(lib.dc_value_denorm(one, 0, 8, 0.0, 1.0, one, None), "dc_value_denorm", "ld_v=0")
    err(lib.dc_value_denorm(one, -128, 8, 0.0, 1.0, one, None), "dc_value_denorm", "ld_v=-128")
    err(lib.dc_value_denorm(None, 1, 8, 0.0, 1.0, one, None), "dc_value_denorm", "null pointer")
    err(lib.dc_value_denorm(one, 1, 8, 0.0, 1.0, None, None), "dc_value_denorm", "null pointer")
    err(lib.dc_value_denorm(one, 1, 8, 0.0, -1.0, one, None), "dc_value_denorm", "sigma")
    err(lib.dc_value_denorm(one, 1, 8, float("nan"), 1.0, one, None), "dc_value_denorm", "mu")
    err(lib.dc_value_head_rescale(one, 0, one, 0.0, 1.0, 0.0, 1.0, None), "dc_value_head_rescale", "n=0")
    err(lib.dc_value_head_rescale(one, -3, one, 0.0, 1.0, 0.0, 1.0, None), "dc_value_head_rescale", "n=-3")
    err(lib.dc_value_head_rescale(None, 8, one, 0.0, 1.0, 0.0, 1.0, None), "dc_value_head_rescale", "null pointer")
    err(lib.dc_value_head_rescale(one, 8, None, 0.0, 1.0, 0.0, 1.0, None), "dc_value_head_rescale", "null pointer")
    err(lib.dc_value_head_rescale(one, 8, one, 0.0, 0.0, 0.0, 1.0, None), "dc_value_head_rescale", "statistics")
    err(lib.dc_value_head_rescale(one, 8, one, 0.0, 1.0, 0.0, -2.0, None), "dc_value_head_rescale", "statistics")


def test_stats_dict_and_hparams_are_off_by_default():
    """``value_norm_stats`` is None without the feature; with it, the identity before any update."""
    from dotaclient_b200.optimizer import DotaOptimizer
    off = DotaOptimizer.__new__(DotaOptimizer)
    off.value_norm = False
    assert off.value_norm_stats is None
    on = DotaOptimizer.__new__(DotaOptimizer)
    on.value_norm, on._value_norm = True, (0.0, 0.0, 0.0)
    assert on.value_norm_stats == {"mean": 0.0, "std": 1.0, "weight": 0.0}
