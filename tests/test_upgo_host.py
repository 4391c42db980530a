"""Host-side checks of UPGO (``DotaOptimizer(upgo_coef=c)``): the settings and the CLI flag, the C-ABI declarations and
their argument checks (every bad call is refused before any CUDA call, so they run without a GPU), and the float64
oracle (``upgo_oracle.py``) against hand-computed values and through its three identities."""
import math
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refresh_oracle as RF  # noqa: E402
import upgo_oracle as UP  # noqa: E402
import vtrace_oracle as VT  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
PPO = (0.98, 0.97, 0.1, 0.5)


# ------------------------------------------------------------------------------------------------ settings / CLI
def test_default_is_off():
    import inspect
    from dotaclient_b200.optimizer import DotaOptimizer, build_arg_parser, check_ppo_settings, main
    for fn in (DotaOptimizer.__init__, check_ppo_settings, main):
        assert inspect.signature(fn).parameters["upgo_coef"].default == 0.0
    assert build_arg_parser().parse_args([]).upgo_coef == 0.0


@pytest.mark.parametrize("bad", [-0.5, -1e-300, float("nan"), float("inf"), -float("inf"), True, False, "0.5", None])
def test_upgo_coef_domain(bad):
    from dotaclient_b200.optimizer import check_ppo_settings, check_upgo_coef
    with pytest.raises(ValueError, match="upgo_coef"):
        check_ppo_settings(*PPO, upgo_coef=bad)
    with pytest.raises(ValueError, match="upgo_coef"):
        check_upgo_coef(bad)


@pytest.mark.parametrize("good", [0.0, 0, 1e-12, 0.5, 1, 7.25, np.float32(0.5), np.float64(2.0)])
def test_upgo_coef_accepted(good):
    from dotaclient_b200.optimizer import check_ppo_settings, check_upgo_coef
    check_ppo_settings(*PPO, upgo_coef=good)
    check_ppo_settings(*PPO, upgo_coef=good, advantage_estimator='vtrace', mask_padding=True, pack_sequences=True,
                       value_norm=True, recompute_advantages=True, recompute_states=True, policy_ratio='joint')
    check_upgo_coef(good)


def test_refused_with_value_heads():
    from dotaclient_b200.optimizer import REWARD_KEYS, DotaOptimizer, check_ppo_settings, check_upgo_coef
    heads = {"win": [REWARD_KEYS[0]], "rest": list(REWARD_KEYS[1:])}
    with pytest.raises(ValueError, match="value_heads"):
        check_ppo_settings(*PPO, upgo_coef=0.5, value_heads=heads)
    with pytest.raises(ValueError, match="value_heads"):
        check_upgo_coef(0.5, heads)
    check_ppo_settings(*PPO, upgo_coef=0.0, value_heads=heads)          # off: no conflict
    with pytest.raises(ValueError, match="upgo_coef"):                  # refused by the constructor before any device use
        DotaOptimizer("h", 1, 1, 1, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, value_heads=heads,
                      upgo_coef=0.5)
    with pytest.raises(ValueError, match="upgo_coef"):
        DotaOptimizer("h", 1, 1, 1, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, upgo_coef=-1.0)


def test_cli_flag():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args(["--upgo-coef", "0.5"]).upgo_coef == 0.5
    assert "--upgo-coef" in p.format_help()
    with pytest.raises(SystemExit):
        p.parse_args(["--upgo-coef", "half"])


# ------------------------------------------------------------------------------------------------ C-ABI
def _declared(name):
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^)]*)\)" % name, text)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


def _ctype(decl):
    from dotaclient_b200 import _lib
    if "*" in decl or decl.startswith("dc_stream_t"):
        return _lib._vp
    return {"int": _lib._i32, "int64_t": _lib._i64, "double": _lib._f64}[decl.rsplit(" ", 1)[0]]


@pytest.mark.parametrize("name", ["dc_upgo_scan", "dc_upgo_scan_indexed"])
def test_header_matches_ctypes_signature(name):
    from dotaclient_b200 import _lib
    res, args = _lib.SIGNATURES[name]
    assert res is _lib._i32
    assert [_ctype(d) for d in _declared(name)] == args
    assert _lib.UPGO_STATS_SLOTS == int(re.search(r"#define DC_UPGO_STATS_SLOTS (\d+)", open(HEADER).read()).group(1))


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


ONE = 4096          # any non-null "pointer": validation fails before it is used


def _plain(lib, rewards=ONE, n_sub=10, values=ONE, lt=None, lb=None, seg=ONE, n_seg=3, rho_clip=1.0, adv=ONE):
    return lib.dc_upgo_scan(rewards, n_sub, values, lt, lb, seg, n_seg, None, None, 0.98, rho_clip, 0.5, adv, None, None)


def _indexed(lib, rewards=ONE, n_sub=10, values=ONE, ld=1, lt=None, lb=None, tok=ONE, seg=ONE, n_seg=3, rho_clip=1.0,
             adv=ONE):
    return lib.dc_upgo_scan_indexed(rewards, n_sub, values, ld, lt, lb, tok, seg, n_seg, None, None, 0.98, rho_clip, 0.5,
                                    adv, None, None)


BAD_COMMON = [dict(n_seg=-1), dict(n_sub=0), dict(n_sub=128), dict(lt=ONE), dict(lb=ONE),
              dict(lt=ONE, lb=ONE, rho_clip=0.0), dict(lt=ONE, lb=ONE, rho_clip=-1.0),
              dict(lt=ONE, lb=ONE, rho_clip=float("nan")), dict(rewards=None), dict(values=None), dict(seg=None),
              dict(adv=None)]


@pytest.mark.parametrize("bad", BAD_COMMON, ids=[str(b) for b in BAD_COMMON])
def test_argument_errors(lib, bad):
    assert lib.dc_version() >= 114
    assert _plain(lib, **bad) == -1 and b"dc_upgo_scan" in lib.dc_last_error()
    assert _indexed(lib, **bad) == -1 and b"dc_upgo_scan_indexed" in lib.dc_last_error()


def test_indexed_argument_errors(lib):
    assert _indexed(lib, ld=0) == -1 and b"ld_values" in lib.dc_last_error()
    assert _indexed(lib, ld=-3) == -1
    assert _indexed(lib, tok=None) == -1 and b"dc_upgo_scan_indexed" in lib.dc_last_error()


def test_no_segments_is_a_no_op(lib):
    """n_seg = 0 launches nothing, so it succeeds without a device, as the other scans do."""
    assert _plain(lib, n_seg=0) == 0
    assert _indexed(lib, n_seg=0) == 0
    assert _plain(lib, n_seg=0, lt=ONE, lb=ONE, rho_clip=2.0) == 0


# ------------------------------------------------------------------------------------------------ the oracle
def test_oracle_by_hand():
    """Three rows, gamma 0.5, boot 2: delta = (1 + 0.5*4 - 2, 0 + 0.5*1 - 4, 3 + 0.5*2 - 1) = (1, -3.5, 3).  Row 0 does
    not go through (delta_1 < 0), row 1 does (delta_2 >= 0), row 2 is the last."""
    r = np.array([1.0, 0.0, 3.0], np.float32)
    v = np.array([2.0, 4.0, 1.0], np.float32)
    au, through = UP.upgo(r, v, 0.5, boot=2.0)
    assert through.tolist() == [False, True, False]
    g2 = 3.0 + 0.5 * 2.0
    g1 = 0.0 + 0.5 * g2
    g0 = 1.0 + 0.5 * 4.0
    np.testing.assert_array_equal(au, [g0 - 2.0, g1 - 4.0, g2 - 1.0])
    np.testing.assert_array_equal(UP.stats(au, through), [3, 1, (g0 - 2) + (g1 - 4) + (g2 - 1)])
    # a tie goes through
    au, through = UP.upgo(np.array([0.0, 1.0], np.float32), np.array([0.0, 1.0], np.float32), 1.0)
    assert through.tolist() == [True, False]
    assert UP.advantages(np.float32(0.25), 2.0, 0.5).item() == np.float32(1.25)


def _segment(seed, n, sign=None):
    g = np.random.default_rng(seed)
    rewards = (g.standard_normal((n, 10)) * 0.1).astype(np.float32)
    values = g.standard_normal(n).astype(np.float32)
    if sign is not None:              # choose the values so that every TD error has the sign asked for
        r = VT.reward_sum(rewards).astype(np.float64)
        v = np.zeros(n + 1)
        v[n] = g.standard_normal()
        for t in range(n - 1, -1, -1):
            v[t] = r[t] + 0.98 * v[t + 1] - sign * (0.05 + g.random())
        values = v[:n].astype(np.float32)
        boot = np.float32(v[n])
        return rewards, values, float(boot)
    return rewards, values, float(g.standard_normal())


@pytest.mark.parametrize("n", [1, 2, 33, 300])
def test_all_through_is_the_discounted_return(n):
    """Every delta >= 0: G is the discounted reward-to-go plus gamma^(n - t) boot, so A^U = ret - V with gae_scan's ret."""
    rewards, values, boot = _segment(n, n, sign=+1)
    au, through = UP.upgo(rewards, values, 0.98, boot=boot)
    r = VT.reward_sum(rewards).astype(np.float64)
    v = values.astype(np.float64)
    delta = r + 0.98 * np.append(v[1:], boot) - v
    assert (delta >= 0).all() and through[:-1].all() and not through[-1]
    _, ret = RF.gae(rewards, values, 0.98, 0.97, boot)
    np.testing.assert_allclose(au, ret - v, rtol=0, atol=1e-12)
    np.testing.assert_allclose(UP.discounted_return(rewards, 0.98, boot), ret, rtol=0, atol=1e-12)


@pytest.mark.parametrize("n", [1, 2, 33, 300])
def test_none_through_is_the_td_error(n):
    """Every delta < 0: A^U_t = delta_t, GAE with lambda = 0."""
    rewards, values, boot = _segment(100 + n, n, sign=-1)
    au, through = UP.upgo(rewards, values, 0.98, boot=boot)
    assert not through.any()
    adv0, _ = RF.gae(rewards, values, 0.98, 0.0, boot)
    np.testing.assert_array_equal(au, adv0)


@pytest.mark.parametrize("n", [1, 32, 257])
def test_vtrace_on_policy_is_the_gae_form(n):
    """Behaviour log-probs equal to the target's: log rho = 0, rhob = 1, and the V-trace form is the GAE form."""
    rewards, values, boot = _segment(200 + n, n)
    lt = -np.abs(np.random.default_rng(n).standard_normal((n, 5))).astype(np.float32)
    au_v, th_v = UP.upgo(rewards, values, 0.98, boot=boot, logrho=VT.log_rho(lt, lt), rho_clip=1.0)
    au_g, th_g = UP.upgo(rewards, values, 0.98, boot=boot)
    np.testing.assert_array_equal(th_v, th_g)
    np.testing.assert_array_equal(au_v, au_g)


def test_vtrace_weights_truncate_and_keep_nan():
    rewards, values, boot = _segment(7, 4)
    lr = np.array([0.0, 5.0, -1.0, math.nan])
    au, _ = UP.upgo(rewards, values, 0.98, boot=boot, logrho=lr, rho_clip=2.0)
    base, _ = UP.upgo(rewards, values, 0.98, boot=boot)
    np.testing.assert_array_equal(au[:3], base[:3] * np.array([1.0, 2.0, math.exp(-1.0)]))
    assert math.isnan(au[3])
