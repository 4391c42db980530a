"""Host-side checks of the V-trace advantage estimator: CLI flags and validation, the C-ABI declaration, the float64 numpy
oracle (``vtrace_oracle.py``) against hand-computed values and against the reference's GAE through two identities, and the
host validation of the rollouts' ``behaviour_logp``."""
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vtrace_oracle as VT  # noqa: E402
from oracle import ref_optimizer as RO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")


# ------------------------------------------------------------------------------------------------ CLI / validation
def test_cli_flags_and_defaults():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    a = p.parse_args([])
    assert (a.advantage_estimator, a.vtrace_rho_clip, a.vtrace_c_clip) == ("gae", 1.0, 1.0)
    a = p.parse_args(["--advantage-estimator", "vtrace", "--vtrace-rho-clip", "2.0", "--vtrace-c-clip", "0.5"])
    assert (a.advantage_estimator, a.vtrace_rho_clip, a.vtrace_c_clip) == ("vtrace", 2.0, 0.5)
    with pytest.raises(SystemExit):
        p.parse_args(["--advantage-estimator", "retrace"])
    text = p.format_help()
    for flag in ("--advantage-estimator", "--vtrace-rho-clip", "--vtrace-c-clip"):
        assert flag in text


BAD_SETTINGS = [dict(advantage_estimator="retrace"), dict(advantage_estimator=None), dict(vtrace_rho_clip=0.0),
                dict(vtrace_rho_clip=-1.0), dict(vtrace_rho_clip=float("nan")), dict(vtrace_c_clip=0.0),
                dict(vtrace_c_clip=-0.5), dict(vtrace_c_clip=float("nan")), dict(vtrace_c_clip="1")]


@pytest.mark.parametrize("bad", BAD_SETTINGS)
def test_constructor_and_main_reject_bad_settings_up_front(bad):
    """Refused with ValueError before any device work (so this runs without a GPU), by the constructor and by main()."""
    from dotaclient_b200.optimizer import DotaOptimizer, check_ppo_settings, main
    name = next(iter(bad))
    with pytest.raises(ValueError, match=name):
        DotaOptimizer("x", 0, 1, 1, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, **bad)
    with pytest.raises(ValueError, match=name):
        main("x", 0, 1, 1, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, **bad)
    with pytest.raises(ValueError, match=name):
        check_ppo_settings(0.98, 0.97, 0.1, 0.5, None, **bad)


def test_accepted_settings():
    from dotaclient_b200.optimizer import check_ppo_settings
    check_ppo_settings(0.98, 0.97, 0.1, 0.5)                                  # the existing positional callers
    check_ppo_settings(0.98, 0.97, 0.1, 0.5, None, advantage_estimator="vtrace", vtrace_rho_clip=1e-6, vtrace_c_clip=100.0)
    check_ppo_settings(0.98, 0.97, 0.1, 0.5, advantage_estimator="gae", vtrace_rho_clip=np.float32(2), vtrace_c_clip=1)


# ------------------------------------------------------------------------------------------------ C ABI
def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2).count(",") + 1
            for m in re.finditer(r"\b(dc_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", text, flags=re.S)}


def test_header_and_lib_table_agree_on_dc_vtrace_scan():
    from dotaclient_b200 import _lib
    protos = _declared()
    assert "dc_vtrace_scan" in protos and "dc_vtrace_scan" in _lib.SIGNATURES
    assert len(_lib.SIGNATURES["dc_vtrace_scan"][1]) == protos["dc_vtrace_scan"] == 17
    defines = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DC_[A-Z0-9_]+)\s+(-?\d+)", open(HEADER).read())}
    assert defines["DC_VTRACE_STATS_SLOTS"] == _lib.VTRACE_STATS_SLOTS == VT.STATS_SLOTS
    # the argument types, in order: pointers, n_sub / n_seg int, the four scalars double
    _c = _lib._c
    args = _lib.SIGNATURES["dc_vtrace_scan"][1]
    assert [i for i, a in enumerate(args) if a is _c.c_int] == [1, 6]
    assert [i for i, a in enumerate(args) if a is _c.c_double] == [9, 10, 11, 12]


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_dc_vtrace_scan_is_exported_and_checks_its_arguments(lib):
    assert lib.dc_version() >= 103
    one = 4096
    ok = (one, 10, one, one, one, one, 3, None, None, 0.98, 0.97)
    for clips in ((0.0, 1.0), (1.0, 0.0), (-1.0, 1.0), (float("nan"), 1.0), (1.0, float("nan"))):
        rc = lib.dc_vtrace_scan(*ok, *clips, one, one, None, None)
        assert rc == -1 and b"clip" in lib.dc_last_error(), clips
    for n_sub in (0, 128):
        assert lib.dc_vtrace_scan(one, n_sub, *ok[2:], 1.0, 1.0, one, one, None, None) == -1
    rc = lib.dc_vtrace_scan(one, 10, one, None, one, one, 3, None, None, 0.98, 0.97, 1.0, 1.0, one, one, None, None)
    assert rc == -1 and b"null" in lib.dc_last_error()
    # no segments: nothing to do, nothing read
    assert lib.dc_vtrace_scan(None, 10, None, None, None, None, 0, None, None, 0.98, 0.97, 1.0, 1.0, None, None, None,
                              None) == 0


# ------------------------------------------------------------------------------------------------ oracle
def test_oracle_against_hand_computed_values():
    # gamma 0.5, lambda 1, r = [1, 2], V = [0.5, 1], boot 0, rho = [2, 0.5]
    r, v = np.array([1.0, 2.0], np.float32), np.array([0.5, 1.0], np.float32)
    lr = np.log([2.0, 0.5])
    pg, vs = VT.vtrace(r, v, lr, gamma=0.5, lam=1.0, rho_clip=1.0, c_clip=1.0)
    # t=1: rhob 0.5, delta 0.5*(2 - 1) = 0.5, vs 1.5, A 0.5;  t=0: rhob 1, c 1, delta 1, vs 0.5 + 1 + 0.5*(1.5-1) = 1.75,
    # A = 1 + 0.5*1.5 - 0.5 = 1.25
    np.testing.assert_allclose(vs, [1.75, 1.5], rtol=1e-15)
    np.testing.assert_allclose(pg, [1.25, 0.5], rtol=1e-15)
    np.testing.assert_allclose(VT.stats(lr, 1.0, 1.0), [2, 0.0, 1.5, 1, 1, 0, 0, 0], atol=1e-15)
    # rho_clip 2, c_clip 0.5: t=0 rhob 2, c 0.5: vs 0.5 + 2 + 0.5*0.5*0.5 = 2.625, A = 2*(1 + 0.75 - 0.5) = 2.5
    pg, vs = VT.vtrace(r, v, lr, gamma=0.5, lam=1.0, rho_clip=2.0, c_clip=0.5)
    np.testing.assert_allclose(vs, [2.625, 1.5], rtol=1e-15)
    np.testing.assert_allclose(pg, [2.5, 0.5], rtol=1e-15)
    np.testing.assert_allclose(VT.stats(lr, 2.0, 0.5), [2, 0.0, 2.5, 0, 1, 0, 0, 0], atol=1e-15)
    # bootstrap value 4: t=1 delta 0.5*(2 + 2 - 1) = 1.5 -> vs 2.5, A 1.5
    pg, vs = VT.vtrace(r, v, lr, gamma=0.5, lam=1.0, boot=4.0)
    assert vs[1] == pytest.approx(2.5, rel=1e-15) and pg[1] == pytest.approx(1.5, rel=1e-15)
    # log rho from dense per-head rows, heads summed in order
    lt = np.array([[-1.0, -2.0, 0, 0, 0]], np.float32)
    lb = np.array([[-1.5, -1.0, 0, 0, 0]], np.float32)
    assert VT.log_rho(lt, lb)[0] == -0.5
    # overflowing weights are truncated, not NaN
    pg, vs = VT.vtrace(r, v, [800.0, -800.0], gamma=0.5, lam=0.9)
    assert np.isfinite(pg).all() and np.isfinite(vs).all()
    assert VT.summary([VT.stats([800.0, -800.0])])["rho_clip_fraction"] == 0.5


@pytest.mark.parametrize("n,gamma,lam", [(1, 0.98, 0.97), (50, 0.98, 0.97), (517, 0.995, 0.9), (64, 0.9, 0.0)])
def test_oracle_identities_against_the_reference_gae(n, gamma, lam):
    """log rho = 0: vs - V is the GAE(lambda) advantage; at lambda = 1 also vs = discounted returns and A = GAE(1)."""
    rng = np.random.RandomState(n)
    rewards = (rng.randn(n, 10) * 0.1).astype(np.float32)
    values = rng.randn(n).astype(np.float32)
    r = np.append(np.sum(rewards, axis=1), np.float32(0)).astype(np.float32)
    v = np.append(values, np.float32(0))
    pg, vs = VT.vtrace(rewards, values, np.zeros(n), gamma, lam)
    adv, _ = RO.advantage_returns(r, v, gamma=gamma, lam=lam)
    np.testing.assert_allclose(vs - values, adv, rtol=0, atol=1e-6 * (1 + np.abs(adv)).max())
    pg, vs = VT.vtrace(rewards, values, np.zeros(n), gamma, 1.0)
    adv1, ret = RO.advantage_returns(r, v, gamma=gamma, lam=1.0)
    np.testing.assert_allclose(vs, ret, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(pg, adv1, rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------------ rollout validation
def _rollout(L=20, seed=3, **extra):
    from dotaclient_b200.synthetic import make_rollout
    d = make_rollout(L, seed, game_id=41, team_id=2)
    d["player_id"] = 7
    d.update(extra)
    return d


def test_behaviour_logp_validation():
    from dotaclient_b200.optimizer import check_behaviour_logp
    L = 20
    good = np.full((L, 5), -0.5, np.float32)
    check_behaviour_logp([_rollout(behaviour_logp=good), _rollout(behaviour_logp=torch.from_numpy(good))])
    with pytest.raises(ValueError, match=r"game_id=41 player_id=7.*no 'behaviour_logp'"):
        check_behaviour_logp([_rollout(behaviour_logp=good), _rollout()])
    for shape in ((L - 1, 5), (L, 4), (L,), (L, 5, 1)):
        with pytest.raises(ValueError, match="game_id=41"):
            check_behaviour_logp([_rollout(behaviour_logp=np.zeros(shape, np.float32))])
    with pytest.raises(ValueError, match="float"):
        check_behaviour_logp([_rollout(behaviour_logp=np.zeros((L, 5), np.int64))])
    d = _rollout()
    acted = np.stack([d["actions"][k].numpy().any(axis=1) for k in ("enum", "x", "y", "target_unit", "ability")], axis=1)
    assert acted.any() and (~acted).any()
    t, h = map(int, np.argwhere(acted)[-1])
    for bad in (float("nan"), float("inf"), -float("inf")):
        blp = good.copy()
        blp[t, h] = bad
        with pytest.raises(ValueError, match="game_id=41 player_id=7.*step %d" % t):
            check_behaviour_logp([_rollout(behaviour_logp=blp)])
    blp = good.copy()
    blp[~acted] = float("nan")                              # heads that did not act: ignored
    check_behaviour_logp([_rollout(behaviour_logp=blp)])
