"""CPU tests of dual-clip PPO (``DotaOptimizer(dual_clip=c)``): the settings and CLI refusals and the flag's way through
``main``, the header against ``_lib``, the C entry point's argument checks, the float64 oracle by hand on a few rows (one
that binds, one that does not, A = 0, an exact tie), and the unchanged default key sets of ``_ppo_stats_dict``."""
import math
import os
import re
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dual_clip_oracle as DO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
BASE = (0.98, 0.97, 0.1, 0.5)
HEADS = DO.HEADS
SIZES = (4, 9, 9, 40, 3)


# ------------------------------------------------------------------------------------------------ settings and CLI
def test_settings_accept_none_and_numbers_above_one():
    from dotaclient_b200.optimizer import check_dual_clip, check_ppo_settings
    check_ppo_settings(*BASE)
    for ok in (None, 3, 3.0, 1.0000001, 1e6):
        check_dual_clip(ok)
        check_ppo_settings(*BASE, dual_clip=ok)
    # it composes with every option of the PPO objective
    check_ppo_settings(*BASE, 0.2, dual_clip=3.0, advantage_estimator="vtrace", mask_padding=True, pack_sequences=True,
                       num_minibatches=4, policy_ratio="joint", value_norm=True, kl_coef=0.1, kl_target=0.01,
                       kl_stop=0.05, recompute_advantages=True, recompute_states=True, teacher_model="t.pt",
                       teacher_coef=0.5, upgo_coef=0.5)


@pytest.mark.parametrize("bad", [1.0, 1, 0.5, 0.0, -3.0, math.nan, math.inf, -math.inf, True, "3", [3.0]])
def test_settings_refuse_bad_values(bad):
    from dotaclient_b200.optimizer import check_dual_clip, check_ppo_settings
    with pytest.raises(ValueError, match="dual_clip="):
        check_dual_clip(bad)
    with pytest.raises(ValueError, match="dual_clip="):
        check_ppo_settings(*BASE, dual_clip=bad)


def test_bc_refuses_dual_clip():
    from dotaclient_b200.optimizer import check_ppo_settings
    check_ppo_settings(*BASE, objective="bc")
    with pytest.raises(ValueError, match=re.escape("dual_clip=3.0") + ".*objective='bc'"):
        check_ppo_settings(*BASE, objective="bc", dual_clip=3.0)


def test_constructor_and_main_refuse_bad_settings_up_front():
    from dotaclient_b200.optimizer import DotaOptimizer, main
    with pytest.raises(ValueError, match="dual_clip="):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, dual_clip=0.9)
    with pytest.raises(ValueError, match="objective='bc'"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, objective="bc",
                      dual_clip=3.0)
    with pytest.raises(ValueError, match="dual_clip="):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, dual_clip=math.nan)


def test_cli_flag():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).dual_clip is None
    assert p.parse_args(["--dual-clip", "3"]).dual_clip == 3.0
    assert "--dual-clip" in p.format_help()
    with pytest.raises(SystemExit):
        p.parse_args(["--dual-clip", "three"])


@pytest.mark.parametrize("dual_clip", [None, 3.0])
def test_main_passes_the_flag(dual_clip, monkeypatch):
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
    O.main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, dual_clip=dual_clip)
    assert seen["dual_clip"] == dual_clip and seen["ran"]


def test_main_refuses_a_cli_value_of_one_before_anything_runs(monkeypatch):
    from dotaclient_b200 import optimizer as O
    args = O.build_arg_parser().parse_args(["--dual-clip", "1"])
    monkeypatch.setattr(O, "DotaOptimizer", lambda **k: pytest.fail("constructed"))
    with pytest.raises(ValueError, match="dual_clip=1.0"):
        O.main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, dual_clip=args.dual_clip)


def test_default_stats_keys_are_unchanged():
    """The per-head and joint key sets of ``_ppo_stats_dict`` are those without dual clip: its fractions are added by the
    step only when the feature is on."""
    from dotaclient_b200 import _lib
    from dotaclient_b200.optimizer import DotaOptimizer
    st = [0.0] * _lib.PPO_STATS_SLOTS
    base = {"approx_kl", "clip_fraction", "explained_variance"} | {p + "/" + k for p in ("approx_kl", "clip_fraction")
                                                                   for k in HEADS}
    assert set(DotaOptimizer._ppo_stats_dict(st)) == base
    assert set(DotaOptimizer._ppo_stats_dict(st, joint=True)) == base | {"approx_kl/joint", "clip_fraction/joint"}
    assert not any("dual" in k for k in DotaOptimizer._ppo_stats_dict(st, joint=True, kl=True))


# ------------------------------------------------------------------------------------------------ header and ABI
def _declared():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(dc_\w+)\s*\(([^;{]*?)\)\s*;", text):
        args = m.group(2).strip()
        protos[m.group(1)] = 0 if args in ("", "void") else args.count(",") + 1
    return protos


def test_header_and_lib_table_agree():
    from dotaclient_b200 import _lib
    protos = _declared()
    name = "dc_ppo_loss_fwd_bwd_dual_clip"
    assert name in protos and name in _lib.SIGNATURES
    # the teacher entry point's arguments plus dual_clip and dual_clip_stats
    assert len(_lib.SIGNATURES[name][1]) == protos[name] == protos["dc_ppo_loss_fwd_bwd_teacher"] + 2
    d = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DC_[A-Z0-9_]+)\s+(-?\d+)", open(HEADER).read())}
    assert d["DC_DUAL_CLIP_STATS_SLOTS"] == _lib.DUAL_CLIP_STATS_SLOTS == 2 + len(HEADS)
    assert d["DC_HPARAM_SLOTS"] == _lib.HPARAM_SLOTS == 10          # c is not a slot of the block
    assert d["DC_PPO_STATS_SLOTS"] == _lib.PPO_STATS_SLOTS


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_point_checks_its_arguments(lib):
    from dotaclient_b200 import _lib
    assert hasattr(lib, "dc_ppo_loss_fwd_bwd_dual_clip") and lib.dc_version() >= 116
    one = 4096
    p5 = _lib._ptr5(*[one] * 5)
    ld = (_lib._c.c_int64 * 5)(4, 9, 9, 40, 3)
    short = (_lib._c.c_int64 * 5)(4, 9, 9, 39, 3)
    f = lib.dc_ppo_loss_fwd_bwd_dual_clip

    def call(c=one, dstats=one, rows=None, coef=None, tstats=None, hparams=one, n=8, old_logp=one, adv=one, ws=one,
             ld_l=ld, ld_v=1):
        return f(p5, ld_l, p5, p5, old_logp, None, rows, adv, one, one, ld_v, None, None, n, hparams, coef, c, 0, p5, ld,
                 one, 1, one, one, None, tstats, dstats, one, ws, None)
    # null dual-clip operands, a partial teacher, a null hyper-parameter block or operand, a bad token count or row pitch:
    # all refused before any CUDA call
    for kw, what in (({"c": None}, b"dual_clip"), ({"dstats": None}, b"dual_clip"),
                     ({"rows": one}, b"teacher"), ({"coef": one}, b"teacher"), ({"tstats": one}, b"teacher"),
                     ({"rows": one, "coef": one}, b"teacher"), ({"rows": one, "tstats": one}, b"teacher"),
                     ({"hparams": None}, b"hyper-parameter"), ({"n": 0}, b"N=0"), ({"n": -5}, b"N=-5"),
                     ({"old_logp": None}, b"null pointer"), ({"adv": None}, b"null pointer"),
                     ({"ws": None}, b"null pointer"), ({"ld_l": short}, b"row pitch of head 3"),
                     ({"ld_v": 0}, b"value pitch")):
        assert call(**kw) == -1, kw
        assert what in lib.dc_last_error(), (kw, lib.dc_last_error())


def test_ops_refuses_dual_clip_with_bc():
    from dotaclient_b200 import ops
    with pytest.raises(ValueError, match="dual clip"):
        ops.ppo_loss_fwd_bwd([torch.zeros(2, n) for n in SIZES], [torch.ones(2, n, dtype=torch.bool) for n in SIZES],
                             [torch.zeros(2, n, dtype=torch.bool) for n in SIZES], None, torch.zeros(2), torch.zeros(2),
                             torch.zeros(2), None, None, None, hparams=torch.zeros(10, dtype=torch.float64), bc=True,
                             dual_clip=torch.tensor([3.0], dtype=torch.float64))


# ------------------------------------------------------------------------------------------------ the oracle by hand
def test_term_by_hand():
    """e_clip = 0.2, c = 3: a row with A < 0 and r = 5 binds (term c A, no gradient); r = 2 does not (r A); A = 0 and A > 0
    keep the clipped surrogate whatever r is; r = c exactly ties (term c A, half the gradient)."""
    r = torch.tensor([5.0, 2.0, 5.0, 5.0, 3.0, 0.5], dtype=torch.float64, requires_grad=True)
    adv = torch.tensor([-1.0, -1.0, 0.0, 2.0, -0.5, -1.0], dtype=torch.float64)
    term, bound = DO.dual_clip_term(r, adv, 0.2, 3.0)
    torch.testing.assert_close(term.detach(), torch.tensor([-3.0, -2.0, 0.0, 2.4, -1.5, -0.8], dtype=torch.float64))
    assert bound.tolist() == [True, False, False, False, False, False]
    term.sum().backward()
    # d term / d r: bound 0; r A -> A; A = 0 -> 0; clipped above (A > 0, r > 1 + e) -> 0; tie -> A / 2; r < 1 - e with
    # A < 0 is clipped at (1 - e) A -> 0
    torch.testing.assert_close(r.grad, torch.tensor([0.0, -1.0, 0.0, 0.0, -0.25, 0.0], dtype=torch.float64))


def _tokens():
    """Four tokens with one action row each, in the enum head only (every other head is unused): uniform logits over four
    legal entries, so p(a) = 1/4 and r = exp(-old) / 4 for an old log-prob ``old``."""
    n = 4
    logits = {k: torch.zeros(n, s, dtype=torch.float64) for k, s in zip(HEADS, SIZES)}
    masks = {k: torch.ones(n, s, dtype=torch.bool) for k, s in zip(HEADS, SIZES)}
    actions = {k: torch.zeros(n, s, dtype=torch.bool) for k, s in zip(HEADS, SIZES)}
    actions["enum"][:, 0] = True
    return logits, masks, actions


@pytest.mark.parametrize("joint", [False, True])
def test_policy_loss_by_hand(joint):
    """Raw advantages (-3, -1, 1, 3) normalise to A = a / std (std = sqrt(20 / 3)); the ratios are (5, 2, 5, 1).  With
    e_clip = 0.2 and c = 3: token 0 binds (-c A_0), token 1 is r A_1, token 2 is clipped (1.2 A_2), token 3 is r A_3.  One
    head with rows, so the per-head mean is a fifth of that head's mean; the joint ratio is the same ratio here."""
    logits, masks, actions = _tokens()
    ratios = torch.tensor([5.0, 2.0, 5.0, 1.0], dtype=torch.float64)
    dense_old = torch.zeros(4, 5, dtype=torch.float64)
    dense_old[:, 0] = torch.log(torch.tensor(0.25, dtype=torch.float64)) - torch.log(ratios)
    adv_raw = torch.tensor([-3.0, -1.0, 1.0, 3.0])
    a = DO.normalised_advantage(adv_raw)
    std = math.sqrt(20.0 / 3.0)
    torch.testing.assert_close(a, adv_raw.double() / (std + 1.1920928955078125e-07))
    lg = {k: v.clone().requires_grad_(True) for k, v in logits.items()}
    p_loss, fr = DO.policy_loss(lg, actions, masks, dense_old, a, 0.2, 3.0, joint=joint)
    terms = torch.stack([3.0 * a[0], 2.0 * a[1], 1.2 * a[2], 1.0 * a[3]])
    want = -terms.mean() if joint else -terms.mean() / 5
    torch.testing.assert_close(p_loss.detach(), want)
    if joint:
        assert fr == dict({"fraction": 0.0, "fraction/joint": 0.25}, **{"fraction/" + k: 0.0 for k in HEADS})
    else:
        assert fr["fraction/enum"] == 0.25 and fr["fraction"] == 0.25 and fr["fraction/joint"] == 0.0
        assert all(fr["fraction/" + k] == 0.0 for k in HEADS[1:])
    p_loss.backward()
    g = lg["enum"].grad
    # the bound token and the clipped one get no gradient at all
    assert bool((g[0] == 0).all()) and bool((g[2] == 0).all())
    assert float(g[1].abs().sum()) > 0 and float(g[3].abs().sum()) > 0
    assert all(lg[k].grad is None or bool((lg[k].grad == 0).all()) for k in HEADS[1:])


def test_a_large_c_is_the_clipped_surrogate():
    """c beyond every ratio: the dual-clipped loss is the base loss of both ratio modes, with the same gradient."""
    import joint_ratio_oracle as JO
    import padding_oracle as PO
    g = torch.Generator().manual_seed(3)
    n = 64
    logits = {k: torch.randn(n, s, generator=g, dtype=torch.float64) for k, s in zip(HEADS, SIZES)}
    masks = {k: torch.rand(n, s, generator=g) < 0.7 for k, s in zip(HEADS, SIZES)}
    for k in HEADS:
        masks[k][:, 0] = True
    actions = {k: torch.zeros(n, s, dtype=torch.bool) for k, s in zip(HEADS, SIZES)}
    for k in HEADS:
        pick = torch.rand(n, generator=g) < 0.6
        actions[k][pick, 0] = True
    dense_old = torch.randn(n, 5, generator=g, dtype=torch.float64) - 2.0
    values, adv, ret = (torch.randn(n, generator=g, dtype=torch.float64) for _ in range(3))
    for joint in (False, True):
        lg = {k: v.clone().requires_grad_(True) for k, v in logits.items()}
        got = DO.dual_clip_ppo_loss(lg, values, actions, masks, dense_old, adv, ret, 5e-4, 0.5, 0.2, 1e6, joint=joint)
        got[0].backward()
        lb = {k: v.clone().requires_grad_(True) for k, v in logits.items()}
        if joint:
            base = JO.joint_ppo_loss(lb, values, actions, masks, dense_old, adv, ret, 5e-4, 0.5, 0.2)
        else:
            base = PO.masked_ppo_loss(lb, values, actions, masks, dense_old, adv, ret, torch.ones(n, dtype=torch.bool),
                                      5e-4, 0.5, 0.2)
        base[0].backward()
        torch.testing.assert_close(got[0].detach(), base[0].detach().double(), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(got[1].detach(), base[1].detach().double(), rtol=1e-12, atol=1e-12)
        assert got[5]["fraction"] == 0.0 and got[5]["fraction/joint"] == 0.0
        for k in HEADS:
            torch.testing.assert_close(lg[k].grad, lb[k].grad, rtol=1e-12, atol=1e-14)
