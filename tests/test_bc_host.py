"""CPU tests of behaviour cloning (``DotaOptimizer(objective='bc')``): every refusal of the settings, the CLI flag and its way
through ``main``, ``check_demonstrations`` on each malformed case, the float64 oracle by hand (a uniform policy), the header
against ``_lib``, and the C entry point's argument checks."""
import copy
import math
import os
import re
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bc_oracle as BO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
BASE = (0.98, 0.97, 0.1, 0.5)
HEADS = BO.HEADS
SIZES = (4, 9, 9, 40, 3)


# ------------------------------------------------------------------------------------------------ settings and CLI
def test_objective_settings():
    from dotaclient_b200.optimizer import OBJECTIVES, check_ppo_settings
    assert OBJECTIVES == ("ppo", "bc")
    check_ppo_settings(*BASE, objective="bc")
    # every option that does not act on the policy-gradient term composes
    check_ppo_settings(*BASE, 0.2, objective="bc", mask_padding=True, pack_sequences=True, num_minibatches=4,
                       recompute_advantages=True, recompute_states=True, value_norm=True)
    from dotaclient_b200.optimizer import REWARD_KEYS
    check_ppo_settings(*BASE, objective="bc", value_heads={"win": ["win"], "rest": [k for k in REWARD_KEYS if k != "win"]})
    for bad in ("BC", "supervised", None, 1):
        with pytest.raises(ValueError, match="objective="):
            check_ppo_settings(*BASE, objective=bad)


@pytest.mark.parametrize("kw,what", [({"advantage_estimator": "vtrace"}, "advantage_estimator='vtrace'"),
                                     ({"policy_ratio": "joint"}, "policy_ratio='joint'"),
                                     ({"kl_coef": 0.1}, "kl_coef=0.1"),
                                     ({"kl_coef": 0.1, "kl_target": 0.01}, "kl_coef=0.1"),
                                     ({"kl_target": 0.01, "kl_coef": 0.2}, "kl_coef=0.2"),
                                     ({"kl_stop": 0.05}, "kl_stop=0.05"),
                                     ({"teacher_model": "t.pt"}, "teacher_model='t.pt'"),
                                     ({"upgo_coef": 0.5}, "upgo_coef=0.5")])
def test_bc_refuses_what_needs_a_policy_gradient(kw, what):
    from dotaclient_b200.optimizer import check_ppo_settings
    check_ppo_settings(*BASE, **kw)                 # each is fine under the default objective
    with pytest.raises(ValueError, match=re.escape(what) + ".*objective='bc'"):
        check_ppo_settings(*BASE, objective="bc", **kw)


def test_constructor_and_main_refuse_bad_settings_up_front():
    from dotaclient_b200.optimizer import DotaOptimizer, main
    with pytest.raises(ValueError, match="objective='bc'"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, objective="bc",
                      kl_coef=0.1)
    with pytest.raises(ValueError, match="objective="):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, objective="dagger")
    with pytest.raises(ValueError, match="objective='bc'"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, objective="bc", upgo_coef=1.0)


def test_cli_flag():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).objective == "ppo"
    assert p.parse_args(["--objective", "bc"]).objective == "bc"
    assert "--objective" in p.format_help()
    with pytest.raises(SystemExit):
        p.parse_args(["--objective", "dagger"])


@pytest.mark.parametrize("objective", ["ppo", "bc"])
def test_main_passes_the_objective(objective, monkeypatch):
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
    O.main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, objective=objective)
    assert seen["objective"] == objective and seen["ran"]


# ------------------------------------------------------------------------------------------------ check_demonstrations
def _demo(seed=3, L=30, game_id=11):
    from dotaclient_b200.synthetic import make_rollout
    return make_rollout(L, seed, game_id=game_id)


def _step(d, kind):
    """The first step whose enum action is ``kind``."""
    return int(torch.nonzero(d["actions"]["enum"][:, kind])[0])


def test_check_demonstrations_accepts_the_wire_format():
    from dotaclient_b200.optimizer import check_demonstrations
    datas = [_demo(s, L) for s, L in ((1, 30), (2, 1), (3, 57))]
    check_demonstrations(datas)
    u8 = copy.deepcopy(datas[0])                    # the agent's uint8 rows, and [L, 1, n] rows
    u8["actions"] = {k: v.to(torch.uint8).unsqueeze(1) for k, v in u8["actions"].items()}
    u8["masks"] = {k: v.to(torch.uint8).numpy() for k, v in u8["masks"].items()}
    check_demonstrations([u8])


def _malformed(case):
    d = _demo()
    a, m = d["actions"], d["masks"]
    if case == "two entries":
        t = _step(d, 1)
        a["x"][t] = False
        a["x"][t, 2] = a["x"][t, 5] = True
        return d, t, "x", "more than one entry"
    if case == "illegal":
        t = _step(d, 2)
        m["target_unit"][t, 0] = False              # unit 0 is never a legal target
        a["target_unit"][t] = False
        a["target_unit"][t, 0] = True
        return d, t, "target_unit", "illegal"
    if case == "illegal enum":
        t = 4
        m["enum"][t, int(a["enum"][t].int().argmax())] = False
        return d, t, "enum", "illegal"
    if case == "missing sub-head":
        t = _step(d, 1)
        a["y"][t] = False
        return d, t, "y", "has no action row"
    if case == "extra sub-head":
        t = _step(d, 0)
        a["ability"][t, 1] = True
        m["ability"][t] = True
        return d, t, "ability", "does not sample"
    if case == "wrong sub-head":
        t = _step(d, 3)
        a["target_unit"][t, 3] = True
        m["target_unit"][t, 3] = True
        return d, t, "target_unit", "does not sample"
    if case == "no enum":
        t = _step(d, 0)
        a["enum"][t] = False
        return d, t, "enum", "no enum row"
    raise KeyError(case)


@pytest.mark.parametrize("case", ["two entries", "illegal", "illegal enum", "missing sub-head", "extra sub-head",
                                  "wrong sub-head", "no enum"])
def test_check_demonstrations_refuses(case):
    from dotaclient_b200.optimizer import check_demonstrations
    bad, t, head, why = _malformed(case)
    good = _demo(9, 20, game_id=4)
    with pytest.raises(ValueError) as e:
        check_demonstrations([good, bad])
    msg = str(e.value)
    assert "game_id=11 player_id=0" in msg and "step %d," % t in msg and "head %r" % head in msg and why in msg, msg


def test_check_demonstrations_reports_the_first_step():
    from dotaclient_b200.optimizer import check_demonstrations
    d = _demo()
    late, early = _step(d, 1), _step(d, 3)
    d["actions"]["x"][late] = False                 # a later step's missing row and an earlier step's extra row
    d["actions"]["x"][early, 0] = True
    d["masks"]["x"][early, 0] = True
    with pytest.raises(ValueError, match="step %d, head 'x'" % min(late, early)):
        check_demonstrations([d])


def test_prep_refuses_a_malformed_demonstration_before_anything_runs():
    """``_prepare_rollouts`` runs the check before any device work: a stand-in with only the attributes prep reads first."""
    from dotaclient_b200.optimizer import DotaOptimizer

    class Stub:
        seq_len, device, advantage_estimator, objective = 16, None, "gae", "bc"

        class policy_base:
            num_layers, hidden_size, cell = 1, 128, "lstm"

    bad = _malformed("two entries")[0]
    with pytest.raises(ValueError, match="more than one entry"):
        DotaOptimizer._prepare_rollouts(Stub(), [bad])


# ------------------------------------------------------------------------------------------------ the oracle by hand
def _uniform_case(seed=5, L=64, valid=None):
    d = _demo(seed, L)
    logits = {k: torch.zeros(L, n, dtype=torch.float64) for k, n in zip(HEADS, SIZES)}
    acts = {k: d["actions"][k] for k in HEADS}
    masks = {k: d["masks"][k] for k in HEADS}
    return logits, acts, masks


@pytest.mark.parametrize("with_valid", [False, True])
def test_oracle_on_a_uniform_policy(with_valid):
    """Logits all 0: -log p(a) = log(legal count) on every row, so NLL = (1/T_a) sum_t sum_{h in S_t} log(legal count);
    the arg-max is the lowest legal index; the gradient is (1/T_a)(1/legal - onehot) on the legal entries."""
    L = 64
    logits, acts, masks = _uniform_case(L=L)
    valid = None
    if with_valid:
        valid = torch.arange(L) % 3 != 1
    use = torch.ones(L, dtype=torch.bool) if valid is None else valid
    want, t_a, right_tok = 0.0, 0, 0
    per_sum = {k: 0.0 for k in HEADS}
    per_cnt = {k: 0 for k in HEADS}
    per_right = {k: 0 for k in HEADS}
    for t in range(L):
        if not use[t]:
            continue
        heads = [k for k in HEADS if bool(acts[k][t].any())]
        t_a += bool(heads)
        ok = True
        for k in heads:
            legal = int(masks[k][t].sum())
            want += math.log(legal)
            per_sum[k] += math.log(legal)
            per_cnt[k] += 1
            r = int(torch.nonzero(masks[k][t])[0]) == int(torch.nonzero(acts[k][t])[0])
            per_right[k] += r
            ok &= r
        right_tok += bool(heads) and ok
    lg = {k: v.clone().requires_grad_(True) for k, v in logits.items()}
    got, got_t_a, sums, counts = BO.nll(lg, acts, masks, valid)
    assert got_t_a == t_a > 0 and counts == per_cnt
    assert float(got.detach()) == pytest.approx(want / t_a, rel=1e-12)
    assert all(sums[k] == pytest.approx(per_sum[k], rel=1e-12, abs=1e-12) for k in HEADS)
    acc, acc_h = BO.accuracy(logits, acts, masks, valid)
    assert acc == pytest.approx(right_tok / t_a, rel=1e-12)
    assert all(acc_h[k] == pytest.approx(per_right[k] / per_cnt[k] if per_cnt[k] else 0.0) for k in HEADS)
    got.backward()
    closed = BO.nll_dlogits(logits, acts, masks, valid)
    for k in HEADS:
        torch.testing.assert_close(lg[k].grad, closed[k], rtol=1e-12, atol=1e-15)
        m = masks[k].bool()
        in_s = acts[k].any(dim=1) & use
        by_hand = torch.where(in_s[:, None] & m, (1.0 / m.sum(1).clamp(min=1).double()[:, None] - acts[k].double()) / t_a, 0.0)
        torch.testing.assert_close(closed[k], by_hand, rtol=1e-12, atol=1e-15)


def test_oracle_ties_and_entropy_value_terms():
    """The arg-max takes the lowest index among equal maxima; bc_loss is the NLL plus the default objective's entropy and
    value terms (its policy term is 0 at zero advantages)."""
    import padding_oracle as PO
    L = 40
    logits, acts, masks = _uniform_case(7, L)
    g = torch.Generator().manual_seed(1)
    logits = {k: torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in logits.items()}
    t = int(torch.nonzero(acts["ability"].any(dim=1))[0])
    logits["ability"][t] = torch.tensor([2.0, 2.0, 1.0], dtype=torch.float64)
    for a, right in ((0, 1.0), (1, 0.0)):
        acts["ability"][t] = False
        acts["ability"][t, a] = True
        one = {k: v[t:t + 1] for k, v in logits.items()}
        _, per = BO.accuracy(one, {k: v[t:t + 1] for k, v in acts.items()}, {k: v[t:t + 1] for k, v in masks.items()})
        assert per["ability"] == right
    values = torch.randn(L, generator=g, dtype=torch.float64)
    ret = torch.randn(L, generator=g, dtype=torch.float64)
    loss, l_nll, e_loss, v_loss, _ = BO.bc_loss(logits, values, acts, masks, ret, 0.01, 0.5)
    _, p_loss, e_ref, v_ref, _ = PO.masked_ppo_loss(logits, values, acts, masks, torch.zeros(L, 5, dtype=torch.float64),
                                                    torch.ones(L, dtype=torch.float64), ret,
                                                    torch.ones(L, dtype=torch.bool), 0.01, 0.5, 0.2)
    assert float(e_loss) == float(e_ref) and float(v_loss) == float(v_ref)
    assert float(loss) == pytest.approx(float(l_nll + e_ref + v_ref), rel=1e-14)


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
    name = "dc_ppo_loss_fwd_bwd_bc"
    assert name in protos and name in _lib.SIGNATURES
    # _masked's arguments without old_logp, plus bc_stats
    assert len(_lib.SIGNATURES[name][1]) == protos[name] == protos["dc_ppo_loss_fwd_bwd_masked"]
    d = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DC_[A-Z0-9_]+)\s+(-?\d+)", open(HEADER).read())}
    assert d["DC_BC_STATS_SLOTS"] == _lib.BC_STATS_SLOTS == 2 + 2 * len(HEADS)


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_point_checks_its_arguments(lib):
    from dotaclient_b200 import _lib
    assert hasattr(lib, "dc_ppo_loss_fwd_bwd_bc") and lib.dc_version() >= 115
    one = 4096
    p5 = _lib._ptr5(*[one] * 5)
    ld = (_lib._c.c_int64 * 5)(4, 9, 9, 40, 3)
    short = (_lib._c.c_int64 * 5)(4, 9, 9, 39, 3)
    f = lib.dc_ppo_loss_fwd_bwd_bc

    def call(bc_stats=one, hparams=one, n=8, adv=one, ws=one, ld_l=ld, ld_v=1, logits=p5):
        return f(logits, ld_l, p5, p5, adv, one, one, ld_v, None, None, n, hparams, p5, ld, one, 1, one, one, bc_stats,
                 one, ws, None)
    # null operands, a bad token count or row pitch: refused before any CUDA call
    for kw, what in (({"bc_stats": None}, b"bc_stats"), ({"hparams": None}, b"hyper-parameter"), ({"n": 0}, b"N=0"),
                     ({"n": -5}, b"N=-5"), ({"adv": None}, b"null pointer"), ({"ws": None}, b"null pointer"),
                     ({"logits": _lib._ptr5(one, one, None, one, one)}, b"null pointer"),
                     ({"ld_l": short}, b"row pitch of head 3"), ({"ld_v": 0}, b"value pitch")):
        assert call(**kw) == -1, kw
        assert what in lib.dc_last_error(), (kw, lib.dc_last_error())


def test_ops_refuses_policy_gradient_operands_with_bc():
    from dotaclient_b200 import ops
    with pytest.raises(ValueError, match="behaviour cloning"):
        ops._bc_args(None, "cpu", True, None, None)
    with pytest.raises(ValueError, match="behaviour cloning"):
        ops._bc_args(None, "cpu", False, torch.zeros(1), None)
    with pytest.raises(ValueError, match="behaviour cloning"):
        ops._bc_args(None, "cpu", False, None, torch.zeros(1))
