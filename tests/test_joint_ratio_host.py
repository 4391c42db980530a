"""Host-side checks of ``policy_ratio='joint'``: the setting's validation, the CLI flag and ``main`` passing it through,
the C-ABI declaration and argument checks of ``dc_ppo_loss_fwd_bwd_joint``, the statistics keys, and the CPU oracle
(``joint_ratio_oracle.py``) against a hand-computed two-step example and against the per-head objective when only
``enum`` is ever sampled."""
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import joint_ratio_oracle as JO  # noqa: E402
import padding_oracle as PO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
SIZES = (4, 9, 9, 40, 3)
HEADS = JO.HEADS


# ------------------------------------------------------------------------------------------------ settings / CLI
def test_accepted_settings_and_default():
    from dotaclient_b200.optimizer import POLICY_RATIOS, check_ppo_settings
    assert POLICY_RATIOS == ("per_head", "joint")
    check_ppo_settings(0.98, 0.97, 0.1, 0.5)
    for mode in POLICY_RATIOS:
        check_ppo_settings(0.98, 0.97, 0.1, 0.5, policy_ratio=mode, mask_padding=True, pack_sequences=True,
                           advantage_estimator="vtrace", num_minibatches=4, value_clip=0.2)


@pytest.mark.parametrize("bad", ["Joint", "per-head", "", None, 1, True, ("joint",)])
def test_bad_policy_ratio_refused_up_front(bad):
    """Refused with ValueError before any device work (so this runs without a GPU), by check_ppo_settings, the
    constructor and main()."""
    from dotaclient_b200.optimizer import DotaOptimizer, check_ppo_settings, main
    with pytest.raises(ValueError, match="policy_ratio"):
        check_ppo_settings(0.98, 0.97, 0.1, 0.5, None, policy_ratio=bad)
    with pytest.raises(ValueError, match="policy_ratio"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, policy_ratio=bad)
    with pytest.raises(ValueError, match="policy_ratio"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, policy_ratio=bad)


def test_cli_flag():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).policy_ratio == "per_head"
    assert p.parse_args(["--policy-ratio", "joint"]).policy_ratio == "joint"
    assert p.parse_args(["--policy-ratio", "per_head"]).policy_ratio == "per_head"
    assert "--policy-ratio" in p.format_help()
    with pytest.raises(SystemExit):
        p.parse_args(["--policy-ratio", "product"])


@pytest.mark.parametrize("mode", ["per_head", "joint", None])
def test_main_passes_the_policy_ratio_to_the_optimizer(mode, monkeypatch):
    from dotaclient_b200 import optimizer as O
    seen = {}

    class Fake:
        mq = None

        def __init__(self, **kw):
            seen.update(kw)

        def run(self):
            seen["ran"] = True

    monkeypatch.setattr(O, "DotaOptimizer", Fake)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    kw = {} if mode is None else {"policy_ratio": mode}
    O.main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, mask_padding=True, **kw)
    assert seen["policy_ratio"] == (mode or "per_head") and seen["ran"] and seen["mask_padding"] is True


def test_stats_dict_gains_the_joint_keys_only_in_joint_mode():
    from dotaclient_b200 import _lib
    from dotaclient_b200.optimizer import DotaOptimizer
    st = [float(i) for i in range(_lib.PPO_STATS_SLOTS)]
    default = DotaOptimizer._ppo_stats_dict(st)
    joint = DotaOptimizer._ppo_stats_dict(st, joint=True)
    assert "approx_kl/joint" not in default and "clip_fraction/joint" not in default
    assert set(joint) - set(default) == {"approx_kl/joint", "clip_fraction/joint"}
    assert all(joint[k] == v for k, v in default.items())
    assert joint["approx_kl/joint"] == 13.0 and joint["clip_fraction/joint"] == 14.0


# ------------------------------------------------------------------------------------------------ C ABI
def _params(name):
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^;]*?)\)\s*;" % name, text, flags=re.S)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_header_and_lib_table_agree_on_the_joint_entry_point():
    from dotaclient_b200 import _lib
    assert _params("dc_ppo_loss_fwd_bwd_joint") == _params("dc_ppo_loss_fwd_bwd_masked")
    assert list(_lib.SIGNATURES["dc_ppo_loss_fwd_bwd_joint"][1]) == list(_lib.SIGNATURES["dc_ppo_loss_fwd_bwd_masked"][1])
    text = open(HEADER).read()
    assert re.search(r"#define DC_STAT_JOINT_APPROX_KL %d\b" % _lib.STAT_JOINT_APPROX_KL, text)
    assert re.search(r"#define DC_STAT_JOINT_CLIP_FRACTION %d\b" % _lib.STAT_JOINT_CLIP_FRACTION, text)


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_joint_entry_point_is_exported_and_checks_its_arguments(lib):
    """Argument errors return -1 with a message before any CUDA call (this box may have no GPU)."""
    from dotaclient_b200 import _lib
    assert hasattr(lib, "dc_ppo_loss_fwd_bwd_joint")
    assert lib.dc_version() >= 107
    one = 4096                                   # never dereferenced: validation fails first
    p5 = _lib._ptr5(*[one] * 5)
    ld = (_lib._c.c_int64 * 5)(4, 9, 9, 40, 3)

    def call(logits=p5, ld_l=ld, valid=one, n=8, hparams=one, dlogits=p5, ld_v=1, ws=one):
        return lib.dc_ppo_loss_fwd_bwd_joint(logits, ld_l, p5, p5, one, one, one, one, ld_v, None, valid, n, hparams,
                                             dlogits, ld, one, 1, one, one, one, ws, None)
    assert call(hparams=None) == -1 and b"dc_ppo_loss_fwd_bwd_joint: null hyper-parameter" in lib.dc_last_error()
    for n in (0, -3):
        assert call(n=n) == -1 and b"N=%d" % n in lib.dc_last_error()
    assert call(logits=_lib._ptr5(one, one, None, one, one)) == -1 and b"null pointer" in lib.dc_last_error()
    assert call(ws=None) == -1 and b"null pointer" in lib.dc_last_error()
    assert call(dlogits=_lib._ptr5(one, one, one, None, one)) == -1 and b"null dlogits[3]" in lib.dc_last_error()
    assert call(ld_l=(_lib._c.c_int64 * 5)(4, 9, 9, 39, 3)) == -1 and b"row pitch of head 3" in lib.dc_last_error()
    assert call(ld_v=0) == -1 and b"value pitch" in lib.dc_last_error()
    assert call(valid=None, hparams=None) == -1 and b"hyper-parameter" in lib.dc_last_error()   # NULL valid accepted


def test_ops_refuses_the_joint_loss_without_hparams():
    from dotaclient_b200 import ops
    with pytest.raises(ValueError, match="joint-ratio PPO loss needs the device hyper-parameter block"):
        ops._ppo_dev_args(None, None, None, 4, torch.device("cpu"), None, joint=True)


# ------------------------------------------------------------------------------------------------ CPU oracle
def _empty(n):
    logits = {k: torch.zeros(n, s, dtype=torch.float64) for k, s in zip(HEADS, SIZES)}
    masks = {k: torch.zeros(n, s, dtype=torch.bool) for k, s in zip(HEADS, SIZES)}
    actions = {k: torch.zeros(n, s, dtype=torch.bool) for k, s in zip(HEADS, SIZES)}
    return logits, masks, actions


def test_oracle_against_a_hand_computed_move_and_attack_step():
    """Uniform logits.  Step 0 moves (enum 0, x 2, y 3), step 1 attacks (enum 1, target_unit 0 of 4 visible units); the old
    log-probs are offset so that log r_0 = 0.05 + 0.05 - 0.02 = 0.08 (inside [0.9, 1.1]) and log r_1 = -0.1 - 0.1 = -0.2
    (below).  Advantages [1, 3] normalise to -+1/sqrt(2)."""
    logits, masks, actions = _empty(2)
    masks["enum"][:, :2] = True
    masks["x"][0] = masks["y"][0] = True
    masks["target_unit"][1, :4] = True
    actions["enum"][0, 0] = actions["enum"][1, 1] = True
    actions["x"][0, 2] = actions["y"][0, 3] = True
    actions["target_unit"][1, 0] = True
    old = torch.zeros(2, 5, dtype=torch.float64)
    old[0, 0], old[0, 1], old[0, 2] = math.log(1 / 2) - 0.05, math.log(1 / 9) - 0.05, math.log(1 / 9) + 0.02
    old[1, 0], old[1, 3] = math.log(1 / 2) + 0.1, math.log(1 / 4) + 0.1
    old[0, 3], old[1, 1], old[1, 4] = 123.0, -7.0, 55.0        # heads without an action row: ignored
    adv = torch.tensor([1.0, 3.0], dtype=torch.float64)
    lg = {k: t.clone().requires_grad_(True) for k, t in logits.items()}
    loss, p_loss, e_loss, v_loss, ents = JO.joint_ppo_loss(lg, torch.zeros(2), actions, masks, old, adv, torch.zeros(2),
                                                           0.0, 0.0, 0.1)
    a = 1.0 / (math.sqrt(2.0) + 1.1920928955078125e-07)
    r0, r1 = math.exp(0.08), math.exp(-0.2)
    # step 0: r0 in range, both surrogates equal -r0 a; step 1: r1 < 0.9 and A > 0, so the unclipped r1 a is the minimum
    want = -(-r0 * a + r1 * a) / 2
    assert float(p_loss.detach()) == pytest.approx(want, rel=1e-12)
    assert float(loss.detach()) == float(p_loss.detach()) and float(e_loss) == 0.0 and float(v_loss) == 0.0
    assert float(ents["enum"]) == pytest.approx(math.log(2), rel=1e-12)
    assert float(ents["ability"]) == 0.0
    loss.backward()
    g0, g1 = -0.5 * (-a) * r0, -0.5 * a * r1           # d loss / d logp of every sampled head of the step
    ge = lg["enum"].grad
    np.testing.assert_allclose(ge[0].numpy(), [g0 / 2, -g0 / 2, 0, 0], rtol=1e-12)
    np.testing.assert_allclose(ge[1].numpy(), [-g1 / 2, g1 / 2, 0, 0], rtol=1e-12)
    want_x = np.full(9, -g0 / 9)
    want_x[2] += g0
    np.testing.assert_allclose(lg["x"].grad[0].numpy(), want_x, rtol=1e-12)
    assert float(lg["x"].grad[1].abs().max()) == 0.0
    want_tu = np.zeros(40)
    want_tu[:4] = -g1 / 4
    want_tu[0] += g1
    np.testing.assert_allclose(lg["target_unit"].grad[1].numpy(), want_tu, rtol=1e-12, atol=1e-15)
    assert lg["ability"].grad is None or float(lg["ability"].grad.abs().max()) == 0.0
    st = JO.joint_stats(logits, actions, masks, old, 0.1)
    assert st["approx_kl/joint"] == pytest.approx(((math.expm1(0.08) - 0.08) + (math.expm1(-0.2) + 0.2)) / 2, rel=1e-9)
    assert st["clip_fraction/joint"] == 0.5
    # with step 1 left out, T_a = 1 and only step 0 counts (its advantage alone has a NaN std: compare the statistics)
    st = JO.joint_stats(logits, actions, masks, old, 0.1, valid=torch.tensor([True, False]))
    assert st == {"approx_kl/joint": pytest.approx(math.expm1(0.08) - 0.08, rel=1e-9), "clip_fraction/joint": 0.0}


def test_oracle_with_no_action_rows_has_no_policy_loss():
    logits, masks, actions = _empty(3)
    masks["enum"][:] = True
    lg = {k: t.clone().requires_grad_(True) for k, t in logits.items()}
    out = JO.joint_ppo_loss(lg, torch.zeros(3), actions, masks, torch.zeros(3, 5), torch.tensor([1.0, 2.0, 4.0]),
                            torch.ones(3), 5e-4, 0.5, 0.1)
    assert float(out[1]) == 0.0 and float(out[3]) == pytest.approx(0.25)
    assert JO.joint_stats(logits, actions, masks, torch.zeros(3, 5), 0.1) == {"approx_kl/joint": 0.0,
                                                                               "clip_fraction/joint": 0.0}


@pytest.mark.parametrize("masked", [False, True])
def test_oracle_is_five_times_the_per_head_objective_when_only_enum_is_sampled(masked):
    """Only enum ever sampled: S_t = {enum}, so the joint policy loss is 5x the per-head one (whose mean over five heads
    counts the four unused heads as 0), and so is its gradient (entropy and value terms off)."""
    import test_padding_host as H
    logits, values, actions, masks, old, adv, ret, valid = H._case(300, 17)
    for k in HEADS[1:]:
        actions[k][:] = False
    old[:, 1:] = 0.0
    if not masked:
        valid = torch.ones(300, dtype=torch.bool)
    lj = {k: t.double().requires_grad_(True) for k, t in logits.items()}
    lh = {k: t.double().requires_grad_(True) for k, t in logits.items()}
    joint = JO.joint_ppo_loss(lj, values, actions, masks, old.double(), adv.double(), ret, 0.0, 0.0, 0.1,
                              valid=valid if masked else None)
    head = PO.masked_ppo_loss(lh, values.double(), actions, masks, old.double(), adv.double(), ret.double(), valid, 0.0, 0.0,
                              0.1)
    assert float(head[1]) != 0.0
    assert float(joint[1]) == pytest.approx(5 * float(head[1]), rel=1e-12)
    joint[0].backward()
    head[0].backward()
    for k in HEADS:
        gj = lj[k].grad if lj[k].grad is not None else torch.zeros_like(lj[k])
        gh = lh[k].grad if lh[k].grad is not None else torch.zeros_like(lh[k])
        torch.testing.assert_close(gj, 5 * gh, rtol=1e-12, atol=1e-15)
    assert float(lj["enum"].grad.abs().max()) > 0
