"""Host-side checks of the schedulable PPO settings and the PPO diagnostics: CLI flags, constructor validation, the
persistent ``param_groups``, the new C-ABI symbols, ``ExperienceBatch.old_values``, and the CPU oracle of the statistics and
of the clipped value loss against hand-computed values."""
import math
import os
import re
import sys
import uuid
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ppo_controls_oracle as PC  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
NEW_SYMBOLS = ("dc_ppo_loss_fwd_bwd_dev", "dc_grad_finish_dev")


# ------------------------------------------------------------------------------------------------ CLI / validation
def test_cli_flags_and_defaults():
    from dotaclient_b200.optimizer import GAMMA, LAMBDA, build_arg_parser
    p = build_arg_parser()
    a = p.parse_args([])
    assert (a.gamma, a.gae_lambda, a.clip_range, a.max_grad_norm, a.value_clip) == (GAMMA, LAMBDA, 0.1, 0.5, None)
    assert (GAMMA, LAMBDA) == (0.98, 0.97)
    a = p.parse_args(["--gamma", "0.999", "--gae-lambda", "0.9", "--clip-range", "0.2", "--max-grad-norm", "1.5",
                      "--value-clip", "0.3"])
    assert (a.gamma, a.gae_lambda, a.clip_range, a.max_grad_norm, a.value_clip) == (0.999, 0.9, 0.2, 1.5, 0.3)
    text = p.format_help()
    for flag in ("--gamma", "--gae-lambda", "--clip-range", "--max-grad-norm", "--value-clip"):
        assert flag in text


BAD_SETTINGS = [dict(gamma=0.0), dict(gamma=1.01), dict(gamma=float("nan")), dict(gamma="0.9"), dict(gae_lambda=-0.1),
                dict(gae_lambda=1.5), dict(clip_range=0.0), dict(clip_range=-0.1), dict(max_grad_norm=0.0),
                dict(max_grad_norm=float("nan")), dict(value_clip=-0.2), dict(gamma=True)]


@pytest.mark.parametrize("bad", BAD_SETTINGS)
def test_constructor_and_main_reject_bad_settings_up_front(bad):
    """Refused with ValueError before any device work (so this runs without a GPU), by the constructor and by main()."""
    from dotaclient_b200.optimizer import DotaOptimizer, main
    name = next(iter(bad))
    with pytest.raises(ValueError, match=name):
        DotaOptimizer("x", 0, 1, 1, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, **bad)
    with pytest.raises(ValueError, match=name):
        main("x", 0, 1, 1, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, **bad)


def test_domain_edges_are_accepted():
    from dotaclient_b200.optimizer import check_ppo_settings
    check_ppo_settings(1.0, 0.0, 1e-6, 1e-6, None)
    check_ppo_settings(1e-9, 1.0, 10.0, 100.0, 0.0)
    check_ppo_settings(np.float32(0.99), np.float64(0.95), 0.2, 1, 0.5)


# ------------------------------------------------------------------------------------------------ param_groups
def _adam_handle():
    from dotaclient_b200.flat import FlatParameterSpace
    from dotaclient_b200.optimizer import DotaOptimizer, _FusedAdamHandle
    from dotaclient_b200.policy import Policy
    flat = FlatParameterSpace(Policy(hidden_size=64, cell="gru"))
    owner = SimpleNamespace(flat=flat, exp_avg=torch.zeros_like(flat.param), exp_avg_sq=torch.zeros_like(flat.param),
                            adam_steps=torch.zeros(flat.n_seg, dtype=torch.int32), learning_rate=5e-5,
                            ADAM_BETAS=DotaOptimizer.ADAM_BETAS, ADAM_EPS=DotaOptimizer.ADAM_EPS)
    return owner, _FusedAdamHandle(owner)


def test_param_group_lr_writes_reach_learning_rate():
    owner, h = _adam_handle()
    groups = h.param_groups
    assert groups is h.param_groups and len(groups) == 1          # persistent: the torch idiom writes into a kept dict
    g = groups[0]
    assert g["lr"] == 5e-5 and g["betas"] == (0.9, 0.999) and g["eps"] == 1e-8 and g["weight_decay"] == 0
    assert [p is q for p, q in zip(g["params"], owner.flat.params)] == [True] * owner.flat.n_seg
    h.param_groups[0]["lr"] = 3e-4
    assert owner.learning_rate == 3e-4
    assert h.state_dict()["param_groups"][0]["lr"] == 3e-4
    owner.learning_rate = 1e-5                                     # and the other way round
    assert g["lr"] == 1e-5 and dict(g)["lr"] == 1e-5 and h.state_dict()["param_groups"][0]["lr"] == 1e-5
    for group in h.param_groups:                                  # the scheduler-style loop
        group["lr"] *= 0.5
    assert owner.learning_rate == 5e-6
    assert set(g) == {"lr", "betas", "eps", "weight_decay", "params"} and len(g) == 5
    g["custom"] = 1
    assert g["custom"] == 1 and owner.learning_rate == 5e-6
    with pytest.raises(KeyError):
        del g["lr"]


# ------------------------------------------------------------------------------------------------ C ABI
def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(dc_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", text, flags=re.S):
        args = m.group(2).strip()
        protos[m.group(1)] = 0 if args in ("", "void") else args.count(",") + 1
    return protos


def _defines():
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DC_[A-Z0-9_]+)\s+(-?\d+)", open(HEADER).read())}


def test_header_and_lib_table_agree_on_the_new_entry_points():
    from dotaclient_b200 import _lib
    protos = _declared()
    for name in NEW_SYMBOLS:
        assert name in protos and name in _lib.SIGNATURES, name
        assert len(_lib.SIGNATURES[name][1]) == protos[name], name
    d = _defines()
    assert d["DC_HPARAM_SLOTS"] == _lib.HPARAM_SLOTS and d["DC_PPO_STATS_SLOTS"] == _lib.PPO_STATS_SLOTS
    assert [d["DC_HP_" + k] for k in ("LR", "E_CLIP", "ENTROPY_COEF", "VF_COEF", "MAX_GRAD_NORM", "VALUE_CLIP")] == \
        [_lib.HP_LR, _lib.HP_E_CLIP, _lib.HP_ENTROPY_COEF, _lib.HP_VF_COEF, _lib.HP_MAX_GRAD_NORM, _lib.HP_VALUE_CLIP]
    assert (d["DC_STAT_APPROX_KL"], d["DC_STAT_CLIP_FRACTION"], d["DC_STAT_EXPLAINED_VAR"]) == \
        (_lib.STAT_APPROX_KL, _lib.STAT_CLIP_FRACTION, _lib.STAT_EXPLAINED_VAR)
    assert d["DC_PPO_WORKSPACE_BYTES"] == _lib.PPO_WORKSPACE_BYTES and d["DC_LOSS_SLOTS"] == _lib.LOSS_SLOTS


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_new_symbols_are_exported_and_check_their_arguments(lib):
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name), name
    assert lib.dc_version() >= 102
    from dotaclient_b200 import _lib
    one = 4096
    p5 = _lib._ptr5(*[one] * 5)
    ld = (_lib._c.c_int64 * 5)(4, 9, 9, 40, 3)
    # a null hyper-parameter block is refused before anything is launched
    rc = lib.dc_ppo_loss_fwd_bwd_dev(p5, ld, p5, p5, one, one, one, one, 1, None, 8, None, p5, ld, one, 1, one, one, one,
                                     one, None)
    assert rc == -1 and b"hyper-parameter" in lib.dc_last_error()
    rc = lib.dc_grad_finish_dev(one, one, one, one, one, one, one, one, 3, 100, None, 0.9, 0.999, 1e-8, one, one, one, None)
    assert rc == -1 and b"hyper-parameter" in lib.dc_last_error()


# ------------------------------------------------------------------------------------------------ ExperienceBatch
def _tiny_batch(old_values):
    from dotaclient_b200.optimizer import ExperienceBatch
    S, B = 4, 3
    obs = {"env": torch.zeros(S, B, 3)}
    masks = {"enum": torch.ones(S, B, 4, dtype=torch.bool)}
    actions = {"enum": torch.zeros(S, B, 4, dtype=torch.bool)}
    ov = torch.arange(S * B, dtype=torch.float32).view(S, B) if old_values else None
    return ExperienceBatch(obs, masks, actions, torch.zeros(S, B, 5), torch.ones(S, B), torch.ones(S, B),
                           torch.zeros(1, B, 8), None, old_values=ov)


def test_experience_batch_old_values_is_optional():
    without, with_ = _tiny_batch(False), _tiny_batch(True)
    names = [k for _, k, _ in without.tensors()]
    assert "old_values" not in names and names[-4:] == ["advantages", "returns", "old_logp", "h0"]
    names2 = [k for _, k, _ in with_.tensors()]
    assert names2 == names + ["old_values"]                       # appended: positions of every other tensor unchanged
    assert with_.nbytes() == without.nbytes() + 4 * 12
    from dotaclient_b200.optimizer import ExperienceBatch
    positional = ExperienceBatch(without.observations, without.masks, without.actions, without.old_logp, without.advantages,
                                 without.returns, without.h0)
    assert positional.old_values is None and positional.c0 is None


@pytest.mark.parametrize("old_values", [False, True])
def test_experience_batch_map_keeps_structure(old_values):
    batch = _tiny_batch(old_values)
    doubled = batch.map(lambda v: torch.cat([v, v], dim=-1))
    assert doubled.c0 is None and (doubled.old_values is None) == (not old_values)
    assert [(type(h), k) for h, k, _ in doubled.tensors()] == [(type(h), k) for h, k, _ in batch.tensors()]
    for (_, _, a), (_, _, b) in zip(batch.tensors(), doubled.tensors()):
        assert b.dtype == a.dtype and b.shape == a.shape[:-1] + (2 * a.shape[-1],) and torch.equal(b[..., :a.shape[-1]], a)
    same = batch.map(lambda v: v)
    assert all(a is b for (_, _, a), (_, _, b) in zip(batch.tensors(), same.tensors()))
    assert same.graph_key() == batch.graph_key() == (4, 3, old_values)
    if torch.cuda.is_available():                       # pinning needs the CUDA driver
        assert batch.pin_memory().graph_key() == batch.graph_key()


def test_from_sequences_fills_old_values_from_sequence_values():
    from dotaclient_b200.optimizer import ExperienceBatch, Sequence
    from dotaclient_b200.synthetic import make_rollout
    S = 4
    seqs = []
    for i in range(3):
        r = make_rollout(S, 30 + i)
        seqs.append(Sequence(None, 1, 0, r["observations"], r["actions"], r["masks"],
                             torch.arange(S, dtype=torch.float32).view(1, S, 1) + 10 * i, None, torch.zeros(1, 1, 8),
                             old_logp=torch.zeros(S, 5)))
        seqs[-1].advantages, seqs[-1].returns = torch.zeros(S), torch.zeros(S)
    b = ExperienceBatch.from_sequences(seqs, torch.device("cpu"))
    seqs[1].values = None
    b_none = ExperienceBatch.from_sequences(seqs, torch.device("cpu"))
    assert b.old_values.shape == (S, 3) and b.old_values.dtype == torch.float32
    assert torch.equal(b.old_values[:, 2], torch.arange(S, dtype=torch.float32) + 20)
    assert b_none.old_values is None


# ------------------------------------------------------------------------------------------------ CPU oracle
def _one_head_case(heads_used=("x",)):
    """Two action rows on each used head, uniform logits over 2 masked entries (log-prob -log 2): old log-probs chosen so
    that r = 1.2 on the first row and r = 1 on the second.  Other heads: no action rows."""
    logits, masks, actions, old = {}, {}, {}, {}
    for k, n in zip(PC.HEADS, (4, 9, 9, 40, 3)):
        logits[k] = torch.zeros(3, n)
        masks[k] = torch.zeros(3, n, dtype=torch.bool)
        masks[k][:, :2] = True
        actions[k] = torch.zeros(3, n, dtype=torch.bool)
        old[k] = torch.zeros(0)
        if k in heads_used:
            actions[k][0, 0] = actions[k][1, 1] = True            # row 2: no action (padding-like)
            old[k] = torch.tensor([-math.log(2) - math.log(1.2), -math.log(2)])
    return logits, masks, actions, old


def test_oracle_statistics_against_hand_computed_values():
    logits, masks, actions, old = _one_head_case(("x", "ability"))
    ret = torch.tensor([1.0, 2.0, 3.0])
    v = torch.tensor([1.0, 2.0, 2.0])
    st = PC.ppo_stats(logits, masks, actions, old, v, ret, e_clip=0.1)
    kl_row = 0.2 - math.log(1.2)                                   # (r - 1) - log r at r = 1.2; 0 at r = 1
    for k in ("x", "ability"):
        assert st["approx_kl/" + k] == pytest.approx(kl_row / 2, rel=1e-6)
        assert st["clip_fraction/" + k] == 0.5                     # |1.2 - 1| > 0.1, |1 - 1| is not
    for k in ("enum", "y", "target_unit"):                         # no action rows: 0, left out of the means
        assert st["approx_kl/" + k] == 0.0 and st["clip_fraction/" + k] == 0.0
    assert st["approx_kl"] == pytest.approx(kl_row / 2, rel=1e-6) and st["clip_fraction"] == 0.5
    # ret - v = [0, 0, 1]: Var = 1/3 - 1/9 = 2/9; Var(ret) = 14/3 - 4 = 2/3  ->  1 - 1/3
    assert st["explained_variance"] == pytest.approx(2.0 / 3.0, rel=1e-12)
    st = PC.ppo_stats(logits, masks, actions, old, v, ret, e_clip=0.25)
    assert st["clip_fraction"] == 0.0
    assert math.isnan(PC.ppo_stats(logits, masks, actions, old, v, torch.ones(3), 0.1)["explained_variance"])
    none = PC.ppo_stats(logits, masks, {k: torch.zeros_like(a) for k, a in actions.items()},
                        {k: torch.zeros(0) for k in old}, v, ret, 0.1)
    assert none["approx_kl"] == 0.0 and none["clip_fraction"] == 0.0


def test_oracle_clipped_value_loss_against_hand_computed_values():
    # v = 1, v_old = 0, R = 0.5, eps = 0.2: (v - R)^2 = 0.25 > (0.2 - 0.5)^2 = 0.09 -> the unclipped branch, gradient v - R
    # v = 1, v_old = 0, R = 2,   eps = 0.2: (0.2 - 2)^2 = 3.24 > 1 -> the clipped branch, outside the range: no gradient
    # v = 1, v_old = 0.9, R = 0: inside the range the clipped value is v itself: both branches tie at 1, full gradient
    v = torch.tensor([1.0, 1.0, 1.0], requires_grad=True)
    loss = PC.clipped_value_loss(v, torch.tensor([0.0, 0.0, 0.9]), torch.tensor([0.5, 2.0, 0.0]), vf_coef=0.5,
                                 value_clip=0.2)
    assert float(loss) == pytest.approx(0.5 * 0.5 * (0.25 + 3.24 + 1.0) / 3, rel=1e-6)
    loss.backward()
    np.testing.assert_allclose(v.grad.numpy(), [0.5 * 0.5 / 3, 0.0, 0.5 * 1.0 / 3], rtol=1e-6)


def test_oracle_loss_without_value_clip_is_the_reference_loss():
    from oracle import ref_optimizer as RO
    g = torch.Generator().manual_seed(3)
    logits, masks, actions, old = _one_head_case(("enum", "x"))
    lg = {k: (t + 0.1 * torch.randn(t.shape, generator=g)).unsqueeze(0) for k, t in logits.items()}
    a1 = {k: t.unsqueeze(0) for k, t in actions.items()}
    m1 = {k: t.unsqueeze(0) for k, t in masks.items()}
    vals = torch.randn(1, 3, 1, generator=g)
    adv, ret = torch.randn(1, 3, generator=g), torch.randn(1, 3, generator=g)
    want = RO.ppo_loss(lg, vals, a1, m1, old, adv, ret, 5e-4, 0.5, 0.1)
    got = PC.ppo_loss(lg, vals, a1, m1, old, adv, ret, 5e-4, 0.5, 0.1, old_values=vals.view(1, 3), value_clip=None)
    for a, b in zip(want[:4], got[:4]):
        assert torch.equal(a, b)
    clipped = PC.ppo_loss(lg, vals, a1, m1, old, adv, ret, 5e-4, 0.5, 0.1, old_values=vals.view(1, 3), value_clip=0.2)
    # old values == values: the clipped branch equals the unclipped one, the loss is the reference loss
    assert float(clipped[3]) == pytest.approx(float(want[3]), rel=1e-6)
    assert float(clipped[0]) == pytest.approx(float(want[0]), rel=1e-6)
