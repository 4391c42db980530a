"""CPU tests of the value heads (``DotaOptimizer(value_heads=...)``): every refusal of the settings, the CLI flags, the
fold and split of the value head on a CPU ``Policy`` and against the float64 oracle, and a folded K-head model loading
strictly into the reference's network with the summed value."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import value_heads_oracle as VH  # noqa: E402

from dotaclient_b200.optimizer import build_arg_parser, check_ppo_settings, value_head_groups  # noqa: E402
from dotaclient_b200.policy import REWARD_KEYS, Policy, fold_value_heads, split_value_head  # noqa: E402

TWO = {'win': ['win'], 'shaping': [k for k in REWARD_KEYS if k != 'win']}


def check(**kw):
    check_ppo_settings(0.98, 0.97, 0.1, 0.5, None, **kw)


def test_valid_settings_and_groups():
    check(value_heads=TWO, value_gammas={'win': 0.999})
    vh = value_head_groups(TWO, {'win': 0.999}, 0.98)
    assert vh.names == ('win', 'shaping')
    assert vh.group.tolist() == [1, 0, 1, 1, 1, 1, 1, 1, 1, 1]
    assert vh.gammas.tolist() == [0.999, 0.98]
    assert value_head_groups(None, None, 0.98) is None
    assert value_head_groups({'all': REWARD_KEYS}, None, 0.9).gammas.tolist() == [0.9]


@pytest.mark.parametrize("heads, gammas, match", [
    ({}, None, "non-empty mapping"),
    (['win'], None, "non-empty mapping"),
    ({'': REWARD_KEYS}, None, "match"),
    ({'a-b': REWARD_KEYS}, None, "match"),
    ({'a': 'win'}, None, "must be a list"),
    ({'a': [], 'b': REWARD_KEYS}, None, "no reward keys"),
    ({'a': ['gold'] + REWARD_KEYS}, None, "not a reward key"),
    ({'a': REWARD_KEYS, 'b': ['win']}, None, "more than one"),
    ({'a': REWARD_KEYS[1:]}, None, "leaves the reward keys enemy out"),
    (TWO, {'other': 0.9}, "not a value head"),
    (TWO, {'win': 0.0}, r"\(0, 1\]"),
    (TWO, {'win': 1.5}, r"\(0, 1\]"),
    (TWO, {'win': float('nan')}, r"\(0, 1\]"),
    (TWO, {'win': True}, r"\(0, 1\]"),
    (TWO, [('win', 0.9)], "mapping"),
    (None, {'win': 0.9}, "needs value_heads"),
])
def test_malformed_value_heads_raise(heads, gammas, match):
    with pytest.raises(ValueError, match=match):
        check(value_heads=heads, value_gammas=gammas)


def test_refused_combinations():
    with pytest.raises(ValueError, match="vtrace"):
        check(value_heads=TWO, advantage_estimator='vtrace')
    with pytest.raises(ValueError, match="value_norm"):
        check(value_heads=TWO, value_norm=True)


def test_cli_flags():
    p = build_arg_parser()
    a = p.parse_args(['--value-heads', 'win=win;shaping=enemy,xp,hp,kills,death,lh,denies,tower_hp,mana',
                      '--value-gammas', 'win=0.999'])
    assert list(a.value_heads) == ['win', 'shaping'] and a.value_heads['win'] == ['win']
    assert a.value_heads['shaping'] == TWO['shaping'] and a.value_gammas == {'win': 0.999}
    check(value_heads=a.value_heads, value_gammas=a.value_gammas)
    a = p.parse_args([])
    assert a.value_heads is None and a.value_gammas is None
    for bad in (['--value-heads', 'win'], ['--value-heads', 'a=win;a=xp'], ['--value-gammas', 'win:0.9']):
        with pytest.raises(SystemExit):
            p.parse_args(bad)


def test_policy_value_heads_and_seeded_init():
    torch.manual_seed(7)
    ref = Policy()
    torch.manual_seed(7)
    pol = Policy(value_heads=3)
    assert tuple(pol.affine_value.weight.shape) == (3, 256) and tuple(pol.affine_value.bias.shape) == (3,)
    a, b = ref.state_dict(), pol.state_dict()
    assert list(a) == list(b)
    for k in a:
        if not k.startswith('affine_value'):
            assert torch.equal(a[k], b[k]), k
    for bad in (0, 11, 1.5, True):
        with pytest.raises(ValueError):
            Policy(value_heads=bad)


def test_fold_and_split_round_trips():
    torch.manual_seed(3)
    pol = Policy(hidden_size=64, value_heads=4)
    sd = pol.state_dict()
    folded = fold_value_heads(sd)
    w, b = sd['affine_value.weight'], sd['affine_value.bias']
    fw, fb = VH.fold(w.numpy(), b.numpy())
    np.testing.assert_allclose(folded['affine_value.weight'].numpy(), fw, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(folded['affine_value.bias'].numpy(), fb, rtol=1e-6, atol=1e-7)
    assert folded['affine_value.weight'].dtype == torch.float32 and tuple(folded['affine_value.weight'].shape) == (1, 64)
    # fp32 in head order: the fold is exactly the sequential sum
    seq = w[0] + w[1] + w[2] + w[3]
    assert torch.equal(folded['affine_value.weight'][0], seq)
    assert fold_value_heads(folded) == folded                      # one row: unchanged
    split = split_value_head(folded, 4)
    sw, sb = VH.split(folded['affine_value.weight'].numpy(), folded['affine_value.bias'].numpy(), 4)
    np.testing.assert_allclose(split['affine_value.weight'].numpy(), sw, rtol=1e-7)
    np.testing.assert_allclose(split['affine_value.bias'].numpy(), sb, rtol=1e-7)
    back = fold_value_heads(split)
    torch.testing.assert_close(back['affine_value.weight'], folded['affine_value.weight'], rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(back['affine_value.bias'], folded['affine_value.bias'], rtol=1e-6, atol=1e-7)
    Policy(hidden_size=64, value_heads=4).load_state_dict(split, strict=True)
    with pytest.raises(ValueError):
        split_value_head(sd, 2)


def test_folded_model_loads_strictly_into_the_reference_network():
    from oracle.ref_policy import RefPolicy
    torch.manual_seed(11)
    pol = Policy(value_heads=3)
    folded = fold_value_heads(pol.state_dict())
    ref = RefPolicy()
    ref.load_state_dict(folded, strict=True)
    # the value of a folded head is the sum of the heads' values on the same features
    y = torch.randn(5, 256)
    heads = pol.affine_value(y).double().sum(dim=1)
    torch.testing.assert_close(ref.affine_value(y).double()[:, 0], heads, rtol=1e-5, atol=1e-5)
