"""Host-side checks of ``mask_padding``: the CLI flag and its validation, the C-ABI declaration and argument checks of
``dc_ppo_loss_fwd_bwd_masked``, the scan segment offsets and chunk lengths of experience prep, ``ExperienceBatch.valid``,
and the CPU oracle (``padding_oracle.py``) against hand-computed values, against the compaction identity and on the
reference prep."""
import copy
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import padding_oracle as PO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
SIZES = (4, 9, 9, 40, 3)


# ------------------------------------------------------------------------------------------------ CLI / validation
def test_cli_flag_and_default():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).mask_padding is False
    assert p.parse_args(["--mask-padding"]).mask_padding is True
    assert "--mask-padding" in p.format_help()


@pytest.mark.parametrize("bad", [1, 0, "yes", None, np.bool_(True), 1.0])
def test_non_bool_mask_padding_refused_up_front(bad):
    """Refused with ValueError before any device work (so this runs without a GPU), by the constructor, main() and
    check_ppo_settings."""
    from dotaclient_b200.optimizer import DotaOptimizer, check_ppo_settings, main
    with pytest.raises(ValueError, match="mask_padding"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, mask_padding=bad)
    with pytest.raises(ValueError, match="mask_padding"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, mask_padding=bad)
    with pytest.raises(ValueError, match="mask_padding"):
        check_ppo_settings(0.98, 0.97, 0.1, 0.5, None, mask_padding=bad)


def test_accepted_settings():
    from dotaclient_b200.optimizer import check_ppo_settings
    check_ppo_settings(0.98, 0.97, 0.1, 0.5)
    check_ppo_settings(0.98, 0.97, 0.1, 0.5, mask_padding=True)
    check_ppo_settings(0.98, 0.97, 0.1, 0.5, mask_padding=False)


# ------------------------------------------------------------------------------------------------ C ABI
def _params(name):
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^;]*?)\)\s*;" % name, text, flags=re.S)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_header_and_lib_table_agree_on_the_masked_entry_point():
    from dotaclient_b200 import _lib
    dev, masked = _params("dc_ppo_loss_fwd_bwd_dev"), _params("dc_ppo_loss_fwd_bwd_masked")
    args = _lib.SIGNATURES["dc_ppo_loss_fwd_bwd_masked"][1]
    assert len(masked) == len(args) == len(dev) + 1 == 22
    # the _dev list with `valid` inserted after old_value, before N
    assert masked[:10] == dev[:10] and masked[11:] == dev[10:]
    assert masked[10] == "const uint8_t *valid" and args[10] is _lib._c.c_void_p
    dev_args = _lib.SIGNATURES["dc_ppo_loss_fwd_bwd_dev"][1]
    assert list(args[:10]) == list(dev_args[:10]) and list(args[11:]) == list(dev_args[10:])


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_masked_entry_point_is_exported_and_checks_its_arguments(lib):
    """Argument errors return -1 with a message before any CUDA call (this box may have no GPU)."""
    from dotaclient_b200 import _lib
    assert hasattr(lib, "dc_ppo_loss_fwd_bwd_masked")
    assert lib.dc_version() >= 105
    one = 4096                                   # never dereferenced: validation fails first
    p5 = _lib._ptr5(*[one] * 5)
    ld = (_lib._c.c_int64 * 5)(4, 9, 9, 40, 3)

    def call(logits=p5, ld_l=ld, valid=one, n=8, hparams=one, dlogits=p5, ld_v=1, ws=one):
        return lib.dc_ppo_loss_fwd_bwd_masked(logits, ld_l, p5, p5, one, one, one, one, ld_v, None, valid, n, hparams,
                                              dlogits, ld, one, 1, one, one, one, ws, None)
    assert call(hparams=None) == -1 and b"hyper-parameter" in lib.dc_last_error()
    for n in (0, -3):
        assert call(n=n) == -1 and b"N=%d" % n in lib.dc_last_error()
    assert call(logits=_lib._ptr5(one, one, None, one, one)) == -1 and b"null pointer" in lib.dc_last_error()
    assert call(ws=None) == -1 and b"null pointer" in lib.dc_last_error()
    assert call(dlogits=_lib._ptr5(one, one, one, None, one)) == -1 and b"null dlogits[3]" in lib.dc_last_error()
    assert call(ld_l=(_lib._c.c_int64 * 5)(4, 9, 9, 39, 3)) == -1 and b"row pitch of head 3" in lib.dc_last_error()
    assert call(ld_v=0) == -1 and b"value pitch" in lib.dc_last_error()
    # a NULL valid mask is accepted: the same checks then fail the same way
    assert call(valid=None, hparams=None) == -1 and b"hyper-parameter" in lib.dc_last_error()


def test_ops_refuses_a_valid_mask_without_hparams():
    from dotaclient_b200 import ops
    with pytest.raises(ValueError, match="hyper-parameter"):
        ops._ppo_dev_args(None, None, None, 4, torch.device("cpu"), torch.ones(4, dtype=torch.bool))


# ------------------------------------------------------------------------------------------------ prep layout
@pytest.mark.parametrize("lengths,S,want", [
    ([40, 23, 48], 16, [0, 40, 48, 71, 80, 128, 128]),
    ([32, 16], 16, [0, 32, 32, 48, 48]),                       # exact multiples: every padding segment is empty
    ([1], 16, [0, 1, 16]),
    ([17, 1, 16], 16, [0, 17, 32, 33, 48, 64, 64]),
    ([1000, 1399], 512, [0, 1000, 1024, 2423, 2560]),
])
def test_padded_segment_offsets(lengths, S, want):
    from dotaclient_b200.optimizer import padded_segment_offsets
    got = padded_segment_offsets(lengths, S)
    assert got.dtype == np.int64 and got.tolist() == want
    lps = [(L + S - 1) // S * S for L in lengths]
    assert got[0::2].tolist() == np.concatenate([[0], np.cumsum(lps)]).tolist()    # rollout boundaries as without masking
    assert (np.diff(got)[0::2] == lengths).all() and (np.diff(got) >= 0).all()


def test_chunk_valid_lengths():
    from dotaclient_b200.optimizer import chunk_valid_lengths
    assert chunk_valid_lengths([40, 23, 48], 16) == [16, 16, 8, 16, 7, 16, 16, 16]
    assert chunk_valid_lengths([32, 16], 16) == [16, 16, 16]
    assert chunk_valid_lengths([1, 513], 512) == [1, 512, 1]
    lens = [5, 64, 65, 200]
    got = chunk_valid_lengths(lens, 64)
    assert sum(got) == sum(lens) and len(got) == sum((L + 63) // 64 for L in lens) and min(got) >= 1


# ------------------------------------------------------------------------------------------------ ExperienceBatch
def _tiny_batch(old_values, valid):
    from dotaclient_b200.optimizer import ExperienceBatch
    S, B = 4, 3
    obs = {"env": torch.zeros(S, B, 3)}
    masks = {"enum": torch.ones(S, B, 4, dtype=torch.bool)}
    actions = {"enum": torch.zeros(S, B, 4, dtype=torch.bool)}
    ov = torch.arange(S * B, dtype=torch.float32).view(S, B) if old_values else None
    vd = (torch.arange(S).view(S, 1) < torch.tensor([4, 4, 2])) if valid else None
    return ExperienceBatch(obs, masks, actions, torch.zeros(S, B, 5), torch.ones(S, B), torch.ones(S, B),
                           torch.zeros(1, B, 8), None, old_values=ov, valid=vd)


@pytest.mark.parametrize("old_values", [False, True])
def test_experience_batch_valid_is_optional_and_last(old_values):
    without, with_ = _tiny_batch(old_values, False), _tiny_batch(old_values, True)
    names = [k for _, k, _ in without.tensors()]
    assert "valid" not in names
    assert [k for _, k, _ in with_.tensors()] == names + ["valid"]      # appended: every other position unchanged
    assert with_.nbytes() == without.nbytes() + 12
    assert without.graph_key() == (4, 3, old_values)                     # batches without it: the key they always had
    assert with_.graph_key() == (4, 3, old_values, "valid") != without.graph_key()
    doubled = with_.map(lambda v: torch.cat([v, v], dim=1))
    assert doubled.valid.dtype == torch.bool and doubled.valid.shape == (4, 6)
    assert [(type(h), k) for h, k, _ in doubled.tensors()] == [(type(h), k) for h, k, _ in with_.tensors()]
    assert without.map(lambda v: v).valid is None
    if torch.cuda.is_available():                       # pinning needs the CUDA driver
        assert with_.pin_memory().graph_key() == with_.graph_key()


def test_from_sequences_stacks_valid_when_every_sequence_has_one():
    from dotaclient_b200.optimizer import ExperienceBatch, Sequence
    from dotaclient_b200.synthetic import make_rollout
    S = 4
    seqs = []
    for i in range(3):
        r = make_rollout(S, 40 + i)
        seqs.append(Sequence(None, 1, 0, r["observations"], r["actions"], r["masks"], None, None, torch.zeros(1, 1, 8),
                             old_logp=torch.zeros(S, 5), valid=torch.arange(S) < S - i))
        seqs[-1].advantages, seqs[-1].returns = torch.zeros(S), torch.zeros(S)
    b = ExperienceBatch.from_sequences(seqs, torch.device("cpu"))
    assert b.valid.shape == (S, 3) and b.valid.dtype == torch.bool
    assert b.valid.sum(dim=0).tolist() == [4, 3, 2]
    seqs[1].valid = None
    assert ExperienceBatch.from_sequences(seqs, torch.device("cpu")).valid is None
    assert Sequence(None, 1, 0, {}, {}, {}, None, None, None).valid is None


# ------------------------------------------------------------------------------------------------ CPU oracle
def _case(n, seed, invalid_actions=True):
    """Random flat loss inputs; the invalid rows (the last third, and a few inside) keep their actions when
    ``invalid_actions``."""
    from dotaclient_b200.synthetic import make_rollout
    g = torch.Generator().manual_seed(seed)
    roll = make_rollout(n, seed)
    masks = {k: roll["masks"][k].clone().bool() for k in PO.HEADS}
    actions = {k: roll["actions"][k].clone().bool() for k in PO.HEADS}
    logits = {k: torch.randn(n, s, generator=g) for k, s in zip(PO.HEADS, SIZES)}
    valid = torch.ones(n, dtype=torch.bool)
    valid[2 * n // 3:] = False
    valid[1] = False
    if not invalid_actions:
        for k in PO.HEADS:
            actions[k][~valid] = False
            masks[k][~valid] = False
    old = torch.zeros(n, 5)
    from oracle.ref_policy import masked_softmax
    for h, k in enumerate(PO.HEADS):
        lp = masked_softmax(logits[k] + 0.3 * torch.randn(logits[k].shape, generator=g), masks[k], dim=1)
        old[actions[k].any(dim=1), h] = lp[actions[k]]
    return (logits, torch.randn(n, generator=g), actions, masks, old, torch.randn(n, generator=g),
            torch.randn(n, generator=g), valid)


def test_oracle_against_hand_computed_values():
    """Two valid tokens of four, ratio 1 everywhere (old = new log-prob), one action row per token on 'enum' only:
    advantages [1, 3] normalise to -+1/sqrt(2) over the valid pair (mean 2, unbiased std sqrt(2)), the policy loss is
    -mean(adv_n) = 0 up to eps, and the value loss is 0.5 * vf_coef * mean((R - v)^2) over the pair alone."""
    from oracle.ref_policy import masked_softmax
    n = 4
    logits = {k: torch.zeros(n, s) for k, s in zip(PO.HEADS, SIZES)}
    masks = {k: torch.zeros(n, s, dtype=torch.bool) for k, s in zip(PO.HEADS, SIZES)}
    actions = {k: torch.zeros(n, s, dtype=torch.bool) for k, s in zip(PO.HEADS, SIZES)}
    masks["enum"][:, :2] = True
    actions["enum"][:, 0] = True                              # invalid rows 2, 3 hold actions too: they must not count
    old = torch.zeros(n, 5)
    old[:, 0] = masked_softmax(logits["enum"], masks["enum"], dim=1)[:, 0]           # log 1/2
    adv = torch.tensor([1.0, 3.0, 100.0, -50.0])
    ret = torch.tensor([1.0, 2.0, 9.0, 9.0])
    values = torch.tensor([0.0, 0.0, -9.0, 4.0])
    valid = torch.tensor([True, True, False, False])
    loss, p_loss, e_loss, v_loss, ents = PO.masked_ppo_loss(logits, values, actions, masks, old, adv, ret, valid,
                                                            entropy_coef=0.0, vf_coef=0.5, e_clip=0.1)
    assert abs(float(p_loss)) < 1e-6 / 5
    assert float(v_loss) == pytest.approx(0.5 * 0.5 * (1.0 + 4.0) / 2, rel=1e-6)
    assert float(ents["enum"]) == pytest.approx(math.log(2), rel=1e-6)             # per valid action row
    st = PO.masked_stats(logits, actions, masks, old, values, ret, valid, 0.1)
    assert st["approx_kl/enum"] == 0.0 and st["clip_fraction"] == 0.0
    # ret - v = [1, 2] over the valid pair: Var = 1/4, Var(ret) = 1/4 -> 0
    assert st["explained_variance"] == pytest.approx(0.0, abs=1e-12)
    # with every token valid the outliers enter the normalisation and the value loss
    full = PO.masked_ppo_loss(logits, values, actions, masks, old, adv, ret, torch.ones(n, dtype=torch.bool), 0.0, 0.5, 0.1)
    assert float(full[3]) == pytest.approx(0.5 * 0.5 * (1 + 4 + 324 + 25) / 4, rel=1e-6)


@pytest.mark.parametrize("clip", [None, 0.2])
@pytest.mark.parametrize("invalid_actions", [True, False])
def test_oracle_compaction_identity(clip, invalid_actions):
    """The masked loss and its gradients equal the reference loss on the valid rows alone; invalid rows get exactly
    zero gradient."""
    from oracle import ref_optimizer as RO
    logits, values, actions, masks, old, adv, ret, valid = _case(200, 5, invalid_actions)
    ov = values + 0.1 * torch.randn(200, generator=torch.Generator().manual_seed(1))
    lg = {k: t.clone().requires_grad_(True) for k, t in logits.items()}
    vg = values.clone().requires_grad_(True)
    got = PO.masked_ppo_loss(lg, vg, actions, masks, old, adv, ret, valid, 5e-4, 0.5, 0.1, old_values=ov, value_clip=clip)
    got[0].backward()
    # the valid rows, compacted by hand
    lc = {k: t[valid].clone().unsqueeze(0).requires_grad_(True) for k, t in logits.items()}
    vc = values[valid].clone().view(1, -1, 1).requires_grad_(True)
    ac = {k: a[valid].unsqueeze(0) for k, a in actions.items()}
    mc = {k: m[valid].unsqueeze(0) for k, m in masks.items()}
    oc = {k: old[valid][actions[k][valid].any(dim=1), h] for h, k in enumerate(PO.HEADS)}
    if clip is None:
        want = RO.ppo_loss(lc, vc, ac, mc, oc, adv[valid].view(1, -1), ret[valid].view(1, -1), 5e-4, 0.5, 0.1)
    else:
        want = PO.PC.ppo_loss(lc, vc, ac, mc, oc, adv[valid].view(1, -1), ret[valid].view(1, -1), 5e-4, 0.5, 0.1,
                              old_values=ov[valid].view(1, -1), value_clip=clip)
    want[0].backward()
    for a, b in zip(got[:4], want[:4]):
        assert torch.equal(a, b)
    for k in PO.HEADS:
        g = lg[k].grad if lg[k].grad is not None else torch.zeros_like(logits[k])
        assert torch.equal(g[~valid], torch.zeros_like(g[~valid]))
        gw = lc[k].grad[0] if lc[k].grad is not None else torch.zeros_like(g[valid])
        assert torch.equal(g[valid], gw), k
    assert torch.equal(vg.grad[~valid], torch.zeros(int((~valid).sum())))
    assert torch.equal(vg.grad[valid], vc.grad.view(-1))


def test_oracle_prep_bootstraps_at_the_real_end():
    """Reference prep vs masked prep on the CPU: identical for a rollout of two whole chunks; for a ragged one the real
    rows are GAE over the real steps with a trailing 0, the padded rows are 0, and the last real advantage differs from
    the reference's (which bootstraps from the padded observation's value)."""
    from oracle import ref_optimizer as RO
    from oracle.ref_policy import RefPolicy
    from dotaclient_b200.synthetic import make_rollout
    torch.manual_seed(7)
    pol = RefPolicy(64, "gru")
    S = 8
    whole = make_rollout(16, 3)
    a = RO.experiences_from_rollout(pol, copy.deepcopy(whole), S)
    b = PO.experiences_from_rollout(pol, copy.deepcopy(whole), S)
    for x, y in zip(a, b):
        assert torch.equal(x.advantages, y.advantages) and torch.equal(x.returns, y.returns)
        assert bool(y.valid.all())
    ragged = make_rollout(13, 4)
    a = RO.experiences_from_rollout(pol, copy.deepcopy(ragged), S)
    b = PO.experiences_from_rollout(pol, copy.deepcopy(ragged), S)
    assert [int(s.valid.sum()) for s in b] == [8, 5]
    adv = torch.cat([s.advantages for s in b]).numpy()
    ret = torch.cat([s.returns for s in b]).numpy()
    vals = torch.cat([s.values.reshape(-1) for s in b]).numpy()[:13]
    r = np.sum(np.asarray(ragged["rewards"], dtype=np.float32), axis=1)
    wa, wr = PO.real_advantage_returns(r, vals)
    np.testing.assert_array_equal(adv[:13], wa)
    np.testing.assert_array_equal(ret[:13], wr)
    assert (adv[13:] == 0).all() and (ret[13:] == 0).all()
    ref_adv = torch.cat([s.advantages for s in a]).numpy()
    assert adv[12] != ref_adv[12]
