"""The PPO loss (``csrc/ppo_loss.cu`` through ``ops.ppo_loss_packed``, the path ``DotaOptimizer`` runs) on hard inputs,
against a float64 reference, at the benchmark's token counts.

``reference`` is the loss of ``padding_oracle.masked_ppo_loss`` (per head) and ``joint_ratio_oracle.joint_ppo_loss``
(joint ratio) with their diagnostics, written for any dtype and device: those oracles exponentiate every logit, so a masked
logit of +1e4 overflows and gives NaN gradients, and the joint oracle is float64 on the CPU only.  Here the exponential
is taken on the mask's entries only, as the kernel does.  ``test_reference_matches_the_oracles`` shows, on the CPU, that
it equals those oracles in float64 on ordinary inputs.  The same function in fp32 calibrates the bound every kernel
output must meet, per tensor:

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

Inputs: logits up to |60| on the mask (the masked log-softmax has no max-subtraction and uses ``__expf``), +-1e4 off it,
rows with one entry, log-ratios in +-3 (all four clip cases), advantages with |mean| / std = 1e3, about 10 % padding.

Measured on one H100 80GB HBM3 (700 W power limit), over the 22 cases of ``test_ppo_loss_hard_inputs_vs_fp64``, the
largest ratio max|gpu - f64| / max|torch32 - f64| and, in brackets, the largest max|gpu - f64| / max|f64|:
    dlogits   1.1  (4.6e-5)
    dvalue    1.23 (9.6e-8)
    scalars   174  (5.6e-5)
The scalars (losses, entropies, advantage mean / std, diagnostics) are float64 sums in the kernel and fp32 reductions in
torch, whose error is sometimes far below an fp32 ulp of the result: their floor of 4e-6 of |f64| carries them.  The
dlogits and dvalue bound K = 4 leaves a margin of 3.
Near-constant returns (c + 1e-3 noise, c = 0.7, -2.37, 300): the kernel's explained variance is within 2.4e-8 of the
two-pass float64 value; torch fp32 is up to 6e-4 off at c = 300.

Constant returns: before the explained-variance sums were shifted by the first counting token's values, the kernel
reported -1.2e14 to -2.3e16 instead of NaN for returns of 0.7 or 1.1 in four of the six token-count / padding cases of
``test_explained_variance_of_constant_returns_is_nan``: the rounding of its one-pass float64 sums left a tiny positive
Var(ret).
"""
import math

import pytest
import torch

E_CLIP = 0.2
EPS = float(torch.finfo(torch.float32).eps)             # the advantage normalisation's eps (policy.py:15)
HEADS = ("enum", "x", "y", "target_unit", "ability")
SIZES = (4, 9, 9, 40, 3)
PACK = {"enum": (0, 4), "x": (4, 13), "y": (13, 22), "ability": (22, 25)}     # ops.PACK_COLS
VALUE_COL = 25
# (K, FLOOR) per kind of output
BOUNDS = {"scalar": (8.0, 4e-6), "dlogits": (4.0, 1e-6), "dvalue": (4.0, 1e-6)}
SCALARS = ("loss", "policy", "entropy_loss", "value_loss") + tuple("entropy/" + k for k in HEADS) \
    + tuple("policy/" + k for k in HEADS) + ("adv_mean", "adv_std")
STATS = ("approx_kl",) + tuple("approx_kl/" + k for k in HEADS) + ("clip_fraction",) \
    + tuple("clip_fraction/" + k for k in HEADS) + ("explained_variance", "approx_kl/joint", "clip_fraction/joint")


# ------------------------------------------------------------------------------------------------ inputs
def make_inputs(n, seed, with_valid, device, value_clip=False):
    """Every row has a non-empty mask; about 10 % of them have a single entry.  Each head has an action on about 70 % of
    the tokens (enum on all).  Old log-probs make the log-ratio U(-3, 3) per head; tokens whose per-head or joint ratio
    lies within 2e-4 (in log) of a clip bound are moved off it, so that fp32 and float64 clip the same tokens."""
    g = torch.Generator(device=device).manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, device=device)         # noqa: E731
    scale = 60.0 ** rnd(n, 1)                                            # |logit| up to 60
    logits, masks, actions = [], [], []
    for h, m in enumerate(SIZES):
        mask = rnd(n, m) < 0.6
        act_idx = torch.randint(0, m, (n,), generator=g, device=device)
        mask[torch.arange(n, device=device), act_idx] = True
        single = rnd(n) < 0.1
        mask[single] = False
        mask[single, act_idx[single]] = True
        acted = rnd(n) < (1.0 if h == 0 else 0.7)
        act = torch.zeros(n, m, dtype=torch.bool, device=device)
        act[torch.arange(n, device=device), act_idx] = acted
        lg = (2 * rnd(n, m) - 1) * scale
        off = torch.where(rnd(n, m) < 0.5, -1e4, 1e4)
        logits.append(torch.where(mask, lg, off).float())
        masks.append(mask)
        actions.append(act)
    valid = (rnd(n) >= 0.1) if with_valid else None
    adv = (1e3 + torch.randn(n, generator=g, device=device)).float()
    ret = torch.randn(n, generator=g, device=device).float()
    values = (ret + 0.5 * torch.randn(n, generator=g, device=device)).float()
    old_values = (values + 0.1 * torch.randn(n, generator=g, device=device)).float() if value_clip else None
    with torch.no_grad():
        sel = torch.stack([(log_softmax(l.double(), m) * a).sum(1) for l, m, a in zip(logits, masks, actions)], 1)
    acted = torch.stack([a.any(1) for a in actions], 1)
    old = torch.where(acted, sel - (6 * rnd(n, 5) - 3).double(), torch.full_like(sel, 99.0)).float()
    bounds = torch.tensor([math.log(1 - E_CLIP), math.log(1 + E_CLIP)], dtype=torch.float64, device=device)
    for _ in range(3):
        lr = torch.where(acted, sel - old.double(), torch.zeros_like(sel))
        near = acted & ((lr[..., None] - bounds).abs() < 2e-4).any(-1)
        old = torch.where(near, old - 3e-3, old)
        joint = (sel - old.double()).where(acted, torch.zeros_like(sel)).sum(1)
        near_j = ((joint[:, None] - bounds).abs() < 2e-4).any(-1)
        old[:, 0] = torch.where(near_j, old[:, 0] - 3e-3, old[:, 0])
    return {"logits": logits, "masks": masks, "actions": actions, "old": old, "adv": adv, "ret": ret, "values": values,
            "old_values": old_values, "valid": valid}


def log_softmax(l, mask):
    """Masked log-softmax without max-subtraction (policy.py:169-178), exponentiating the mask's entries only."""
    e = torch.where(mask, l, torch.zeros_like(l)).exp() * mask
    return l - e.sum(1, keepdim=True).log()


# ------------------------------------------------------------------------------------------------ reference
def reference(inp, dtype, joint, entropy_coef=5e-4, vf_coef=0.5, value_clip=None):
    """-> dict of the loss slots and diagnostics (floats), ``dlogits`` (five [N, n_h]) and ``dvalue`` [N], in ``dtype``."""
    n = inp["adv"].shape[0]
    use = inp["valid"] if inp["valid"] is not None else torch.ones(n, dtype=torch.bool, device=inp["adv"].device)
    a = inp["adv"].to(dtype)
    # mean and std on the CPU, where the float64 mean of a constant is exact (the GPU reduction can be an ulp off, which
    # the division by std + eps = eps turns into a normalised advantage of 1e-9)
    au = a.cpu()[use.cpu()]
    adv = (a - float(au.sum() / au.numel())) / (float(au.std()) + EPS)
    lg = [l.to(dtype, copy=True).requires_grad_(True) for l in inp["logits"]]     # copies: the inputs stay leaves
    v = inp["values"].to(dtype, copy=True).requires_grad_(True)
    zero = torch.zeros([], dtype=dtype, device=a.device)
    out = {}
    pols, ents = [], []
    log_r_j = torch.zeros(n, dtype=dtype, device=a.device)
    has = torch.zeros(n, dtype=torch.bool, device=a.device)
    kls, clips = [], []
    for h, k in enumerate(HEADS):
        act = inp["actions"][h] & use[:, None]
        step = act.any(1)
        n_h = int(step.sum())
        out["n_actions/" + k] = n_h
        if n_h == 0:
            pols.append(zero)
            ents.append(zero)
            out["approx_kl/" + k] = out["clip_fraction/" + k] = 0.0
            continue
        mask = inp["masks"][h]
        e = torch.where(mask, lg[h], torch.zeros_like(lg[h])).exp() * mask
        se = e.sum(1, keepdim=True)
        lp = lg[h] - se.log()
        p = e / se
        ent_terms = torch.where(mask & use[:, None], p * lp, torch.zeros_like(lp))
        ents.append(-ent_terms.sum() / n_h)
        lr = (lp * act).sum(1) - inp["old"][:, h].to(dtype)
        lr_s = lr[step]
        r = lr_s.exp()
        s1, s2 = r * adv[step], r.clamp(1 - E_CLIP, 1 + E_CLIP) * adv[step]
        pols.append(-torch.min(s1, s2).sum() / n_h)
        with torch.no_grad():
            out["approx_kl/" + k] = float((torch.expm1(lr_s) - lr_s).mean())
            out["clip_fraction/" + k] = float(((r - 1).abs() > E_CLIP).to(dtype).mean())
        kls.append(out["approx_kl/" + k])
        clips.append(out["clip_fraction/" + k])
        log_r_j = log_r_j + torch.where(step, lr, torch.zeros_like(lr))
        has |= step
    if joint:
        t_a = int(has.sum())
        lr_s = log_r_j[has]
        r = lr_s.exp()
        s1, s2 = r * adv[has], r.clamp(1 - E_CLIP, 1 + E_CLIP) * adv[has]
        policy = -torch.min(s1, s2).sum() / t_a
        with torch.no_grad():
            out["approx_kl/joint"] = float((torch.expm1(lr_s) - lr_s).mean())
            out["clip_fraction/joint"] = float(((r - 1).abs() > E_CLIP).to(dtype).mean())
        pols_out = [0.0] * 5
    else:
        policy = torch.stack(pols).mean()
        pols_out = [float(x.detach()) for x in pols]
    e_loss = -entropy_coef * torch.stack(ents).sum()
    ret, vu = inp["ret"].to(dtype)[use], v[use]
    if value_clip:
        vo = inp["old_values"].to(dtype)[use]
        vc = vo + (vu - vo).clamp(-value_clip, value_clip)
        v_loss = vf_coef * (0.5 * torch.maximum((vu - ret).pow(2), (vc - ret).pow(2)).mean())
    else:
        v_loss = vf_coef * (0.5 * (ret - vu).pow(2).mean())
    loss = policy + e_loss + v_loss
    loss.backward()
    with torch.no_grad():
        d = ret - vu
        var_r = float(ret.var(unbiased=False))
        out["explained_variance"] = math.nan if var_r == 0.0 else 1.0 - float(d.var(unbiased=False)) / var_r
    out["approx_kl"] = sum(kls) / len(kls) if kls else 0.0
    out["clip_fraction"] = sum(clips) / len(clips) if clips else 0.0
    for name, x in zip(("loss", "policy", "entropy_loss", "value_loss"), (loss, policy, e_loss, v_loss)):
        out[name] = float(x.detach())
    for k, x, pl in zip(HEADS, ents, pols_out):
        out["entropy/" + k] = float(x.detach())
        out["policy/" + k] = pl
    out["adv_mean"], out["adv_std"] = float(a[use].mean()), float(a[use].std())
    out["dlogits"] = [x.grad if x.grad is not None else torch.zeros_like(x) for x in lg]
    out["dvalue"] = v.grad
    return out


# ------------------------------------------------------------------------------------------------ kernel
def packed_operands(inp, offset=False):
    """The packed [N, 128] GEMM output (four small heads and the value; junk in the other columns), the [N, 40]
    target-unit logits and the other operands; with ``offset`` every float operand is a view at a 1-float storage offset
    and every byte operand at a 1-byte offset."""
    n = inp["adv"].shape[0]
    d = inp["adv"].device

    def shifted(t):
        if not offset:
            return t.contiguous()
        buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=d)
        view = buf[1:].view(t.shape)
        view.copy_(t)
        return view
    packed = torch.full((n, 128), 3.0, device=d)
    for h, k in enumerate(HEADS):
        if k in PACK:
            packed[:, PACK[k][0]:PACK[k][1]] = inp["logits"][h]
    packed[:, VALUE_COL] = inp["values"]
    return {"packed": shifted(packed), "tu": shifted(inp["logits"][3]), "masks": [shifted(m) for m in inp["masks"]],
            "actions": [shifted(a) for a in inp["actions"]], "old": shifted(inp["old"]), "adv": shifted(inp["adv"]),
            "ret": shifted(inp["ret"]),
            "old_values": None if inp["old_values"] is None else shifted(inp["old_values"]),
            "valid": None if inp["valid"] is None else shifted(inp["valid"])}


def run_kernel(inp, joint, entropy_coef=5e-4, vf_coef=0.5, value_clip=None, offset=False):
    from dotaclient_b200 import ops
    o = packed_operands(inp, offset)
    hp = ops.hparam_block(o["adv"].device, e_clip=E_CLIP, entropy_coef=entropy_coef, vf_coef=vf_coef,
                          value_clip=value_clip)
    out, n_act, d_packed, d_tu, stats = ops.ppo_loss_packed(
        o["packed"], o["tu"], o["masks"], o["actions"], o["old"], o["adv"], o["ret"], None, None, None, hparams=hp,
        old_value=o["old_values"], valid=o["valid"], joint=joint)
    torch.cuda.synchronize()
    return out, n_act, d_packed, d_tu, stats


def kernel_results(res):
    out, n_act, d_packed, d_tu, stats = res
    o, s = out.cpu().tolist(), stats.cpu().tolist()
    r = dict(zip(SCALARS, o))
    r.update(zip(STATS, s[0:6] + s[6:12] + s[12:15]))
    r["dlogits"] = [d_packed[:, PACK[k][0]:PACK[k][1]] if k in PACK else d_tu for k in HEADS]
    r["dvalue"] = d_packed[:, VALUE_COL]
    r["n_actions"] = n_act.cpu().tolist()
    r["pad_cols"] = d_packed[:, 26:]
    return r


def bound(kind, got, ref, cal, ratios, failures, name):
    k, floor = BOUNDS[kind]
    got, ref, cal = (torch.as_tensor(x, dtype=torch.float64) for x in (got, ref, cal))
    err = float((got - ref).abs().max())
    c = float((cal - ref).abs().max())
    scale = float(ref.abs().max())
    r = err / c if c > 0 else (0.0 if err == 0 else float("inf"))
    ratios[kind] = max(ratios.get(kind, 0.0), r)
    ratios["rel " + kind] = max(ratios.get("rel " + kind, 0.0), err / max(scale, 1e-30))
    if not err <= k * c + floor * scale:
        failures.append("%s: max|err| %.3e, torch fp32 %.3e, max|f64| %.3e" % (name, err, c, scale))


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("joint", [False, True], ids=["per_head", "joint"])
@pytest.mark.parametrize("with_valid", [False, True], ids=["all", "valid"])
@pytest.mark.parametrize("value_clip", [None, 0.05])
def test_reference_matches_the_oracles(joint, with_valid, value_clip):
    """In float64 on ordinary inputs (logits N(0, 1) on the mask and 0 off it), ``reference`` equals
    ``padding_oracle.masked_ppo_loss`` / ``joint_ratio_oracle.joint_ppo_loss`` and their diagnostics, gradients too."""
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import joint_ratio_oracle as JO
    import padding_oracle as PO
    n = 700
    inp = make_inputs(n, 3, with_valid, torch.device("cpu"), value_clip=bool(value_clip))
    g = torch.Generator().manual_seed(4)
    inp["logits"] = [torch.where(m, torch.randn(l.shape, generator=g), torch.zeros_like(l))
                     for l, m in zip(inp["logits"], inp["masks"])]
    sel = torch.stack([(log_softmax(l.double(), m) * a).sum(1) for l, m, a in zip(inp["logits"], inp["masks"],
                                                                                     inp["actions"])], 1)
    acted = torch.stack([a.any(1) for a in inp["actions"]], 1)
    inp["old"] = torch.where(acted, sel - 2 * torch.rand(n, 5, generator=g, dtype=torch.float64) + 1,
                             torch.zeros_like(sel)).float()
    got = reference(inp, torch.float64, joint, value_clip=value_clip)
    use = inp["valid"] if with_valid else torch.ones(n, dtype=torch.bool)
    lg = {k: l.double().requires_grad_(True) for k, l in zip(HEADS, inp["logits"])}
    vg = inp["values"].double().requires_grad_(True)
    acts = dict(zip(HEADS, inp["actions"]))
    msks = dict(zip(HEADS, inp["masks"]))
    ov = None if value_clip is None else inp["old_values"].double()
    args = (lg, vg, acts, msks, inp["old"].double(), inp["adv"].double(), inp["ret"].double())
    if joint:
        want = JO.joint_ppo_loss(*args, 5e-4, 0.5, E_CLIP, valid=use, old_values=ov, value_clip=value_clip)
        st = JO.joint_stats(dict(zip(HEADS, inp["logits"])), acts, msks, inp["old"], E_CLIP, use)
        assert got["approx_kl/joint"] == pytest.approx(st["approx_kl/joint"], rel=1e-6, abs=1e-9)
        assert got["clip_fraction/joint"] == pytest.approx(st["clip_fraction/joint"], rel=1e-9, abs=1e-12)
    else:
        want = PO.masked_ppo_loss(*args[:4], args[4], args[5], args[6], use, 5e-4, 0.5, E_CLIP, old_values=ov,
                                  value_clip=value_clip)
    want[0].backward()
    for name, w in zip(("loss", "policy", "entropy_loss", "value_loss"), want[:4]):
        assert got[name] == pytest.approx(float(w.detach()), rel=1e-9, abs=1e-12), name
    for k in HEADS:
        assert got["entropy/" + k] == pytest.approx(float(want[4][k].detach()), rel=1e-9, abs=1e-12), k
        g_ref = lg[k].grad if lg[k].grad is not None else torch.zeros_like(lg[k])
        torch.testing.assert_close(got["dlogits"][HEADS.index(k)], g_ref, rtol=1e-9, atol=1e-12)
    torch.testing.assert_close(got["dvalue"], vg.grad, rtol=1e-9, atol=1e-12)
    stats = PO.masked_stats(dict(zip(HEADS, inp["logits"])), acts, msks, inp["old"], inp["values"], inp["ret"], use,
                            E_CLIP)
    for k, w in stats.items():
        assert got[k] == pytest.approx(w, rel=1e-5, abs=1e-9), k       # the oracle's log-probs are fp32


# ------------------------------------------------------------------------------------------------ GPU
CASES = [(n, joint, valid, None) for n in (16384, 131072, 131035, 262144, 524288) for joint in (False, True)
         for valid in (False, True)] + [(131035, False, True, 0.05), (262144, True, False, 0.05)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,joint,with_valid,value_clip", CASES,
                         ids=["%d-%s-%s%s" % (n, "joint" if j else "per_head", "valid" if v else "all",
                                              "-vclip" if c else "") for n, j, v, c in CASES])
def test_ppo_loss_hard_inputs_vs_fp64(n, joint, with_valid, value_clip):
    """Loss slots, entropies, per-head policies, advantage mean / std, diagnostics, dlogits and dvalue within the bound;
    n_actions exact; dlogits exactly 0 off the mask, on padded tokens and in the packed gradient's unused columns."""
    d = torch.device("cuda", 0)
    inp = make_inputs(n, n + 17 * joint + 5 * with_valid, with_valid, d, value_clip=bool(value_clip))
    f64 = reference(inp, torch.float64, joint, value_clip=value_clip)
    f32 = reference(inp, torch.float32, joint, value_clip=value_clip)
    got = kernel_results(run_kernel(inp, joint, value_clip=value_clip))
    use = inp["valid"] if with_valid else torch.ones(n, dtype=torch.bool, device=d)
    # the four clip cases of the per-head ratio (enum: an action on every token)
    lr = ((log_softmax(inp["logits"][0].double(), inp["masks"][0]) * inp["actions"][0]).sum(1)
          - inp["old"][:, 0].double())[use]
    a = inp["adv"].double()[use]
    a = a - a.mean()
    for side in (lr > math.log(1 + E_CLIP), lr < math.log(1 - E_CLIP)):
        assert bool((side & (a > 0)).any()) and bool((side & (a < 0)).any())
    failures, ratios = [], {}
    assert got["n_actions"] == [f64["n_actions/" + k] for k in HEADS]
    names = SCALARS + STATS if joint else SCALARS + STATS[:-2]
    for name in names:
        bound("scalar", got[name], f64[name], f32[name], ratios, failures, name)
    for h, k in enumerate(HEADS):
        g = got["dlogits"][h]
        bound("dlogits", g.cpu(), f64["dlogits"][h].cpu(), f32["dlogits"][h].cpu(), ratios, failures, "dlogits/" + k)
        if bool((g[~inp["masks"][h]] != 0).any()):
            failures.append("dlogits/%s: non-zero off the mask" % k)
        if with_valid and bool((g[~use] != 0).any()):
            failures.append("dlogits/%s: non-zero on a padded token" % k)
    bound("dvalue", got["dvalue"].cpu(), f64["dvalue"].cpu(), f32["dvalue"].cpu(), ratios, failures, "dvalue")
    if bool((got["pad_cols"] != 0).any()):
        failures.append("the packed gradient's unused columns are not zero")
    print("\n%d %s %s ratios: %s" % (n, "joint" if joint else "per_head", "valid" if with_valid else "all",
                                     ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert not failures, failures


@pytest.mark.gpu
@pytest.mark.parametrize("n", [16384, 131072, 524288])
@pytest.mark.parametrize("with_valid", [False, True], ids=["all", "valid"])
def test_explained_variance_of_constant_returns_is_nan(n, with_valid):
    """Var(ret) = 0 -> NaN, for constants whose one-pass sums round to a positive variance (0.7, 1.1) and to a
    non-positive one (-2.37); padded tokens carry a return of 0, as prep leaves them, and the first token is padding."""
    d = torch.device("cuda", 0)
    inp = make_inputs(n, 11, with_valid, d)
    if with_valid:
        inp["valid"][0] = False
    for c in (0.7, 1.1, -2.37):
        inp["ret"] = torch.full((n,), c, device=d)
        if with_valid:
            inp["ret"][~inp["valid"]] = 0.0
        got = kernel_results(run_kernel(inp, False))
        assert math.isnan(got["explained_variance"]), (c, got["explained_variance"])
        assert math.isnan(reference(inp, torch.float64, False)["explained_variance"])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [16384, 524288])
@pytest.mark.parametrize("with_valid", [False, True], ids=["all", "valid"])
def test_explained_variance_of_near_constant_returns(n, with_valid):
    """ret = c + 1e-3 noise: the explained variance within the bound of the two-pass float64 value."""
    d = torch.device("cuda", 0)
    inp = make_inputs(n, 12, with_valid, d)
    g = torch.Generator(device=d).manual_seed(n)
    for c in (0.7, -2.37, 300.0):
        inp["ret"] = (c + 1e-3 * torch.randn(n, generator=g, device=d)).float()
        inp["values"] = (inp["ret"] + 5e-4 * torch.randn(n, generator=g, device=d)).float()
        got = kernel_results(run_kernel(inp, False))
        f64, f32 = reference(inp, torch.float64, False), reference(inp, torch.float32, False)
        failures, ratios = [], {}
        bound("scalar", got["explained_variance"], f64["explained_variance"], f32["explained_variance"], ratios,
              failures, "explained_variance c=%g" % c)
        print("\nnear-constant %g: kernel %.9g, f64 %.9g, torch32 %.9g" % (c, got["explained_variance"],
                                                                          f64["explained_variance"],
                                                                          f32["explained_variance"]))
        assert not failures, failures


@pytest.mark.gpu
@pytest.mark.parametrize("joint", [False, True], ids=["per_head", "joint"])
def test_constant_advantages_normalise_to_zero(joint):
    """Constant advantages: the normalised advantage is exactly 0 (as in float64), so the policy loss and, without an
    entropy term, every dlogits entry are exactly 0."""
    d = torch.device("cuda", 0)
    n = 131072
    inp = make_inputs(n, 13, True, d)
    inp["adv"] = torch.full((n,), 1.7, device=d)
    f64 = reference(inp, torch.float64, joint, entropy_coef=0.0)
    assert f64["policy"] == 0.0
    got = kernel_results(run_kernel(inp, joint, entropy_coef=0.0))
    assert got["policy"] == 0.0 and all(got["policy/" + k] == 0.0 for k in HEADS)
    assert got["adv_mean"] == pytest.approx(1.7, rel=1e-7)
    assert all(bool((g == 0).all()) for g in got["dlogits"])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["per_head", "masked", "joint"])
def test_unaligned_operands_are_bitwise_equal(mode):
    """Logits, old log-probs, advantages, returns, values (and old values) at a 1-float storage offset, masks, actions and
    valid at a 1-byte offset: the unaligned staging paths give the aligned call's results bit for bit."""
    d = torch.device("cuda", 0)
    n = 131035
    inp = make_inputs(n, 14, mode == "masked", d, value_clip=True)
    o = packed_operands(inp, offset=True)
    assert o["tu"].data_ptr() % 16 == 4 and o["old"].data_ptr() % 16 == 4 and o["masks"][0].data_ptr() % 16 == 1
    a = run_kernel(inp, mode == "joint", value_clip=0.05)
    b = run_kernel(inp, mode == "joint", value_clip=0.05, offset=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
