"""One whole ``DotaOptimizer.train`` step under KL control, kickstarting, behaviour cloning, value heads and PopArt, at the
benchmark's shapes, against a float64 reference: encoder, recurrence, packed heads, the compact target-unit branch (every
case has at least 4,096 tokens), the loss instantiation of the option (``kKl``, ``kTeacher`` with and without ``kKl``
and in both ratio modes, ``kBc``, ``dc_value_heads_loss``, the normalised value term), backward and gradient finish.

The method is ``test_gpu_step_fp64``'s, whose machinery this file imports: the full ``[S, B]`` batch with ``valid = False``
outside a sample R of columns, the grid encoder, the pre-RNN ReLU off its kink, old log-probabilities and old values
fitted off the clip bounds, and ``StackedRefPolicy`` in float64 on R.  The loss is ``objectives_reference.reference``:
``test_gpu_ppo_fp64.reference`` plus the option's terms, written for any dtype, so that the same reference in fp32
calibrates the bound every output meets, with ``test_gpu_step_fp64.BOUNDS`` unchanged:

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

Per option, the inputs the step reads beyond the default batch:
  KL control / teacher  ``old_log_probs`` / ``teacher_log_probs`` [S, B, 65]: on R the masked log-softmax of the float64
                        logits plus N(0, 0.25^2) / N(0, 1) noise (``kl_oracle.masked_log_rows``), 0 elsewhere.  The step
                        reads only the teacher's rows, so the teacher model is the reference's GRU-256 initialisation.
  value heads           ``returns`` / ``old_values`` [S, B, K]; the clipped value loss of every head fitted off its tie.
                        The reference policy has a K-row value layer, and its forward keeps every value column.
  PopArt                ``opt._value_norm`` preset to mu = -1.3, sigma = 3.7; raw returns mu + sigma N(0, 1), fitted in
                        normalised units; the reference reads fp32((R - mu) / sigma) as the kernel does.
  behaviour cloning     the advantages are not read.  ``bc/accuracy*`` are arg-max decisions: they must equal the float64
                        ones up to one flipped decision per row (token) whose top two masked logits lie within 1e-4
                        (counted per head and for the token accuracy, reported).
Every value the step reports for the option is compared ('scalar': losses, entropies, norms, KL, teacher KL, NLL, the
heads' value losses; 'diagnostic': approximate KL, clip fractions, explained variances), ``kl_skipped`` must be 0, and a
reported name the test does not know fails it.

``test_reference_and_bound_on_the_cpu`` shows without a GPU, per option at B 12 x S 16 x H 32, that the reference on R
equals, to 1e-10 in float64, a transcription over the whole masked batch through the feature suites' own oracles
(``kl_oracle.kl_ppo_loss``, ``teacher_oracle.teacher_ppo_loss``, ``bc_oracle.bc_loss``,
``value_heads_oracle.value_heads_loss``, ``value_norm_oracle.normalise`` with ``padding_oracle.masked_ppo_loss``)
differentiated through the network, that the fp32 transcription passes the bound and that every mutant fails it.

Measured on one H100 80GB HBM3 (700 W power limit): the largest ratio max|gpu - f64| / max|torch32 - f64| per kind
(scalar / diagnostic / weight / recurrent), the largest max|gpu - f64| / max|f64| of the weight and recurrent gradients
in brackets, the largest share of its bound any output uses, and the wall time of the case (reference included):
    c2-kl                    24 /  83 /   57 /  34  (1.6e-5, 1.2e-5)  0.55   3 s
    c2-joint-kl-teacher    1320 / 7.9 /   69 /  26  (3.6e-5, 1.1e-5)  0.66   2 s   (graph)
    c3-teacher (clip on)     18 /  13 /  8.2 / 2.3  (3.9e-5, 1.1e-5)  0.77   3 s
    c2-bc                   7.3 / 0.06 /  93 /  45  (7.1e-6, 8.3e-6)  0.38   3 s   (graph; 38 near-tie tokens)
    c5-bc                   5.7 / 0.73 /  44 /  25  (4.9e-5, 9.7e-6)  0.63   1 s   (1 near-tie token)
    c2-heads3               5.1 / 272 /   86 /  19  (1.0e-5, 9.0e-6)  0.41   2 s
    c3-heads10              3.2 /  23 /  131 /  44  (1.4e-5, 1.2e-5)  0.27   3 s
    c2-popart               6.7 / 7.2 /   69 /  24  (7.7e-6, 7.8e-6)  0.44   3 s   (graph)
    c2-packed-kl-teacher     83 /  54 /   68 /  52  (5.3e-5, 1.7e-5)  0.94   5 s
The KL is about 0.05 and the teacher KL about 0.62 in every case that has them.  Where torch fp32 is nearly exact on a
scalar (1320 at c2-joint-kl-teacher) the floor carries the bound.  The graph replays are bitwise equal to the eager step.

Mutants (``test_objective_mutants_fail_the_bound``), all failing the bound: the largest share of its bound an output uses,
the largest max|gpu - f64| / max|f64| of a weight gradient, the first outputs over it, and whether the per-tensor
gradient criterion of the fp32-oracle tests (cosine > 0.9999, norm within 2e-3) catches them:
    kl_swap (c2-kl)                  96x    5e-3   norms, kl/enum, encoder         NOT caught
    teacher_coef (joint-kl-teacher)  2487x  1.5e-2 loss, norms, loss/teacher       caught
    bc_scale (c2-bc, dlogits x T_a/(T_a+1)) 20x    2e-4   norms, encoder                  NOT caught
    heads_swap (c2-heads3)           11563x 1.9e-2 loss, value_loss, norms         caught
    sigma (c2-popart)                4695x  2.5e-2 loss, value_loss, norms         caught
The whole file runs in 60 to 75 s on the H100.
"""
import math
import time

import pytest
import torch
import torch.nn as nn

import bc_oracle as BO
import joint_ratio_oracle as JO
import kl_oracle as KO
import objectives_reference as OR
import padding_oracle as PO
import teacher_oracle as TO
import test_gpu_step_fp64 as ST
import value_heads_oracle as VH
import value_norm_oracle as VN
from dotaclient_b200.policy import REWARD_KEYS
from stacked_oracle import StackedRefPolicy
from test_gpu_value_heads import GAMMAS3, THREE

HEADS = ST.HEADS
E_CLIP = ST.E_CLIP
BOUNDS = ST.BOUNDS
BETA, LAMBDA = 0.7, 1.3
NORM_STATE = (-1.3, 3.7 ** 2 + 1.3 ** 2, 1.0)      # (m, q, w): mu = -1.3, sigma = 3.7
OLD_SCALE, TEACHER_SCALE = 0.25, 1.0               # the noise on the float64 logits that makes the prep-time / teacher rows


class Case(ST.Case):
    def __init__(self, name, cell, B, S, H, rows, beta=0.0, lam=0.0, bc=False, heads=None, gammas=None, norm=False,
                 value_clip=False, **kw):
        super().__init__(name, cell, B, S, H, rows, **kw)
        self.value_clip = ST.VALUE_CLIP if value_clip else None
        self.beta, self.lam, self.bc, self.heads, self.gammas, self.norm = beta, lam, bc, heads, gammas, norm
        self.K = len(heads) if heads else 1
        self.head_names = list(heads) if heads else None


C2, C3 = ST.C2_ROWS, ST.C3_ROWS
C5 = (0, 31, 32, 511, 512, 991, 992, 1023)
CASES = [
    Case("c2-kl", "lstm", 256, 512, 128, C2, beta=1.0),
    Case("c2-joint-kl-teacher", "lstm", 256, 512, 128, C2, joint=True, beta=BETA, lam=LAMBDA, value_clip=True, graph=True),
    Case("c3-teacher", "lstm", 512, 512, 256, C3, lam=LAMBDA, clip=True),
    Case("c2-bc", "lstm", 256, 512, 128, C2, bc=True, value_clip=True, graph=True),
    Case("c5-bc", "gru", 1024, 16, 256, C5, bc=True),
    Case("c2-heads3", "lstm", 256, 512, 128, C2, heads=THREE, gammas=GAMMAS3, value_clip=True),
    Case("c3-heads10", "lstm", 512, 512, 256, C3, heads={k: [k] for k in REWARD_KEYS}),
    Case("c2-popart", "lstm", 256, 512, 128, C2, norm=True, value_clip=True, graph=True),
    Case("c2-packed-kl-teacher", "lstm", 256, 512, 128, C2, packed=True, beta=BETA, lam=LAMBDA),
]
CASE = {c.name: c for c in CASES}


def norm_of(case):
    return VN.moments(NORM_STATE) if case.norm else None


# ------------------------------------------------------------------------------------------------ reference
class HeadsRefPolicy(StackedRefPolicy):
    """``StackedRefPolicy`` with a K-row value layer; its forward returns the values as [..., K, 1], so that
    ``test_gpu_step_fp64.ref_forward`` (which takes value column 0) keeps all K columns."""

    def __init__(self, H, cell, layers, K):
        super().__init__(H, cell, layers)
        self.affine_value = nn.Linear(H, K)

    def forward(self, *a, **kw):
        logits, value, hidden = super().forward(*a, **kw)
        return logits, value.unsqueeze(-1), hidden


def ref_policy(state_dict, case, dtype):
    if case.K == 1:
        return ST.ref_policy(state_dict, case, dtype)
    pol = HeadsRefPolicy(case.H, case.cell, case.layers, case.K)
    pol.load_state_dict({k: v.detach().cpu() for k, v in state_dict.items()})
    return pol.to(dtype)


class PreRnnView:
    """What ``test_gpu_step_fp64.clear_relu_ties`` reads of a policy: its state with the value layer cut to one row (the
    pre-RNN ReLU does not depend on it) and its pre-RNN layer, whose bias it shifts."""

    def __init__(self, pol):
        self._pol, self.affine_pre_rnn = pol, pol.affine_pre_rnn

    def state_dict(self):
        sd = dict(self._pol.state_dict())
        sd["affine_value.weight"], sd["affine_value.bias"] = sd["affine_value.weight"][:1], sd["affine_value.bias"][:1]
        return sd


def perturbed_rows(logits, masks, seed, scale):
    """[N, 65] fp32: the masked log-softmax rows of ``logits`` (float64) plus N(0, scale^2) noise, 0 at illegal entries."""
    g = torch.Generator().manual_seed(seed)
    moved = {k: v.double() + scale * torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in logits.items()}
    return KO.masked_log_rows(moved, masks).float()


def fit_rows(r, logits, case, seed):
    """The prep-time and teacher rows of R from the float64 forward (``logits`` {head: [S, R, n]})."""
    S, R = r["valid"].shape
    lg = {k: logits[k].reshape(S * R, -1) for k in HEADS}
    msk = {k: r["masks"][k].reshape(S * R, -1) for k in HEADS}
    if case.beta:
        r["old_log_probs"] = perturbed_rows(lg, msk, seed, OLD_SCALE).view(S, R, OR.ROW)
    if case.lam:
        r["teacher_log_probs"] = perturbed_rows(lg, msk, seed + 1, TEACHER_SCALE).view(S, R, OR.ROW)


def fit_values(r, values, case, seed):
    """Under value clipping, the old values (|v - v_old| in 0..2 clip, off the clip bound) and returns (off the tie of the
    clipped loss's two squares) of every head, as ``test_gpu_step_fp64.fit_to_reference`` does for one; PopArt: in
    normalised units, stored raw."""
    if not case.value_clip:
        return
    vc, norm = case.value_clip, norm_of(case)
    g = torch.Generator().manual_seed(seed)
    shape = r["returns"].shape
    v = values.reshape(-1, case.K)
    dv = (torch.rand(v.shape, generator=g, dtype=torch.float64) * 4 - 2) * vc
    dv = torch.where((dv.abs() - vc).abs() < 2e-3, dv + 5e-3 * dv.sign(), dv)
    vo = (v - dv).float().double()
    ret = r["returns"].reshape(-1, case.K).double()
    if norm:
        ret = (ret - norm[0]) / norm[1]
    vcl = vo + (v - vo).clamp(-vc, vc)
    ret = torch.where((2 * ret - v - vcl).abs() < 2e-3, ret + 0.01, ret)
    if norm:
        ret, vo = norm[0] + norm[1] * ret, norm[0] + norm[1] * vo
    r["returns"], r["old_values"] = ret.float().view(shape), vo.float().view(shape)


def ref_step(pol, r, case, dtype, fwd=None):
    """The loss of sample ``r`` under ``pol`` in ``dtype`` (``objectives_reference.reference``), its backward and the
    global-norm clip -> (scalars, clipped gradients)."""
    pol.zero_grad(set_to_none=True)
    logits, values = fwd if fwd is not None else ST.ref_forward(pol, r, dtype)
    S, R = values.shape[:2]
    n = S * R
    vs = (n, case.K) if case.K > 1 else (n,)
    lgs, msks = [], []
    for k in HEADS:
        m = r["masks"][k].reshape(n, -1)
        empty = ~m.any(1, keepdim=True)
        lgs.append(torch.where(empty, 0.0, logits[k].detach().reshape(n, -1)))
        msks.append(m | (empty & (torch.arange(m.shape[1]) == 0)))
    inp = {"logits": lgs, "masks": msks, "actions": [r["actions"][k].reshape(n, -1) for k in HEADS],
           "old": r["old_logp"].reshape(n, 5), "adv": r["advantages"].reshape(n), "ret": r["returns"].reshape(vs),
           "values": values.detach().reshape(vs), "old_values": r["old_values"].reshape(vs), "valid": r["valid"].reshape(n)}
    out = OR.reference(inp, dtype, case.joint, value_clip=case.value_clip,
                       old_rows=r["old_log_probs"].reshape(n, OR.ROW) if case.beta else None, beta=case.beta,
                       teacher_rows=r["teacher_log_probs"].reshape(n, OR.ROW) if case.lam else None, lam=case.lam,
                       bc=case.bc, head_names=case.head_names, norm=norm_of(case))
    torch.autograd.backward([logits[k] for k in HEADS] + [values],
                            [d.view_as(logits[k]) for d, k in zip(out["dlogits"], HEADS)] + [out["dvalue"].view_as(values)])
    return ST.finish(pol, out, case.max_grad_norm)


# ------------------------------------------------------------------------------------------------ comparison
ACCURACY = ["bc/accuracy"] + ["bc/accuracy/" + k for k in HEADS]


def names(case):
    """-> (scalar names, diagnostic names) the step reports for ``case``."""
    scal = ["loss", "policy", "entropy_loss", "value_loss", "unclipped", "clipped"] + ["entropy/" + k for k in HEADS]
    diag = ["explained_variance"]
    if not case.bc:
        diag += ["approx_kl", "clip_fraction"] + ["approx_kl/" + k for k in HEADS] + ["clip_fraction/" + k for k in HEADS]
        diag += ["approx_kl/joint", "clip_fraction/joint"] if case.joint else []
    if case.beta:
        scal += ["kl", "kl_penalty", "kl_all_ranks"] + ["kl/" + k for k in HEADS]
    if case.lam:
        scal += ["teacher/kl", "loss/teacher"] + ["teacher/kl/" + k for k in HEADS]
    if case.bc:
        scal += ["bc/nll/" + k for k in HEADS]
    if case.heads:
        scal += ["loss/value/" + h for h in case.head_names]
        diag += ["explained_variance/" + h for h in case.head_names]
    return scal, diag


def compare(got, f64, f32, case):
    """``test_gpu_step_fp64.compare`` over the names of ``case``; behaviour cloning's accuracies against float64's arg-max
    decisions, up to one flipped decision per near-tie row; ``kl_skipped`` 0."""
    ratios, over = ST.compare_names(got, f64, f32, *names(case))
    if case.bc:     # the number of right decisions; each near-tie row (token) may flip one
        for n in ACCURACY:
            near, cnt = f64[0]["near_ties/" + n], f64[0]["rows/" + n]
            if abs(round(got[0][n] * cnt) - round(f64[0][n] * cnt)) > near:
                over.append("%s: %r, float64 %r, %d near-tie rows of %d" % (n, got[0][n], f64[0][n], near, cnt))
    if case.beta:
        if got[0].get("kl_skipped", 0.0) != 0.0:
            over.append("kl_skipped")
    return ratios, over


def unchecked(got, case):
    """The names the step reported that ``compare`` does not check for ``case``."""
    scal, diag = names(case)
    known = set(scal) | set(diag) | (set(ACCURACY) if case.bc else set()) | ({"kl_skipped"} if case.beta else set())
    return sorted(set(got[0]) - known)


# ------------------------------------------------------------------------------------------------ CPU: reference and bound
def transcription_step(pol, f, case, mutant=None):
    """An independent transcription of the step over the WHOLE masked batch through the feature suites' oracles,
    differentiated through the network, then the clip.  ``mutant``: 'kl_swap' swaps the enum rows of old_log_probs of
    two adjacent tokens of R's third column, 'teacher_coef' runs lambda as 0.99 lambda, 'bc_scale' scales the logits'
    gradient (the NLL's and the entropy term's) by T_a / (T_a + 1), 'heads_swap' swaps the returns of heads 0 and 1 on the first 2 tokens of R's third column,
    'sigma' normalises with 1.01 sigma."""
    S, B = f["valid"].shape
    n = S * B
    f = dict(f)
    b, lam, norm = case.rows[2], case.lam, norm_of(case)
    if mutant == "kl_swap":
        t = f["old_log_probs"].clone()
        t[[5, 6], b, 0:4] = t[[6, 5], b, 0:4]
        f["old_log_probs"] = t
    elif mutant == "teacher_coef":
        lam = 0.99 * lam
    elif mutant == "heads_swap":
        t = f["returns"].clone()
        t[0:2, b, 0], t[0:2, b, 1] = f["returns"][0:2, b, 1], f["returns"][0:2, b, 0]
        f["returns"] = t
    elif mutant == "sigma":
        norm = (norm[0], 1.01 * norm[1])
    dtype = next(pol.parameters()).dtype
    pol.zero_grad(set_to_none=True)
    logits, values = ST.ref_forward(pol, dict(f, reset_slot=None), dtype)
    lg = {k: logits[k].reshape(n, -1) for k in HEADS}
    act = {k: f["actions"][k].reshape(n, -1) for k in HEADS}
    msk = {k: f["masks"][k].reshape(n, -1) for k in HEADS}
    valid = f["valid"].reshape(n)
    vs = (n, case.K) if case.K > 1 else (n,)
    v, ret, ov = values.reshape(vs), f["returns"].reshape(vs), f["old_values"].reshape(vs)
    old, adv, vc = f["old_logp"].reshape(n, 5), f["advantages"].reshape(n), case.value_clip
    rows = f["old_log_probs"].reshape(n, OR.ROW).double() if case.beta else None
    t_rows = f["teacher_log_probs"].reshape(n, OR.ROW).double() if case.lam else None
    if norm:
        ret = torch.from_numpy(VN.normalise(ret.numpy(), *norm)).to(dtype)
        ov = torch.from_numpy(VN.normalise(ov.numpy(), *norm)).to(dtype)
    out = {}
    if case.bc:
        loss, p_loss, e_loss, v_loss, ents = BO.bc_loss(lg, v, act, msk, ret, 5e-4, 0.5, valid, ov, vc)
        _, t_a, sums, counts = BO.nll(lg, act, msk, valid)
        if mutant == "bc_scale":       # the policy heads' logit gradients (NLL and entropy terms) times T_a / (T_a + 1)
            for x in lg.values():
                x.register_hook(lambda g: g * (t_a / (t_a + 1.0)))
        out.update({"bc/nll/" + k: sums[k] / counts[k] if counts[k] else 0.0 for k in HEADS})
        acc, per = BO.accuracy(lg, act, msk, valid)
        out["bc/accuracy"] = acc
        out.update({"bc/accuracy/" + k: a for k, a in per.items()})
    elif case.lam:
        loss, p_loss, e_loss, v_loss, ents, kl_t = TO.teacher_ppo_loss(
            lg, v, act, msk, old, rows, t_rows, adv, ret, 5e-4, 0.5, E_CLIP, case.beta, lam, joint=case.joint,
            valid=valid, old_values=ov, value_clip=vc)
        _, _, _, per = TO.teacher_kl(lg, act, msk, t_rows, valid)
        out.update({"teacher/kl": float(kl_t), "loss/teacher": lam * float(kl_t)})
        out.update({"teacher/kl/" + k: x for k, x in per.items()})
    elif case.beta:
        loss, p_loss, e_loss, v_loss, ents, _ = KO.kl_ppo_loss(lg, v, act, msk, old, rows, adv, ret, 5e-4, 0.5, E_CLIP,
                                                               case.beta, joint=case.joint, valid=valid, old_values=ov,
                                                               value_clip=vc)
    elif case.heads:
        loss, p_loss, e_loss, _, ents = PO.masked_ppo_loss(lg, v[:, 0], act, msk, old, adv, ret[:, 0], valid, 5e-4, 0.0,
                                                           E_CLIP)
        tot, dv, per, ev, ev_tot = VH.value_heads_loss(v.detach().double().numpy(), ret.double().numpy(), 0.5,
                                                       ov.double().numpy(), vc or 0.0, valid.numpy())
        loss = loss + (v * torch.from_numpy(dv).to(v.dtype)).sum()
        v_loss = torch.tensor(float(tot), dtype=torch.float64)
        out.update({"loss/value/" + h: float(per[k]) for k, h in enumerate(case.head_names)})
        out.update({"explained_variance/" + h: float(ev[k]) for k, h in enumerate(case.head_names)})
    else:
        loss, p_loss, e_loss, v_loss, ents = PO.masked_ppo_loss(lg, v, act, msk, old, adv, ret, valid, 5e-4, 0.5, E_CLIP,
                                                                old_values=ov, value_clip=vc)
    loss.backward()
    if case.beta:
        kl, _, _, per = KO.exact_kl({k: x.detach() for k, x in lg.items()}, act, msk, rows, valid)
        out.update({"kl": float(kl), "kl_all_ranks": float(kl), "kl_penalty": case.beta * float(kl)})
        out.update({"kl/" + k: x for k, x in per.items()})
    with torch.no_grad():
        st = PO.masked_stats(lg, act, msk, old, v[:, 0] if case.heads else v, ret[:, 0] if case.heads else ret, valid,
                             E_CLIP)
        if case.joint:
            st.update(JO.joint_stats(lg, act, msk, old, E_CLIP, valid))
    out = dict(st, **out)
    if case.heads:
        out["explained_variance"] = float(ev_tot)
    total = float(loss.detach()) - (float((v.detach() * torch.from_numpy(dv).to(v.dtype)).sum()) - float(v_loss)
                                    if case.heads else 0.0)
    out.update(loss=total, policy=float(p_loss.detach()), entropy_loss=float(e_loss.detach()),
               value_loss=float(v_loss.detach()))
    out.update({"entropy/" + k: float(x.detach()) for k, x in ents.items()})
    return ST.finish(pol, out, case.max_grad_norm)


CPU_ROWS = (0, 3, 4, 5, 6, 11)
CPU_CASES = [Case("cpu-kl", "lstm", 12, 16, 32, CPU_ROWS, beta=1.0),
             Case("cpu-kl-teacher", "lstm", 12, 16, 32, CPU_ROWS, beta=BETA, lam=LAMBDA, value_clip=True),
             Case("cpu-bc", "lstm", 12, 16, 32, CPU_ROWS, bc=True, value_clip=True),
             Case("cpu-heads3", "lstm", 12, 16, 32, CPU_ROWS, heads=THREE, value_clip=True),
             Case("cpu-popart", "lstm", 12, 16, 32, CPU_ROWS, norm=True, value_clip=True)]
CPU_MUTANTS = {"cpu-kl": ("kl_swap",), "cpu-kl-teacher": ("teacher_coef",), "cpu-bc": ("bc_scale",),
               "cpu-heads3": ("heads_swap",), "cpu-popart": ("sigma",)}


def extend_batch(f, case, seed):
    """The fields ``test_gpu_step_fp64.make_batch`` leaves out: K-column returns and old values, PopArt's raw returns
    and old values (mu + sigma N(0, 1)), and zero prep-time / teacher rows (R's are set by ``fit_rows``)."""
    S, B = f["valid"].shape
    d = f["valid"].device
    g = torch.Generator(device=d).manual_seed(seed)
    if case.K > 1:
        f["returns"] = torch.randn(S, B, case.K, generator=g, device=d)
        f["old_values"] = torch.randn(S, B, case.K, generator=g, device=d)
    if case.norm:
        mu, sigma = norm_of(case)
        f["returns"], f["old_values"] = mu + sigma * f["returns"], mu + sigma * f["old_values"]
    if case.beta:
        f["old_log_probs"] = torch.zeros(S, B, OR.ROW, device=d)
    if case.lam:
        f["teacher_log_probs"] = torch.zeros(S, B, OR.ROW, device=d)


def sample(f, rows):
    r = ST.sample(f, rows)
    idx = torch.tensor(rows, device=f["valid"].device)
    for k in ("old_log_probs", "teacher_log_probs"):
        r[k] = f[k].index_select(1, idx).cpu() if f.get(k) is not None else None
    return r


FITTED = ("old_logp", "returns", "old_values", "old_log_probs", "teacher_log_probs")


def fit(r, fwd, case, seed):
    logits = {k: v.detach() for k, v in fwd[0].items()}
    values = fwd[1].detach()
    ST.fit_to_reference(r, logits, values[..., 0] if case.K > 1 else values, seed, None)
    fit_values(r, values, case, seed + 1)
    fit_rows(r, logits, case, seed + 2)


@pytest.mark.parametrize("case", CPU_CASES, ids=[c.name for c in CPU_CASES])
def test_reference_and_bound_on_the_cpu(case):
    """At B 12 x S 16 x H 32: (1) the float64 reference on R equals the float64 transcription over the whole masked batch
    through the feature oracles, to 1e-10; (2) the fp32 transcription passes the bound; (3) each mutant applied to it
    fails."""
    torch.manual_seed(7)
    base = HeadsRefPolicy(case.H, case.cell, 1, case.K) if case.K > 1 else StackedRefPolicy(case.H, case.cell, 1)
    ST.grid_encoder(base, 3)
    f = ST.make_batch(case, 5, torch.device("cpu"))
    extend_batch(f, case, 6)
    r = sample(f, case.rows)
    ST.clear_relu_ties(PreRnnView(base), r, case)
    sd = base.state_dict()
    p64 = ref_policy(sd, case, torch.float64)
    fwd = ST.ref_forward(p64, r, torch.float64)
    fit(r, fwd, case, 9)
    for k in FITTED:
        if f.get(k) is not None:
            f[k][:, list(case.rows)] = r[k]
    f64 = ref_step(p64, r, case, torch.float64, fwd)
    f32 = ref_step(ref_policy(sd, case, torch.float32), r, case, torch.float32)
    if case.beta or case.lam:
        assert f64[0].get("kl", 0.0) > 0.01 and (not case.lam or f64[0]["teacher/kl"] > 0.05), f64[0]

    dbl = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in f.items()}
    full64 = transcription_step(ref_policy(sd, case, torch.float64), dbl, case)
    scal, diag = names(case)
    for n in scal + diag + (ACCURACY if case.bc else []):
        # the diagnostics oracle (padding_oracle.masked_stats) takes its log-probabilities in fp32
        tol = 1e-5 if n.startswith(("approx_kl", "clip_fraction")) else 1e-10
        assert abs(full64[0][n] - f64[0][n]) <= tol * max(1.0, abs(f64[0][n])), (n, full64[0][n], f64[0][n])
    for n, g in f64[1].items():
        assert float((full64[1][n] - g).abs().max()) <= 1e-10 * max(1e-30, float(g.abs().max())), n

    got = transcription_step(ref_policy(sd, case, torch.float32), f, case)
    ratios, over = compare(got, f64, f32, case)
    assert not over, (ratios, over)
    for mutant in CPU_MUTANTS[case.name]:
        m = transcription_step(ref_policy(sd, case, torch.float32), f, case, mutant)
        _, over = compare(m, f64, f32, case)
        assert over, "the %s mutant passed the bound" % mutant


# ------------------------------------------------------------------------------------------------ GPU
def save_teacher(tmp_path):
    """The reference's GRU-256 at its seeded initialisation, saved as a published model: the step reads only the rows."""
    from dotaclient_b200.policy import Policy
    torch.manual_seed(7)
    path = str(tmp_path / "teacher_gru256.pt")
    torch.save({k: v.detach().cpu() for k, v in Policy().state_dict().items()}, path)
    return path


def prepare(case, tmp_path):
    """-> (optimizer, device batch, float64 result, fp32 result), as ``test_gpu_step_fp64.prepare`` with the option's
    inputs fitted to the float64 forward."""
    from dotaclient_b200.optimizer import ExperienceBatch
    d = torch.device("cuda", 0)
    kw = {}
    if case.beta:
        kw["kl_coef"] = case.beta
    if case.lam:
        kw.update(teacher_model=save_teacher(tmp_path), teacher_coef=case.lam)
    if case.bc:
        kw["objective"] = "bc"
    if case.heads:
        kw.update(value_heads=case.heads, value_gammas=case.gammas)
    if case.norm:
        kw["value_norm"] = True
    opt = ST.make_optimizer(tmp_path, case, **kw)
    if case.norm:
        opt._value_norm = NORM_STATE
        assert opt._value_norm_moments() == norm_of(case)
    ST.grid_encoder(opt.policy_base, case.seed)
    f = ST.make_batch(case, case.seed + 1, d)
    extend_batch(f, case, case.seed + 3)
    r = sample(f, case.rows)
    ties = ST.clear_relu_ties(PreRnnView(opt.policy_base), r, case)
    sd = opt.policy_base.state_dict()
    p64 = ref_policy(sd, case, torch.float64)
    fwd = ST.ref_forward(p64, r, torch.float64)
    fit(r, fwd, case, case.seed + 2)
    idx = torch.tensor(case.rows, device=d)
    for k in FITTED:
        if f.get(k) is not None:
            f[k].index_copy_(1, idx, r[k].to(d))
    f64 = ref_step(p64, r, case, torch.float64, fwd)
    del fwd, p64
    f32 = ref_step(ref_policy(sd, case, torch.float32), r, case, torch.float32)
    if case.clip:
        assert f64[0]["clip_coef"] < 0.5, f64[0]["clip_coef"]
    else:
        assert f64[0]["clip_coef"] == 1.0
    f64[0]["relu_ties"] = ties
    return opt, ExperienceBatch(**f), f64, f32


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_objective_step_vs_fp64(case, tmp_path):
    """Every value the step reports for the option and every parameter's gradient within the bound; for the graph cases,
    the third call on the same batch (a graph replay) equals the first (eager) bit for bit."""
    t0 = time.perf_counter()
    ST.gc.collect()
    torch.cuda.empty_cache()
    opt, batch, f64, f32 = prepare(case, tmp_path)
    snap = ST.snapshot(opt)
    got = ST.gpu_step(opt, batch)
    params = opt.flat.param.clone()
    ratios, over = compare(got, f64, f32, case)
    left = unchecked(got, case)
    if left:
        over.append("reported but not compared: %s" % left)
    if case.graph:
        for call in (2, 3):                              # 2: capture + replay, 3: replay
            ST.restore(opt, snap)
            again = ST.gpu_step(opt, batch)
            if call == 3:
                assert any(not isinstance(v, str) for v in opt._graphs.values()), "the step was not captured"
                over += ["replayed %s differs" % k for k in got[0]
                         if not (got[0][k] == again[0][k] or (math.isnan(got[0][k]) and math.isnan(again[0][k])))]
                over += ["replayed gradient of %s differs" % n for n in got[1] if not torch.equal(got[1][n], again[1][n])]
                if not torch.equal(opt.flat.param, params):
                    over.append("replayed parameters differ")
    ST.release(opt)
    extra = (", KL %.4g, teacher KL %.4g" % (f64[0].get("kl", 0.0), f64[0].get("teacher/kl", 0.0))
             + (", accuracy %.4g (%d near-tie tokens)" % (f64[0]["bc/accuracy"], f64[0]["near_ties/bc/accuracy"])
                if case.bc else ""))
    print("\n%s: ratios %s, clip coef %.3g, old criterion %s, ReLU pre-activations within 1e-5 of 0 before the bias shift "
          "%d%s, %.1f s" % (case.name, ", ".join("%s %.3g" % kv for kv in ratios.items()), f64[0]["clip_coef"],
                            ST.old_criterion(got, f64), f64[0]["relu_ties"], extra, time.perf_counter() - t0))
    assert not over, over


MUTANTS = {"c2-kl": "kl_swap", "c2-joint-kl-teacher": "teacher_coef", "c2-bc": "bc_scale", "c2-heads3": "heads_swap",
           "c2-popart": "sigma"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MUTANTS))
def test_objective_mutants_fail_the_bound(name, tmp_path, monkeypatch):
    """Each mutant, applied inside this test only, must fail the bound: ``kl_swap`` swaps the enum rows of old_log_probs
    of tokens 5 and 6 of R's third column, ``teacher_coef`` writes lambda to the device as 0.99 lambda, ``bc_scale``
    scales the loss's dlogits (the NLL's and the entropy term's gradient) by T_a / (T_a + 1), ``heads_swap`` swaps the
    returns of heads 0 and 1 on the first 2 tokens of R's third column, ``sigma`` uploads 1.01 sigma."""
    from dotaclient_b200 import ops
    case = CASE[name]
    mutant = MUTANTS[name]
    opt, batch, f64, f32 = prepare(case, tmp_path)
    opt.use_cuda_graph = False
    col = case.rows[2]
    b = batch
    with monkeypatch.context() as m:
        if mutant == "kl_swap":
            b = batch.map(lambda v: v)
            b.old_log_probs = batch.old_log_probs.clone()
            b.old_log_probs[[5, 6], col, 0:4] = batch.old_log_probs[[6, 5], col, 0:4]
        elif mutant == "teacher_coef":
            opt.teacher_coef = 0.99 * case.lam
        elif mutant == "bc_scale":
            t_a = float(batch.valid.sum())            # the enum head has an action row on every token
            orig = ops.ppo_loss_packed

            def scaled(*a, **kw):
                out = list(orig(*a, **kw))
                out[2] = out[2].clone()
                out[2][..., :25] *= t_a / (t_a + 1)
                out[3] = out[3] * (t_a / (t_a + 1))
                return tuple(out)
            m.setattr(ops, "ppo_loss_packed", scaled)
        elif mutant == "heads_swap":
            b = batch.map(lambda v: v)
            b.returns = batch.returns.clone()
            b.returns[0:2, col, 0], b.returns[0:2, col, 1] = batch.returns[0:2, col, 1], batch.returns[0:2, col, 0]
        else:
            mu, sigma = opt._value_norm_moments()
            m.setattr(opt, "_value_norm_moments", lambda: (mu, 1.01 * sigma))
        got = ST.gpu_step(opt, b)
    ratios, over = compare(got, f64, f32, case)
    ST.release(opt)
    print("\n%s mutant %s: fails bound %s, passes old criterion %s, ratios %s"
          % (name, mutant, [o.split(":")[0] for o in over][:4], ST.old_criterion(got, f64),
             {k: round(v, 3) for k, v in ratios.items()}))
    assert over, "the %s mutant passed the bound" % mutant
