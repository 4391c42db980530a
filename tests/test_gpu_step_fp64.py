"""One whole ``DotaOptimizer.train`` step (encoder, pre-RNN row, recurrence with or without resets, packed heads, target-unit
head, masked PPO loss, backward through every kernel, gradient finish) at the benchmark's shapes, against a float64
reference.

Sampling: the step runs the full ``[S, B]`` batch with ``mask_padding=True`` and ``valid = False`` on every token outside
a sample R of columns, so the loss depends on R alone while every kernel still runs the full shape, and the columns
outside R get an exactly zero upstream gradient.  The reference is ``StackedRefPolicy`` (``RefPolicy`` at one layer) in
float64 on R only -- every segment of a packed column run on its own from its start state -- followed by the
dtype-generic masked loss ``test_gpu_ppo_fp64.reference``, its backward and ``clip_grad_norm_``.  The same reference in
fp32 calibrates the bound every output must meet, per tensor:

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

R sits on both sides of the tile, cluster and M-tile boundaries of the design under test (the rows of
``test_gpu_rnn_fp64.CASES``).  Encoder weights and observations lie on coarse grids (``test_gpu_encoder._grid``), so the
encoder forward is exact and max-pool ties resolve the same way on both sides; the other weights are the seeded fp32
initialisation, upcast for the reference.  Old log-probabilities and old values are set from the float64 forward so
that no token lies within 1e-3 of a clip bound (fp32 and float64 then clip the same tokens).  For the same reason the
pre-RNN ReLU is kept off its kink (``clear_relu_ties``): the pre-RNN row multiplies the exact encoder row by seeded fp32
weights, and every case has some of R's pre-activations within 1e-5 of 0 (0 to 69 per case), where fp32 and float64 can
disagree on a token's ReLU mask.  Before this was done, c3, c3-packed and gru256-packed (which then drew the same data)
failed the bound in affine_pre_rnn's and the encoder's gradients alone (8e-4 of their magnitude, up to 9e-2 at S 64);
with the ties cleared they pass with the margins below.

``test_sampling_and_bound_on_the_cpu`` shows without a GPU, on a plain and a packed batch, that the reference on R equals
the full-batch masked loss (the sampling is exact; packed: the reference's per-segment runs against ``ResetLSTM``), that
an independent fp32 transcription of the step passes the bound and that the mutants below, applied to it, fail it.

K and FLOOR per kind (``BOUNDS``): losses, entropies and gradient norms 8 and 4e-6; PPO diagnostics (approximate KL,
clip fractions, explained variance: nonlinear in the log-ratios) 8 and 1e-5; recurrent weight gradients 4 and 1e-4, as
``test_gpu_rnn_fp64``; encoder, pre-RNN and head weight gradients 8 and 5e-5 at every token count.  The weight floor
used to grow as (T / 131072)^1.5 above c2 (to 4e-4 at c4), and the recurrent one was 5e-4, because the weight-gradient
GEMM's error grew with the tokens one accumulator summed: c4's largest weight and recurrent errors were 1.9e-4 and
2.1e-4 of max|f64| (820 and 495 times torch's).  Since that GEMM flushes its accumulator every 4096 rows
(``test_gpu_wgrad_length``) they are 1.7e-5 and 1.5e-5.  Measured on one H100 80GB HBM3 (700 W power limit): the
largest ratio max|gpu - f64| / max|torch32 - f64| per kind (scalar / diagnostic / weight / recurrent), the largest
max|gpu - f64| / max|f64| of the weight and recurrent gradients in brackets, the largest share of its bound any output
uses, and the wall time of the case (reference included); before the flush, c3 read 15 / 13 / 5.0 / 14 (2.4e-5, 6.5e-5)
and c4 5.0 / 68 / 820 / 495 (1.9e-4, 2.1e-4):
    c1              4.5 /  43 /  128 /  16  (5.9e-6, 6.8e-6)  0.34   5 s
    c2              6.1 / 5.3 / 7560 /  28  (7.1e-6, 8.6e-6)  0.46   3 s
    c3 (clip on)     15 /  13 /  2.0 / 2.5  (9.6e-6, 1.2e-5)  0.27   3 s
    c4              4.5 /  68 /   91 /  27  (1.7e-5, 1.5e-5)  0.32   6 s
    c5 (clip on)     18 /  45 /  3.5 / 2.7  (5.6e-6, 4.1e-6)  0.71   1 s
    c2-2layers      7.2 /  21 /   24 /  23  (8.5e-6, 9.2e-6)  0.39   3 s
    c2-packed (on)  4.4 / 3.4 /  3.5 / 3.6  (4.8e-6, 6.4e-6)  0.34   5 s
    c3-packed       1.8 / 6.4 /   40 /  41  (9.0e-6, 1.3e-5)  0.20   6 s
    gru256-packed   10  /  13 /  2.3 / 1.1  (8.3e-6, 4.5e-6)  0.22   7 s   (clip on)
    c2-joint         15 / 253 /   86 /  21  (9.2e-6, 8.2e-6)  0.35   2 s
Where fp32 on the grid encoder is nearly exact (weight ratio 7560 at c2) the floor carries the bound.

Mutants (``test_mutants_fail_the_bound``), all failing the bound; the largest share of its bound an output uses, the
first outputs over it, and whether the per-tensor gradient criterion of the fp32-oracle tests (cosine > 0.9999, norm
within 2e-3) catches them:
    d_tu * 0.99 (c2)                 301x   norms, encoder          caught
    swap h0 of columns 1, 2 (c2)     1890x  losses                  caught
    W_hh rounded to TF32 (c2)        1.8x   encoder weights         NOT caught
    no reset dW_hh term (c2-packed)  329x   norms, encoder, W_hh    caught (W_hh's gradient moves by 17 %)
The graph replays of c2 and c2-packed are bitwise equal to the eager step; the masked all-valid step at c2 is bitwise
the unmasked step.  The whole file runs in about 55 s on the H100.
"""
import copy
import gc
import math
import time
import uuid
import zlib

import numpy as np
import pytest
import torch

import test_gpu_ppo_fp64 as PF
from padding_oracle import masked_ppo_loss, masked_stats
from stacked_oracle import StackedRefPolicy
from test_gpu_encoder import _grid
from test_gpu_rnn_fp64 import bound_check, tf32_rna

HEADS = PF.HEADS
SIZES = dict(zip(PF.HEADS, PF.SIZES))
E_CLIP = PF.E_CLIP                 # the clip range the float64 loss reference is written for
VALUE_CLIP = 0.2
ENCODER = ("affine_env", "affine_unit_basic_stats") + tuple("affine_unit_" + s for s in ("ah", "eh", "anh", "enh", "ath", "eth"))

# (K, FLOOR) per kind of output: the losses, entropies, PPO diagnostics and gradient norms; the gradients of the
# encoder, pre-RNN and head weights; the gradients of the recurrent weights (sums over thousands of tokens of h2h terms)
BOUNDS = {"scalar": (8.0, 4e-6), "diagnostic": (8.0, 1e-5), "weight": (8.0, 5e-5), "recurrent": (4.0, 1e-4)}
OLD_COSINE, OLD_NORM = 0.9999, 2e-3    # the fp32-oracle tests' gradient criterion: per-tensor cosine and norm ratio


class Case:
    def __init__(self, name, cell, B, S, H, rows, layers=1, packed=False, joint=False, clip=False, graph=False):
        self.name, self.cell, self.B, self.S, self.H, self.rows = name, cell, B, S, H, tuple(rows)
        self.seed = zlib.crc32(name.encode()) % 2 ** 31     # every case draws its own weights and data
        self.layers, self.packed, self.joint, self.clip, self.graph = layers, packed, joint, clip, graph
        self.max_grad_norm = 0.01 if clip else 1e9          # clip on: far below the step's gradient norm; off: never reached
        self.value_clip = VALUE_CLIP if joint else None


C2_ROWS = (0, 1, 2, 127, 128, 129, 254, 255)                         # resident H 128: 2-sequence tiles
C3_ROWS = (0, 31, 32, 255, 256, 480, 481, 511)                       # cluster H 256: 32 sequences per cluster
CASES = [
    Case("c1", "lstm", 1, 64, 128, (0,)),
    Case("c2", "lstm", 256, 512, 128, C2_ROWS, graph=True),
    Case("c3", "lstm", 512, 512, 256, C3_ROWS, clip=True),
    Case("c4", "lstm", 512, 1024, 512, (0, 127, 128, 255, 256, 383, 384, 511)),     # step-wise H 512: 128-row M tiles
    Case("c5", "gru", 1024, 16, 256, (0, 31, 32, 511, 512, 991, 992, 1023), clip=True),   # 32 clusters
    Case("c2-2layers", "lstm", 256, 512, 128, C2_ROWS, layers=2),
    Case("c2-packed", "lstm", 256, 512, 128, C2_ROWS, packed=True, clip=True, graph=True),
    Case("c3-packed", "lstm", 512, 512, 256, C3_ROWS, packed=True),
    Case("gru256-packed", "gru", 512, 512, 256, C3_ROWS, packed=True, clip=True),
    Case("c2-joint", "lstm", 256, 512, 128, C2_ROWS, joint=True),
]
CASE = {c.name: c for c in CASES}


# ------------------------------------------------------------------------------------------------ inputs
def reset_pattern(S, B, rows):
    """``reset_slot [S, B]`` int32 and K: the patterns of ``test_gpu_packing.reset_pattern`` stretched to S, and every
    column carries at least one reset: t = S/3 / t = 0 / t = 1 and S-1 / consecutive S/2, S/2 + 1 / four resets / t = S-1.
    Column b takes pattern b % 6, the sampled columns take patterns 0..5 in turn."""
    pats = [[S // 3], [0], [1, S - 1], [S // 2, S // 2 + 1], [S // 8, S // 2 - 1, 3 * S // 4, S - 2], [S - 1]]
    pick = np.arange(B) % 6
    pick[list(rows)] = np.arange(len(rows)) % 6
    slot = np.full((S, B), -1, dtype=np.int32)
    for b in range(B):
        for k, t in enumerate(pats[pick[b]]):
            slot[t, b] = k
    return slot, max(len(p) for p in pats)


def grid_encoder(pol, seed):
    """Encoder weights on the grids of ``test_gpu_encoder``: every encoder product is exact in fp32 (and in each TF32 half)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        pol.affine_env.weight.copy_(_grid(g, (128, 3), 32, 64))
        pol.affine_env.bias.copy_(_grid(g, (128,), 8, 64))
        pol.affine_unit_basic_stats.weight.copy_(_grid(g, (128, 12), 4, 8))
        pol.affine_unit_basic_stats.bias.copy_(_grid(g, (128,), 16, 32))
        for name in ENCODER[2:]:
            getattr(pol, name).weight.copy_(_grid(g, (128, 128), 8, 64))
            getattr(pol, name).bias.copy_(_grid(g, (128,), 8, 64))


def make_batch(case, seed, device):
    """The training batch of ``case`` as ``ExperienceBatch`` fields on ``device``: grid observations, actions and masks
    with the distributions of ``synthetic.make_rollout``, non-zero h0 / c0, ``valid`` False outside R and on the padding
    tail of R's second and second-last columns, and for a packed case the resets and their state tables.  The old
    log-probabilities, advantages, returns and old values of R are set later (``fit_to_reference``)."""
    S, B, H, L, d = case.S, case.B, case.H, case.layers, device
    g = torch.Generator(device=d).manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, device=d)              # noqa: E731
    rint = lambda lo, hi, *s: torch.randint(lo, hi, s, generator=g, device=d)       # noqa: E731
    grid = lambda shape, k, scale: rint(-k, k + 1, *shape).float() / scale          # noqa: E731  (_grid on the device)
    from dotaclient_b200.synthetic import OBS_SHAPES
    obs = {k: grid((S, B) + shp, 48 if k == "env" else 4, 16 if k == "env" else 4) for k, shp in OBS_SHAPES.items()}
    n = S * B
    rows = torch.arange(n, device=d)
    masks = {k: torch.zeros(n, m, dtype=torch.bool, device=d) for k, m in SIZES.items()}
    actions = {k: torch.zeros(n, m, dtype=torch.bool, device=d) for k, m in SIZES.items()}
    enum = rint(0, 4, n)
    masks["enum"][:] = True
    actions["enum"][rows, enum] = True
    for k, e in (("x", 1), ("y", 1), ("ability", 3)):
        pick = rint(0, SIZES[k], n)
        used = enum == e
        masks[k][used] = True
        actions[k][rows[used], pick[used]] = True
    attack = enum == 2
    units = rnd(n, 40) < 0.5
    units[:, 0] = False
    units[rows, rint(1, 40, n)] = True
    target = rnd(n, 40).masked_fill(~units, -1.0).argmax(dim=1)
    masks["target_unit"][attack] = units[attack]
    actions["target_unit"][rows[attack], target[attack]] = True
    masks = {k: v.view(S, B, -1) for k, v in masks.items()}
    actions = {k: v.view(S, B, -1) for k, v in actions.items()}
    valid = torch.zeros(S, B, dtype=torch.bool, device=d)
    valid[:, list(case.rows)] = True
    for j in {1, len(case.rows) - 2} if len(case.rows) > 2 else {0}:
        valid[S - max(1, S // 5):, case.rows[j]] = False                 # a padding tail after a real prefix
    f = dict(observations=obs, masks=masks, actions=actions, old_logp=torch.zeros(S, B, 5, device=d),
             advantages=torch.randn(S, B, generator=g, device=d), returns=torch.randn(S, B, generator=g, device=d),
             h0=0.5 * torch.randn(L, B, H, generator=g, device=d), old_values=torch.randn(S, B, generator=g, device=d),
             valid=valid)
    f["c0"] = 0.5 * torch.randn(L, B, H, generator=g, device=d) if case.cell == "lstm" else None
    if case.packed:
        slot, K = reset_pattern(S, B, case.rows)
        f["reset_slot"] = torch.from_numpy(slot).to(d)
        f["reset_h"] = 0.5 * torch.randn(K, B, L * H, generator=g, device=d)
        f["reset_c"] = 0.5 * torch.randn(K, B, L * H, generator=g, device=d) if case.cell == "lstm" else None
    return f


def sample(f, rows):
    """The R columns of the batch fields, on the CPU."""
    idx = torch.tensor(rows, device=f["valid"].device)
    col = lambda t: None if t is None else t.index_select(1, idx).cpu()            # noqa: E731
    out = {k: col(f.get(k)) for k in ("old_logp", "advantages", "returns", "old_values", "valid", "h0", "c0", "reset_slot",
                                      "reset_h", "reset_c")}
    for k in ("observations", "masks", "actions"):
        out[k] = {key: col(v) for key, v in f[k].items()}
    return out


RELU_MARGIN = 1e-4        # least |pre-activation| of the pre-RNN ReLU on R after clear_relu_ties


def clear_relu_ties(pol, r, case):
    """Keeps the pre-RNN ReLU away from its kink on R: its inputs are the exact grid encoder row times seeded fp32 weights,
    so some of R's thousands of pre-activations z lie within the fp32 rounding of z (about 1e-6) of 0, where fp32 and
    float64 can disagree on the ReLU mask of a token -- a whole token's gradient through that unit.  Per unit whose
    float64 z on R comes closer than 2 * RELU_MARGIN to 0, ``affine_pre_rnn.bias`` is shifted by the least amount that
    puts 0 in the middle of a gap of at least 6 * RELU_MARGIN between that unit's z values.  Returns the number of z on R
    with |z| < 1e-5 before the shift."""
    p64 = ref_policy(pol.state_dict(), case, torch.float64)
    zs = []
    hook = p64.affine_pre_rnn.register_forward_hook(lambda m, i, o: zs.append(o.detach().reshape(-1, o.shape[-1])))
    with torch.no_grad():
        ref_forward(p64, r, torch.float64)
    hook.remove()
    z = torch.cat(zs).numpy()
    near = int((np.abs(z) < 1e-5).sum())
    shift = np.zeros(z.shape[1])
    for j in range(z.shape[1]):
        if np.abs(z[:, j]).min() >= 2 * RELU_MARGIN:
            continue
        v = np.sort(z[:, j])
        mid = (v[:-1] + v[1:]) / 2
        wide = v[1:] - v[:-1] >= 6 * RELU_MARGIN
        shift[j] = -mid[wide][np.argmin(np.abs(mid[wide]))]
    bias = pol.affine_pre_rnn.bias
    before = bias.detach().cpu().double().numpy()
    with torch.no_grad():
        bias.add_(torch.from_numpy(shift).to(bias))
    after = z + (bias.detach().cpu().double().numpy() - before)
    assert np.abs(after).min() >= RELU_MARGIN, np.abs(after).min()
    return near


# ------------------------------------------------------------------------------------------------ reference
def ref_policy(state_dict, case, dtype):
    pol = StackedRefPolicy(case.H, case.cell, case.layers)
    pol.load_state_dict({k: v.detach().cpu() for k, v in state_dict.items()})
    return pol.to(dtype)


def ref_forward(pol, r, dtype):
    """Time-major ``[S, R]`` sample ``r`` -> (logits {head: [S, R, n]}, values [S, R]) of ``pol``; a packed column runs
    segment by segment, each from h0 / c0 or from its reset's rows of the state tables."""
    L, H, lstm = pol.num_layers, pol.hidden_size, pol.cell == "lstm"
    obs = {k: v.to(dtype).transpose(0, 1) for k, v in r["observations"].items()}          # batch-first [R, S, ...]
    h0 = r["h0"].to(dtype)
    c0 = r["c0"].to(dtype) if lstm else None
    if r["reset_slot"] is None:
        logits, values, _ = pol(**obs, hidden=(h0, c0) if lstm else h0)
        return {k: v.transpose(0, 1) for k, v in logits.items()}, values[..., 0].transpose(0, 1)
    slot = r["reset_slot"].numpy()
    S, R = slot.shape
    cols = []
    for b in range(R):
        starts = [0] + [t for t in range(1, S) if slot[t, b] >= 0] + [S]
        parts = []
        for t0, t1 in zip(starts, starts[1:]):
            k = int(slot[t0, b])
            if k >= 0:
                h = r["reset_h"][k, b].to(dtype).view(L, 1, H)
                c = r["reset_c"][k, b].to(dtype).view(L, 1, H) if lstm else None
            else:
                h, c = h0[:, b:b + 1], (c0[:, b:b + 1] if lstm else None)
            lg, v, _ = pol(**{key: val[b:b + 1, t0:t1] for key, val in obs.items()}, hidden=(h, c) if lstm else h)
            parts.append((lg, v))
        cols.append(({k: torch.cat([p[0][k] for p in parts], 1) for k in HEADS}, torch.cat([p[1] for p in parts], 1)))
    logits = {k: torch.cat([c[0][k] for c in cols], 0).transpose(0, 1) for k in HEADS}
    return logits, torch.cat([c[1] for c in cols], 0)[..., 0].transpose(0, 1)


def fit_to_reference(r, logits, values, seed, value_clip):
    """Old log-probabilities (log-ratios in +-0.5) and, under value clipping, old values (|v - v_old| in 0..2 clip) of R
    from the float64 forward, with every token more than 1e-3 away from a clip bound (per head and joint, and away from a
    tie of the clipped value loss's two squares)."""
    g = torch.Generator().manual_seed(seed)
    S, R = values.shape
    with torch.no_grad():
        sel = torch.stack([(PF.log_softmax(logits[k].reshape(S * R, -1), r["masks"][k].reshape(S * R, -1))
                            * r["actions"][k].reshape(S * R, -1)).sum(1) for k in HEADS], 1)
        acted = torch.stack([r["actions"][k].reshape(S * R, -1).any(1) for k in HEADS], 1)
        old = sel - (torch.rand(S * R, 5, generator=g, dtype=torch.float64) - 0.5)
        bounds = torch.tensor([math.log(1 - E_CLIP), math.log(1 + E_CLIP)], dtype=torch.float64)
        for _ in range(4):
            lr = torch.where(acted, sel - old, torch.zeros_like(sel))
            near = acted & ((lr[..., None] - bounds).abs() < 1e-3).any(-1)
            old = torch.where(near, old - 3e-3, old)
            joint = lr.sum(1)
            near_j = ((joint[:, None] - bounds).abs() < 1e-3).any(-1)
            old[:, 0] = torch.where(near_j, old[:, 0] - 3e-3, old[:, 0])
        r["old_logp"] = torch.where(acted, old, torch.zeros_like(old)).float().view(S, R, 5)
        if value_clip:
            v = values.reshape(-1)
            dv = (torch.rand(S * R, generator=g, dtype=torch.float64) * 4 - 2) * value_clip
            dv = torch.where((dv.abs() - value_clip).abs() < 2e-3, dv + 5e-3 * dv.sign(), dv)
            vo = (v - dv).float().double()
            ret = r["returns"].reshape(-1).double()
            vc = vo + (v - vo).clamp(-value_clip, value_clip)
            tie = (2 * ret - v - vc).abs() < 2e-3
            r["returns"] = torch.where(tie, ret + 0.01, ret).float().view(S, R)
            r["old_values"] = vo.float().view(S, R)


def ref_step(pol, r, case, dtype, fwd=None):
    """The masked loss of sample ``r`` under ``pol`` in ``dtype``, its backward and the global-norm clip -> (scalars
    {name: float}, clipped gradients {parameter name: tensor})."""
    pol.zero_grad(set_to_none=True)
    logits, values = fwd if fwd is not None else ref_forward(pol, r, dtype)
    S, R = values.shape
    n = S * R
    # a row whose mask is empty (the head is not in use) counts for nothing; it enters the loss reference as a logit of 0
    # under a one-entry mask, which is exactly 0 in its entropy and gradient (0/0 otherwise)
    lgs, msks = [], []
    for k in HEADS:
        m = r["masks"][k].reshape(n, -1)
        empty = ~m.any(1, keepdim=True)
        lgs.append(torch.where(empty, 0.0, logits[k].detach().reshape(n, -1)))
        msks.append(m | (empty & (torch.arange(m.shape[1]) == 0)))
    inp = {"logits": lgs, "masks": msks, "actions": [r["actions"][k].reshape(n, -1) for k in HEADS],
           "old": r["old_logp"].reshape(n, 5), "adv": r["advantages"].reshape(n), "ret": r["returns"].reshape(n),
           "values": values.detach().reshape(n), "old_values": r["old_values"].reshape(n), "valid": r["valid"].reshape(n)}
    out = PF.reference(inp, dtype, case.joint, value_clip=case.value_clip)
    torch.autograd.backward([logits[k] for k in HEADS] + [values],
                            [d.view_as(logits[k]) for d, k in zip(out["dlogits"], HEADS)] + [out["dvalue"].view_as(values)])
    return finish(pol, out, case.max_grad_norm)


def finish(pol, out, max_grad_norm):
    """``mean_gradient_norm`` before and after ``clip_grad_norm_(max_grad_norm)`` and the clipped gradients."""
    grads = {n: (p.grad if p.grad is not None else torch.zeros_like(p)).detach().clone() for n, p in pol.named_parameters()}
    norms = torch.stack([g.norm() for g in grads.values()])
    coef = min(1.0, max_grad_norm / (float(norms.pow(2).sum().sqrt()) + 1e-6))
    scal = {k: float(v) for k, v in out.items() if isinstance(v, (int, float))}
    scal["unclipped"] = float(norms.mean())
    scal["clipped"] = float(norms.mean()) * coef
    scal["clip_coef"] = coef
    return scal, {n: g * coef for n, g in grads.items()}


def scalar_names(case):
    names = ["loss", "policy", "entropy_loss", "value_loss", "unclipped", "clipped"] + ["entropy/" + k for k in HEADS]
    return names + diagnostic_names(case)


def diagnostic_names(case):
    names = ["approx_kl", "clip_fraction", "explained_variance"] + ["approx_kl/" + k for k in HEADS] \
        + ["clip_fraction/" + k for k in HEADS]
    return names + (["approx_kl/joint", "clip_fraction/joint"] if case.joint else [])


def compare(got, f64, f32, case):
    """-> (largest ratio max|got - f64| / max|f32 - f64| per kind, the largest max|got - f64| / max|f64| of the gradients,
    and the largest share of its bound any output uses; the tensors over their bound)."""
    diag = diagnostic_names(case)
    return compare_names(got, f64, f32, [n for n in scalar_names(case) if n not in diag], diag)


def compare_names(got, f64, f32, scalars, diag):
    """``compare`` of the reported values named in ``scalars`` (kind 'scalar') and ``diag`` (kind 'diagnostic') and of
    every gradient."""
    names = list(scalars) + list(diag)
    as_t = lambda d: {n: torch.tensor(float(d[n]), dtype=torch.float64) for n in names}      # noqa: E731
    groups = [("scalar", list(scalars), as_t(got[0]), as_t(f64[0]), as_t(f32[0])),
              ("diagnostic", list(diag), as_t(got[0]), as_t(f64[0]), as_t(f32[0]))]
    for kind in ("weight", "recurrent"):
        groups.append((kind, [n for n in f64[1] if n.startswith("rnn.") == (kind == "recurrent")], got[1], f64[1], f32[1]))
    ratios, over, used = {}, [], 0.0
    for kind, ns, a, b, c in groups:
        r, o = bound_check(a, b, c, ns, BOUNDS[kind])
        ratios[kind] = max((v for n, v in r.items() if not n.startswith("rel ") and math.isfinite(v)), default=0.0)
        if kind in ("weight", "recurrent"):
            ratios[kind + " rel"] = max(v for n, v in r.items() if n.startswith("rel "))
        over += o
        k, floor = BOUNDS[kind]
        for n in ns:
            err = float((a[n].double() - b[n]).abs().max())
            bound = k * float((c[n].double() - b[n]).abs().max()) + floor * float(b[n].abs().max())
            used = max(used, err / bound if bound > 0 else (0.0 if err == 0 else math.inf))
    ratios["of bound"] = used
    return ratios, over


def old_criterion(got, f64):
    """True when every gradient passes the fp32-oracle tests' per-tensor cosine > 0.9999 / norm within 2e-3."""
    for n, ref in f64[1].items():
        a, b = got[1][n].double().reshape(-1), ref.reshape(-1)
        na, nb = float(a.norm()), float(b.norm())
        if nb == 0:
            if na != 0:
                return False
            continue
        if not (float(a @ b) / (na * nb + 1e-300) > OLD_COSINE and abs(na / nb - 1) <= OLD_NORM):
            return False
    return True


# ------------------------------------------------------------------------------------------------ CPU: sampling and bound
class ResetLSTM(torch.nn.Module):
    """One batch-first ``nn.LSTM`` layer with the state resets of a packed batch, for the transcription: each column runs
    as one sequence, and the step at a reset is written out from the cell equations with the table row as its state.
    ``drop_correction``: that step's h2h product pairs its gate gradient with the state the column carried into it
    (what dW_hh is without the reset correction of ``ops.RnnSequence.backward``) while its value keeps the table row."""

    def __init__(self, lstm, slot, h_tab, c_tab, drop_correction=False):
        super().__init__()
        assert lstm.num_layers == 1
        for n, p in lstm.named_parameters():
            self.register_parameter(n, p)                # the same Parameters: they keep their gradients and names
        self._lstm = [lstm]
        self.slot, self.h_tab, self.c_tab, self.drop = slot, h_tab, c_tab, drop_correction

    def forward(self, x, hidden):
        lstm = self._lstm[0]
        h0, c0 = hidden
        B, S, H = x.shape[0], x.shape[1], h0.shape[-1]
        w_ih, w_hh, b_ih, b_hh = self.weight_ih_l0, self.weight_hh_l0, self.bias_ih_l0, self.bias_hh_l0
        ys = []
        for b in range(B):
            h, c = h0[:, b:b + 1], c0[:, b:b + 1]
            starts = [0] + [t for t in range(1, S) if self.slot[t, b] >= 0] + [S]
            outs = []
            for t0, t1 in zip(starts, starts[1:]):
                k = int(self.slot[t0, b])
                if k >= 0:
                    hr, cr = self.h_tab[k, b].to(x.dtype), self.c_tab[k, b].to(x.dtype)
                    if self.drop:
                        carried = h.reshape(H).detach()
                        gh = carried @ w_hh.t() + (hr - carried) @ w_hh.detach().t() + b_hh
                    else:
                        gh = hr @ w_hh.t() + b_hh
                    i, f, g, o = (x[b, t0] @ w_ih.t() + b_ih + gh).chunk(4)
                    c = (torch.sigmoid(f) * cr + torch.sigmoid(i) * torch.tanh(g)).view(1, 1, H)
                    h = (torch.sigmoid(o) * torch.tanh(c)).view(1, 1, H)
                    outs.append(h)
                    t0 += 1
                if t1 > t0:
                    y, (h, c) = lstm(x[b:b + 1, t0:t1], (h, c))
                    outs.append(y)
            ys.append(torch.cat(outs, 1))
        return torch.cat(ys, 0), None


def transcription_step(pol, f, case, mutant=None):
    """An fp32 transcription of the step independent of ``ref_step``: the policy over the WHOLE batch (not R alone), with
    ``ResetLSTM`` for the resets of a packed batch, the loss of ``padding_oracle.masked_ppo_loss`` / ``masked_stats``
    differentiated straight through the network, then the clip.  ``mutant``: 'd_tu' scales the target-unit logits'
    gradient by 0.99, 'swap_h0' swaps h0 / c0 of R's second and third columns (adjacent), 'tf32_whh' rounds W_hh to
    TF32, 'drop_reset_dwhh' drops the reset steps' dW_hh correction (``ResetLSTM(drop_correction=True)``)."""
    S, B = f["valid"].shape
    f = dict(f)
    if mutant == "swap_h0":
        a, b = case.rows[1], case.rows[2]
        for k in ("h0", "c0"):
            if f[k] is not None:
                t = f[k].clone()
                t[:, [a, b]] = t[:, [b, a]]
                f[k] = t
    if mutant == "tf32_whh":
        pol = copy.deepcopy(pol)
        with torch.no_grad():
            for k in range(case.layers):
                w = getattr(pol.rnn, "weight_hh_l%d" % k)
                w.copy_(tf32_rna(w))
    if f.get("reset_slot") is not None:
        pol.rnn = ResetLSTM(pol.rnn, f["reset_slot"].numpy(), f["reset_h"], f["reset_c"], mutant == "drop_reset_dwhh")
    pol.zero_grad(set_to_none=True)
    full = dict(f, reset_slot=None)
    logits, values = ref_forward(pol, full, next(pol.parameters()).dtype)
    if mutant == "d_tu":
        logits["target_unit"].register_hook(lambda g: g * 0.99)
    n = S * B
    lg = {k: logits[k].reshape(n, -1) for k in HEADS}
    act = {k: f["actions"][k].reshape(n, -1) for k in HEADS}
    msk = {k: f["masks"][k].reshape(n, -1) for k in HEADS}
    loss, p_loss, e_loss, v_loss, ents = masked_ppo_loss(lg, values.reshape(n), act, msk, f["old_logp"].reshape(n, 5),
                                                         f["advantages"].reshape(n), f["returns"].reshape(n),
                                                         f["valid"].reshape(n), 5e-4, 0.5, E_CLIP)
    loss.backward()
    with torch.no_grad():
        st = masked_stats(lg, act, msk, f["old_logp"].reshape(n, 5), values.reshape(n), f["returns"].reshape(n),
                          f["valid"].reshape(n), E_CLIP)
    out = dict(st, loss=float(loss), policy=float(p_loss), entropy_loss=float(e_loss), value_loss=float(v_loss))
    out.update({"entropy/" + k: float(v) for k, v in ents.items()})
    return finish(pol, out, case.max_grad_norm)


@pytest.mark.parametrize("packed", [False, True], ids=["plain", "packed"])
def test_sampling_and_bound_on_the_cpu(packed):
    """At B 12 x S 16 x H 32: (1) the float64 reference on R equals the float64 transcription over the whole masked batch
    (the sampling trick is exact; packed: the reference's segments against ``ResetLSTM``); (2) the fp32 transcription
    passes the bound; (3) each mutant applied to it fails."""
    case = Case("cpu-packed" if packed else "cpu", "lstm", 12, 16, 32, (0, 3, 4, 5, 6, 11), packed=packed)
    torch.manual_seed(7)
    base = StackedRefPolicy(case.H, case.cell, 1)
    grid_encoder(base, 3)
    f = make_batch(case, 5, torch.device("cpu"))
    r = sample(f, case.rows)
    clear_relu_ties(base, r, case)
    sd = base.state_dict()
    p64, p32 = ref_policy(sd, case, torch.float64), ref_policy(sd, case, torch.float32)
    fwd = ref_forward(p64, r, torch.float64)
    fit_to_reference(r, {k: v.detach() for k, v in fwd[0].items()}, fwd[1].detach(), 9, case.value_clip)
    for k in ("old_logp", "returns", "old_values"):
        f[k][:, list(case.rows)] = r[k]
    f64 = ref_step(p64, r, case, torch.float64, fwd)
    f32 = ref_step(p32, r, case, torch.float32)

    full64 = transcription_step(ref_policy(sd, case, torch.float64), {k: (v.double() if torch.is_tensor(v) and
                                                                           v.is_floating_point() else v)
                                                                       for k, v in f.items()}, case)
    for n in ["loss", "policy", "entropy_loss", "value_loss", "unclipped", "clipped"] + ["entropy/" + k for k in HEADS]:
        assert abs(full64[0][n] - f64[0][n]) <= 1e-10 * max(1.0, abs(f64[0][n])), (n, full64[0][n], f64[0][n])
    for n, g in f64[1].items():
        assert float((full64[1][n] - g).abs().max()) <= 1e-10 * max(1e-30, float(g.abs().max())), n

    got = transcription_step(ref_policy(sd, case, torch.float32), f, case)
    ratios, over = compare(got, f64, f32, case)
    assert not over, (ratios, over)
    for mutant in ("drop_reset_dwhh",) if packed else ("d_tu", "swap_h0", "tf32_whh"):
        _, over = compare(transcription_step(ref_policy(sd, case, torch.float32), f, case, mutant), f64, f32, case)
        assert over, "the %s mutant passed the bound" % mutant


def test_reset_pattern_covers_every_sampled_column():
    for case in CASES:
        if case.packed:
            slot, K = reset_pattern(case.S, case.B, case.rows)
            assert ((slot >= 0).sum(0) >= 1).all() and K * case.B >= 4 * 128
            assert slot[0, case.rows[1]] == 0 and slot[case.S - 1, case.rows[5]] == 0
            assert (slot[:, case.rows[4]] >= 0).sum() == 4


# ------------------------------------------------------------------------------------------------ GPU
def make_optimizer(tmp_path, case, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    kw = dict(dict(mask_padding=True, clip_range=E_CLIP, max_grad_norm=case.max_grad_norm, value_clip=case.value_clip,
                   policy_ratio="joint" if case.joint else "per_head"), **kw)
    return DotaOptimizer(rmq_host="step-fp64", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=1,
                         seq_len=case.S, learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                         log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=case.H,
                         cell=case.cell, num_layers=case.layers, **kw)


def prepare(case, tmp_path):
    """-> (optimizer, device batch, float64 result, fp32 result): the batch's R columns carry the old log-probabilities,
    returns and old values fitted to the float64 forward."""
    from dotaclient_b200.optimizer import ExperienceBatch
    d = torch.device("cuda", 0)
    opt = make_optimizer(tmp_path, case)
    grid_encoder(opt.policy_base, case.seed)
    f = make_batch(case, case.seed + 1, d)
    r = sample(f, case.rows)
    ties = clear_relu_ties(opt.policy_base, r, case)
    sd = opt.policy_base.state_dict()
    p64 = ref_policy(sd, case, torch.float64)
    fwd = ref_forward(p64, r, torch.float64)
    fit_to_reference(r, {k: v.detach() for k, v in fwd[0].items()}, fwd[1].detach(), case.seed + 2, case.value_clip)
    idx = torch.tensor(case.rows, device=d)
    for k in ("old_logp", "returns", "old_values"):
        f[k].index_copy_(1, idx, r[k].to(d))
    f64 = ref_step(p64, r, case, torch.float64, fwd)
    del fwd, p64
    f32 = ref_step(ref_policy(sd, case, torch.float32), r, case, torch.float32)
    if case.clip:
        assert f64[0]["clip_coef"] < 0.5, f64[0]["clip_coef"]
    else:
        assert f64[0]["clip_coef"] == 1.0
    f64[0]["relu_ties"] = ties
    batch = ExperienceBatch(**f)
    return opt, batch, f64, f32


def gpu_step(opt, batch):
    """One ``train`` step -> (scalars, gradients on the CPU) in the reference's naming."""
    losses, entropies, norms = opt.train(batch)
    out = {"loss": losses["loss"], "policy": losses["policy_loss"], "entropy_loss": losses["entropy_loss"],
           "value_loss": losses["value_loss"], "unclipped": norms["unclipped"], "clipped": norms["clipped"]}
    out.update({"entropy/" + k: v for k, v in entropies.items()})
    out.update(opt.last_ppo_stats)
    return {k: float(v) for k, v in out.items()}, {n: opt.flat.grad_of(n).cpu() for n in opt.flat.names}


def snapshot(opt):
    return [t.clone() for t in (opt.flat.param, opt.exp_avg, opt.exp_avg_sq, opt.adam_steps)]


def restore(opt, snap):
    for t, s in zip((opt.flat.param, opt.exp_avg, opt.exp_avg_sq, opt.adam_steps), snap):
        t.copy_(s)


def release(opt):
    opt.close()
    del opt
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_step_vs_fp64(case, tmp_path):
    """Losses, entropies, PPO diagnostics, gradient norms and every parameter's gradient of one step within the bound; for
    the graph cases, the third call on the same batch (a graph replay) equals the first (eager) bit for bit."""
    t0 = time.perf_counter()
    gc.collect()
    torch.cuda.empty_cache()
    opt, batch, f64, f32 = prepare(case, tmp_path)
    snap = snapshot(opt)
    got = gpu_step(opt, batch)
    params = opt.flat.param.clone()
    ratios, over = compare(got, f64, f32, case)
    if case.graph:
        for call in (2, 3):                              # 2: capture + replay, 3: replay
            restore(opt, snap)
            again = gpu_step(opt, batch)
            if call == 3:
                assert any(not isinstance(v, str) for v in opt._graphs.values()), "the step was not captured"
                over += ["replayed %s differs" % k for k in got[0]
                         if not (got[0][k] == again[0][k] or (math.isnan(got[0][k]) and math.isnan(again[0][k])))]
                over += ["replayed gradient of %s differs" % n for n in got[1] if not torch.equal(got[1][n], again[1][n])]
                if not torch.equal(opt.flat.param, params):
                    over.append("replayed parameters differ")
    release(opt)
    print("\n%s: ratios %s, clip coef %.3g, old criterion %s, ReLU pre-activations within 1e-5 of 0 before the bias shift %d, "
          "%.1f s" % (case.name, ", ".join("%s %.3g" % kv for kv in ratios.items()), f64[0]["clip_coef"],
                      old_criterion(got, f64), f64[0]["relu_ties"], time.perf_counter() - t0))
    assert not over, over


MUTANTS = {"c2": ("d_tu", "swap_h0", "tf32_whh"), "c2-packed": ("drop_reset_dwhh",)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutants_fail_the_bound(name, tmp_path, monkeypatch):
    """Each mutant, applied inside this test only, must fail the bound: ``d_tu`` scales the target-unit logits' upstream
    gradient by 0.99, ``swap_h0`` swaps h0 / c0 of two adjacent sampled columns, ``tf32_whh`` rounds W_hh to TF32 before the
    step, ``drop_reset_dwhh`` drops the reset tokens' dW_hh correction (every reset-table row marked unused)."""
    from dotaclient_b200 import ops
    case = CASE[name]
    opt, batch, f64, f32 = prepare(case, tmp_path)
    opt.use_cuda_graph = False
    snap = snapshot(opt)
    report = []
    for mutant in MUTANTS[name]:
        restore(opt, snap)
        b = batch
        with monkeypatch.context() as m:
            if mutant == "d_tu":
                orig = ops.ppo_loss_packed

                def scaled(*a, **kw):
                    out = list(orig(*a, **kw))
                    out[3] = out[3] * 0.99
                    return tuple(out)
                m.setattr(ops, "ppo_loss_packed", scaled)
            elif mutant == "swap_h0":
                i, j = case.rows[1], case.rows[2]
                b = batch.map(lambda v: v)
                b.h0 = batch.h0.clone()
                b.h0[:, [i, j]] = batch.h0[:, [j, i]]
                if batch.c0 is not None:
                    b.c0 = batch.c0.clone()
                    b.c0[:, [i, j]] = batch.c0[:, [j, i]]
            elif mutant == "tf32_whh":
                with torch.no_grad():
                    for k in range(case.layers):
                        w = getattr(opt.policy_base.rnn, "weight_hh_l%d" % k)
                        w.copy_(tf32_rna(w))
            else:
                orig_rows = ops._reset_rows
                m.setattr(ops, "_reset_rows", lambda slot, K: (orig_rows(slot, K)[0],
                                                               torch.zeros_like(orig_rows(slot, K)[1])))
            got = gpu_step(opt, b)
        ratios, over = compare(got, f64, f32, case)
        report.append((mutant, [o.split(":")[0] for o in over][:4], old_criterion(got, f64), ratios))
    release(opt)
    print("\n%s mutants: %s" % (name, "; ".join("%s fails bound %s, passes old criterion %s, ratios %s"
                                                 % (m, o, c, {k: round(v, 3) for k, v in r.items()})
                                                 for m, o, c, r in report)))
    assert all(o for _, o, _, _ in report), [m for m, o, _, _ in report if not o]


@pytest.mark.gpu
def test_masked_all_valid_step_is_bitwise_the_unmasked_step(tmp_path):
    """At C2 with every token valid, ``mask_padding=True`` gives the losses, gradients, parameters and Adam moments of the
    unmasked step the benchmark runs (no ``valid``, ``mask_padding=False``), bit for bit."""
    from dotaclient_b200.optimizer import ExperienceBatch
    case = CASE["c2"]
    d = torch.device("cuda", 0)
    f = make_batch(case, 21, d)
    f["valid"] = torch.ones_like(f["valid"])
    f["old_logp"] = -torch.rand(case.S, case.B, 5, device=d) * 3
    bench = dict(clip_range=0.1, max_grad_norm=0.5)               # bench.py's optimizer settings
    masked, plain = make_optimizer(tmp_path, case, **bench), make_optimizer(tmp_path, case, mask_padding=False, **bench)
    assert torch.equal(masked.flat.param, plain.flat.param)
    rm = masked.train(ExperienceBatch(**f))
    rp = plain.train(ExperienceBatch(**dict(f, valid=None)))
    for a, b in zip(rm, rp):
        assert all(torch.equal(torch.as_tensor(a[k]), torch.as_tensor(b[k])) for k in a), (a, b)
    assert masked.last_ppo_stats == plain.last_ppo_stats
    for a, b in ((masked.flat.grad, plain.flat.grad), (masked.flat.param, plain.flat.param),
                 (masked.exp_avg, plain.exp_avg), (masked.exp_avg_sq, plain.exp_avg_sq)):
        assert torch.equal(a, b)
    release(masked)
    release(plain)
