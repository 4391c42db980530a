"""The actor step (``Policy.act_batched``: encoder on ``[1, A]`` tokens, the recurrence at S = 1 with the state carried from
step to step, the packed head GEMM and ``dc_select_actions``) at agent-pool sizes, against ``StackedRefPolicy`` in float64
on the CPU.

The actor's output is used twice by training: its log-probabilities are the ``behaviour_logp`` V-trace divides by, and its
carried state is the ``initial_hidden`` that cut rollouts start prep from.  Agents are independent, so the float64
reference runs only on a sample R of agents: 0, A-1 and the agents on both sides of a batch-tile, cluster or M-tile
boundary of the recurrence design under test.  It steps with its own carried state, and the same reference in fp32
calibrates the bound (``test_gpu_rnn_fp64.bound_check``), per step and per tensor:

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

applied to the five heads' logits, the value, h (and c), and the returned log-probability of every sampled head against the
float64 masked log-softmax at the chosen index.

Sampling is held to the float64 inverse CDF of the float64 logits with the same uniform u.  A pick must be a legal index
whose float64 interval [c_{i-1}, c_i) lies within delta of u; outside a band of width delta around every float64
cumulative boundary that leaves exactly the float64 pick, inside it the two adjacent indices.  delta is twice the
first-order change of the cumulative masses under the row's measured logit error, exp(2 eps) - 1, plus the fp32
rounding of the draw itself (``draw_delta``).  The enum decides the sub-heads (1: x and y, 2: target_unit, 3: ability),
the others must be -1.

``dc_select_actions`` is also called directly on 100003 agents (a ragged last 128-thread block) with the product's pitches
(128 for the four small heads as columns of the packed output, 40 for target_unit) and hard inputs: legal logits up to
|60| and +-1e4 off the mask, single-entry rows, u = 0 and the largest fp32 below 1, and u on and one ulp either side of
the cumulative boundaries ``oracle.ref_policy.sample_index`` computes.

The CPU tests run the same checks on an independent fp32 transcription of the actor step, which passes, and on five
mutants of it, each of which must fail: state not carried, two agents' states swapped between steps, the u of the wrong
head, the log-probability of the neighbouring index, W_hh rounded to TF32.

K is larger than the recurrence's 16 (``test_gpu_rnn_fp64``) because of the dense GEMMs in front of and behind the
recurrence.  ``ops.linear`` (3xTF32 wgmma, documented at about 1e-6 * sum|a||b|) has an error of 6.5e-6 of max|y| at
K = 896 (``affine_pre_rnn``) for every M from 1 to 4096, which is 10x torch fp32's at M 4096 and 30-45x at M <= 8, where
torch's largest error over a few rows is small.  The recurrence passes that input error on (h and c), and the heads add
their own.  The bounds are therefore 1.5 to 2.2 times the largest measured ratio: 256 for the logits and the value, 128
for h and c, 64 for logp, each with a floor of 1e-6 * max|f64|.  They still reject every mutant below: a TF32-rounded
W_hh alone gives ratios of 1000 to 5700.

Measured on one H100 SXM (700 W power limit), T = 8 steps: the largest ratio max|gpu - f64| / max|torch32 - f64| per
case over the steps, logits and value / h and c / logp:
    resident LSTM A 264 / 265 (2- and 4-sequence tiles)     27 / 21 /  8.7,   43 / 26 / 13
    resident GRU  A 265 / 512 (3-sequence tiles)            54 / 36 / 17,     42 / 31 / 13
    cluster GRU   A 1 / 33 / 40 / 1024                     117 / 61 / 25,     80 / 64 / 13,   84 / 50 / 11,   76 / 53 / 29
    step-wise LSTM A 1 / 129 / 300                         173 / 19 / 13,    103 / 16 / 18,   44 / 15 / 18
    generic GRU   A 5 / 40                                 137 / 53 / 14,     47 / 31 /  9.9
    resident LSTM, 2 layers, A 40                           23 / 20 /  3.5
Over all 14 cases, one pick fell in a band and none differed from the float64 pick.  The file runs in 44 s.

``dc_select_actions`` on the hard inputs: max|logp - f64| is 5.8e-6, at most 0.21 of the rounding bound ``draw_delta``.
Every pick lies in its float64 band.  37,094 picks have u inside a band, and 2,773 picks differ from ``sample_index``:
1,155 enum, 425 x, 428 y, 472 target_unit and 293 ability.  All 2,773 are inside the band, and so is
``sample_index``'s own pick.  The kernel and the oracle round exp, log and the normaliser differently (CUDA expf
and a sequential sum against torch's exp and sum), so index selection equals ``sample_index`` only outside the band.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from stacked_oracle import StackedRefPolicy  # noqa: E402
from test_gpu_rnn_fp64 import bound_check, loop_fp32, tf32_rna  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402
from oracle.ref_policy import INPUT_KEYS, UNIT_GROUPS, masked_softmax, sample_index  # noqa: E402

HEADS = ("enum", "x", "y", "target_unit", "ability")
SIZES = (4, 9, 9, 40, 3)
FOLLOW = {0: (), 1: (1, 2), 2: (3,), 3: (4,)}      # enum pick -> the sub-heads it samples (policy.py:203-214)
T = 8
# (K, FLOOR) per kind of output; the dense 3xTF32 GEMMs upstream set K (see above)
HEAD_BOUND = (256.0, 1e-6)     # the five heads' logits and the value
STATE_BOUND = (128.0, 1e-6)    # h, c
LOGP_BOUND = (64.0, 1e-6)      # log-probability of the sampled index

# (case id, cell, H, num_layers, pool size A ("2sm", "2sm+1" or a number))
CASES = [
    # resident, H 128: 2-sequence tiles while (A+1)/2 <= SMs, then 4 (LSTM) / 3 (GRU) with a ragged last tile
    ("resident-lstm-a2sm", "lstm", 128, 1, "2sm"),
    ("resident-lstm-a2sm+1", "lstm", 128, 1, "2sm+1"),
    ("resident-gru-a2sm+1", "gru", 128, 1, "2sm+1"),
    ("resident-gru-a512", "gru", 128, 1, 512),
    # cluster, H 256 (the reference's width and cell): 32 agents per cluster
    ("cluster-gru-a1", "gru", 256, 1, 1),
    ("cluster-gru-a33", "gru", 256, 1, 33),
    ("cluster-gru-a40", "gru", 256, 1, 40),
    ("cluster-gru-a1024", "gru", 256, 1, 1024),
    # step-wise, H 512: 128-row M tiles
    ("stepwise-lstm-a1", "lstm", 512, 1, 1),
    ("stepwise-lstm-a129", "lstm", 512, 1, 129),
    ("stepwise-lstm-a300", "lstm", 512, 1, 300),
    # generic, H 192: 4-sequence CTAs
    ("generic-gru-a5", "gru", 192, 1, 5),
    ("generic-gru-a40", "gru", 192, 1, 40),
    # two resident LSTM layers
    ("resident-2layer-lstm-a40", "lstm", 128, 2, 40),
]


# ------------------------------------------------------------------------------------------------ helpers
def boundary_rows(A, tile):
    """0, A-1 and the agents on both sides of the first tile boundary, one in the middle and the last one."""
    mid = (A // 2) // tile * tile
    last = (A - 1) // tile * tile
    return tuple(sorted({r for r in (0, tile - 1, tile, mid - 1, mid, last - 1, last, A - 1) if 0 <= r < A}))


def make_masks(A, g):
    """Fresh legal masks: about 60 % legal, at least one legal entry per head, target_unit entry 0 never legal; a sixth
    of the rows may only no-op, another sixth has a single legal entry in every sub-head."""
    m = {k: torch.rand(A, n, generator=g) < 0.6 for k, n in zip(HEADS, SIZES)}
    rows = torch.arange(A)
    for k, n in zip(HEADS, SIZES):
        lo = 1 if k == "target_unit" else 0
        m[k][rows, torch.randint(lo, n, (A,), generator=g)] = True
    m["target_unit"][:, 0] = False
    kind = torch.randint(0, 6, (A,), generator=g)
    m["enum"][kind == 0] = torch.tensor([True, False, False, False])
    single = rows[kind == 1]
    for k, n in zip(HEADS[1:], SIZES[1:]):
        lo = 1 if k == "target_unit" else 0
        m[k][single] = False
        m[k][single, torch.randint(lo, n, (len(single),), generator=g)] = True
    return m


def masked_log_softmax64(logits, mask):
    """float64 log-probabilities over the legal entries (-inf elsewhere)."""
    l = logits.double().masked_fill(~mask, -math.inf)
    return l - torch.logsumexp(l, dim=1, keepdim=True)


def draw_delta(logits, mask):
    """Per row: a bound on how far the fp32 draw (``dc_select_actions``, ``sample_index``) can move a cumulative
    boundary of the exact masses: |l - log s| rounds at ulp(max|l| + log n), exp / log / the sums add a few ulp per term."""
    big = logits.double().abs().masked_fill(~mask, 0).amax(1)
    return 4.0 * (2.0 * big + 2.0 * mask.shape[1] + 8.0) * 2.0 ** -24


def allowed_picks(l64, mask, u, delta):
    """-> (allowed [R, n] bool, exact pick [R]): the legal indices whose float64 inverse-CDF interval [c_{i-1}, c_i) lies
    within ``delta`` of u, and the float64 pick itself (the first legal index with c_i > u)."""
    p = torch.exp(masked_log_softmax64(l64, mask))
    c = torch.cumsum(p, dim=1)
    u = u.double()[:, None]
    d = delta.double()[:, None]
    allowed = mask & (c - p - d <= u) & (u < c + d)
    above = mask & (c > u)
    last_legal = (mask.long() * torch.arange(1, mask.shape[1] + 1)).argmax(1)
    exact = torch.where(above.any(1), above.long().argmax(1), last_legal)
    return allowed, exact


def check_sampling(chosen, logits_err, l64, masks, u):
    """Every pick against the float64 inverse CDF -> (failures, number of picks in a band, number that differ from the
    float64 pick).  ``logits_err`` {head: [R]} is the measured max |logit - f64| of each row."""
    failures, in_band, differ = [], 0, 0
    R = chosen.shape[0]
    allow, exact = {}, {}
    for h, k in enumerate(HEADS):
        eps = logits_err[k]
        delta = 2.0 * torch.expm1(2.0 * eps) + draw_delta(l64[k], masks[k])
        allow[h], exact[h] = allowed_picks(l64[k], masks[k], u[:, h], delta)
    for r in range(R):
        e = int(chosen[r, 0])
        for h in range(5):
            pick = int(chosen[r, h])
            if h > 0 and h not in FOLLOW.get(e, ()):
                if pick != -1:
                    failures.append("agent %d: %s = %d where the enum %d does not sample it" % (r, HEADS[h], pick, e))
                continue
            if not 0 <= pick < SIZES[h] or not bool(allow[h][r, pick]):
                failures.append("agent %d: %s = %d, float64 pick %d, allowed %s" % (
                    r, HEADS[h], pick, int(exact[h][r]), allow[h][r].nonzero().flatten().tolist()))
                continue
            in_band += int(allow[h][r].sum()) > 1
            differ += pick != int(exact[h][r])
    return failures, in_band, differ


def check_step(got, chosen, logp, f64, f32, masks, u, cell):
    """One actor step on R: logits, value and state against the bound, the returned log-probabilities against the
    float64 masked log-softmax at the chosen index, the picks against the float64 inverse CDF -> (ratios, failures,
    picks in a band, picks that differ from the float64 pick)."""
    ratios, failures = bound_check(got, f64, f32, HEADS + ("value",), HEAD_BOUND)
    r, over = bound_check(got, f64, f32, ("h", "c") if cell == "lstm" else ("h",), STATE_BOUND)
    ratios.update(r)
    failures += over
    lp = {"gpu": [], "f64": [], "f32": []}
    for h, k in enumerate(HEADS):
        sel = chosen[:, h] >= 0
        if not bool(sel.any()):
            continue
        idx = chosen[sel, h].long()[:, None]
        lp["gpu"].append(logp[sel, h].double())
        lp["f64"].append(masked_log_softmax64(f64[k][sel], masks[k][sel]).gather(1, idx)[:, 0])
        l32 = masked_softmax(f32[k][sel].float(), masks[k][sel], dim=1)
        lp["f32"].append(l32.gather(1, idx)[:, 0].double())
    lp = {n: {"logp": torch.cat(v)} for n, v in lp.items()}
    r, over = bound_check(lp["gpu"], lp["f64"], lp["f32"], ("logp",), LOGP_BOUND)
    ratios.update(r)
    failures += over
    err = {k: (got[k].double() - f64[k]).abs().masked_fill(~masks[k], 0).amax(1) for k in HEADS}
    fails, in_band, differ = check_sampling(chosen, err, f64, masks, u)
    return ratios, failures + fails, in_band, differ


def reference_step(ref, obs, hidden):
    """One step of ``StackedRefPolicy`` on the agents of ``obs`` ({key: [R, ...]}) -> (outputs, new hidden)."""
    dt = next(ref.parameters()).dtype
    with torch.no_grad():
        logits, value, hidden = ref(**{k: v.to(dt)[:, None] for k, v in obs.items()}, hidden=hidden)
    out = {k: v[:, 0] for k, v in logits.items()}
    out["value"] = value[:, 0, 0]
    h, c = hidden if isinstance(hidden, tuple) else (hidden, None)
    out["h"] = h
    if c is not None:
        out["c"] = c
    return out, hidden


def draw_fp32(logits, mask, u):
    """The kernel's draw restated in fp32 (masked log-softmax without max-subtraction, sequential inverse CDF) for rows of
    one head -> (pick [R], logp [R])."""
    l = logits.float().numpy()
    m = mask.numpy()
    R, n = l.shape
    picks, lps = np.full(R, -1, np.int64), np.zeros(R, np.float32)
    for r in range(R):
        s = np.float32(0)
        for i in range(n):
            if m[r, i]:
                s = np.float32(s + np.exp(l[r, i]))
        log_s = np.log(s)
        p = np.where(m[r], np.exp(l[r] - log_s), np.float32(0)).astype(np.float32)
        total = np.float32(0)
        for i in range(n):
            total = np.float32(total + p[i])
        target, acc = np.float32(np.float32(u[r]) * total), np.float32(0)
        for i in range(n):
            if not m[r, i]:
                continue
            picks[r] = i
            acc = np.float32(acc + p[i])
            if acc > target:
                break
        lps[r] = l[r, picks[r]] - log_s if picks[r] >= 0 else 0
    return picks, lps


def transcribed_step(sd, cell, L, obs, hidden, masks, u, mutant=None):
    """The actor step in fp32, written out from the network's equations (encoder, L cell steps, heads) and the kernel's
    draw: an implementation independent of the reference modules.  ``mutant``: 'tf32' (W_hh rounded to TF32), 'u' (each
    head draws with the next head's u), 'logp' (the log-probability of the neighbouring index)."""
    def lin(x, name):
        return x @ sd[name + ".weight"].float().t() + sd[name + ".bias"].float()
    embs, maxes = [], {}
    for suffix, key, _ in UNIT_GROUPS:
        basic = torch.relu(lin(obs[key].float(), "affine_unit_basic_stats"))
        embs.append(lin(basic, "affine_unit_" + suffix))
        maxes[suffix] = embs[-1].amax(1)
    maxes["eth"] = maxes["enh"]            # the reference takes the enemy-tower max from the enemy-nonhero embedding
    x = torch.cat([torch.relu(lin(obs["env"].float(), "affine_env"))] + [maxes[s] for s, _, _ in UNIT_GROUPS], 1)
    x = torch.relu(lin(x, "affine_pre_rnn"))
    h0, c0 = hidden if cell == "lstm" else (hidden, None)
    hs, cs = [], []
    for k in range(L):
        w = {n + "_l0": sd["rnn.%s_l%d" % (n, k)].float() for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")}
        if mutant == "tf32":
            w["weight_hh_l0"] = tf32_rna(w["weight_hh_l0"])
        out = loop_fp32(cell, w, x[None], h0[k], c0[k] if cell == "lstm" else None)
        x = out["h_n"]
        hs.append(out["h_n"])
        cs.append(out.get("c_n"))
    att = lin(x, "affine_unit_attention")
    logits = {"enum": lin(x, "affine_head_enum"), "x": lin(x, "affine_move_x"), "y": lin(x, "affine_move_y"),
              "target_unit": (torch.cat(embs, 1) * att[:, None, :]).sum(-1), "ability": lin(x, "affine_head_ability")}
    got = dict(logits, value=lin(x, "affine_value")[:, 0], h=torch.stack(hs))
    if cell == "lstm":
        got["c"] = torch.stack(cs)
    R = x.shape[0]
    chosen, logp = torch.full((R, 5), -1, dtype=torch.int64), torch.zeros(R, 5)
    for h, k in enumerate(HEADS):
        uh = u[:, (h + 1) % 5] if mutant == "u" else u[:, h]
        pick, lp = draw_fp32(logits[k], masks[k], uh.numpy())
        if mutant == "logp":
            nxt = (pick + 1) % SIZES[h]
            lp = (logits[k] - torch.log((torch.exp(logits[k]) * masks[k]).sum(1, keepdim=True))).gather(
                1, torch.from_numpy(nxt)[:, None])[:, 0].numpy()
        sampled = torch.ones(R, dtype=torch.bool) if h == 0 else torch.tensor(
            [h in FOLLOW.get(int(e), ()) for e in chosen[:, 0]])
        chosen[sampled, h] = torch.from_numpy(pick)[sampled]
        logp[sampled, h] = torch.from_numpy(lp)[sampled]
    new_hidden = (got["h"], got["c"]) if cell == "lstm" else got["h"]
    return got, chosen, logp, new_hidden


def pool_inputs(A, rows, seed):
    """Observations of ``make_rollout`` ([T, A, ...] per key), masks and uniforms of every step, and the initial state."""
    rolls = [make_rollout(T, seed + a) for a in range(A)]
    obs = {k: torch.stack([r["observations"][k] for r in rolls], 1) for k in INPUT_KEYS}
    g = torch.Generator().manual_seed(seed)
    masks = [make_masks(A, g) for _ in range(T)]
    u = [torch.rand(A, 5, generator=g) for _ in range(T)]
    return obs, masks, u, g


def make_reference(H, cell, L, seed=7):
    torch.manual_seed(seed)
    return StackedRefPolicy(H, cell, L)


def run_reference(ref32, obs, rows, hidden0, cell):
    """The float64 and fp32 reference on R over T steps -> ([f64 outputs per step], [f32 outputs per step])."""
    ref64 = make_reference(ref32.hidden_size, cell, ref32.num_layers)
    ref64.load_state_dict(ref32.state_dict())
    ref64.double()
    idx = torch.tensor(rows)
    outs = {torch.float64: [], torch.float32: []}
    for ref, dt in ((ref64, torch.float64), (ref32, torch.float32)):
        hid = tuple(x[:, idx].to(dt) for x in hidden0) if cell == "lstm" else hidden0[:, idx].to(dt)
        for t in range(T):
            o, hid = reference_step(ref, {k: v[t, idx] for k, v in obs.items()}, hid)
            outs[dt].append(o)
    return outs[torch.float64], outs[torch.float32]


def initial_hidden(L, A, H, cell, g):
    h = torch.randn(L, A, H, generator=g) * 0.5
    return (h, torch.randn(L, A, H, generator=g) * 0.5) if cell == "lstm" else h


def summarise(ratios_per_step, cell):
    """Largest ratio over the steps: logits and value / h and c / logp."""
    groups = ((HEADS + ("value",)), ("h", "c") if cell == "lstm" else ("h",), ("logp",))
    return tuple(max(r[n] for r in ratios_per_step for n in grp) for grp in groups)


# ------------------------------------------------------------------------------------------------ CPU: the checks themselves
def _transcription_run(cell, L, mutant=None):
    H, R = 64, 8
    ref32 = make_reference(H, cell, L, seed=11)
    sd = {k: v.detach() for k, v in ref32.state_dict().items()}
    rows = tuple(range(R))
    obs, masks, u, g = pool_inputs(R, rows, 900 + L)
    hidden0 = initial_hidden(L, R, H, cell, g)
    f64, f32 = run_reference(ref32, obs, rows, hidden0, cell)
    hid = hidden0
    failures, ratios = [], []
    for t in range(T):
        if mutant == "no-carry" and t > 0:
            hid = tuple(torch.zeros_like(x) for x in hid) if cell == "lstm" else torch.zeros_like(hid)
        got, chosen, logp, hid = transcribed_step(sd, cell, L, {k: v[t] for k, v in obs.items()}, hid, masks[t], u[t],
                                                  mutant)
        r, f, _, _ = check_step(got, chosen, logp, f64[t], f32[t], masks[t], u[t], cell)
        ratios.append(r)
        failures += ["step %d: %s" % (t, s) for s in f]
        if mutant == "swap":
            perm = torch.tensor([1, 0] + list(range(2, R)))
            hid = tuple(x[:, perm] for x in hid) if cell == "lstm" else hid[:, perm]
    return failures, ratios


@pytest.mark.parametrize("cell,L", [("gru", 1), ("lstm", 1), ("lstm", 2)])
def test_transcription_passes_the_checks(cell, L):
    """An independent fp32 actor step passes the bound, the log-probability check and the sampling check."""
    failures, ratios = _transcription_run(cell, L)
    assert not failures, failures
    print("\ntranscription %s L%d: logits/value %.3g, state %.3g, logp %.3g" % ((cell, L) + summarise(ratios, cell)))


@pytest.mark.parametrize("mutant", ["no-carry", "swap", "u", "logp", "tf32"])
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_mutants_fail_the_checks(cell, mutant):
    """State not carried, two agents' states swapped between steps, the u of the wrong head, the log-probability of the
    neighbouring index, W_hh rounded to TF32: each must fail."""
    failures, _ = _transcription_run(cell, 1, mutant)
    assert failures, "the %s mutant passed" % mutant


def test_sampling_band_on_the_cpu():
    """The band logic: u exactly on a float64 boundary admits both neighbours, u outside every band only the float64 pick,
    and an index whose mass underflows in fp32 is admitted only while u is within delta of its interval."""
    l = torch.tensor([[0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0], [-60.0, -60.0, 0.0, 60.0]], dtype=torch.float64)
    m = torch.ones(3, 4, dtype=torch.bool)
    u = torch.tensor([0.5, 0.6, 0.0], dtype=torch.float64)
    allowed, exact = allowed_picks(l, m, u, torch.full((3,), 1e-6, dtype=torch.float64))
    assert allowed[0].tolist() == [False, True, True, False] and exact[0] == 2
    assert allowed[1].tolist() == [False, False, True, False] and exact[1] == 2
    assert allowed[2].tolist() == [True, True, True, True] and exact[2] == 0
    allowed, _ = allowed_picks(l, m, torch.tensor([0.5, 0.6, 0.3], dtype=torch.float64), torch.full((3,), 1e-6, dtype=torch.float64))
    assert allowed[2].tolist() == [False, False, False, True]


# ------------------------------------------------------------------------------------------------ GPU
def _sm_count():
    import ctypes
    from dotaclient_b200 import _lib
    sm, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().dc_device_info(ctypes.byref(sm), ctypes.byref(major), ctypes.byref(minor)), "dc_device_info")
    return sm.value


def _tile(cell, H, A, sm):
    """Agents per CTA, cluster or M tile of the recurrence design that runs width H."""
    if H == 128:
        return 2 if (A + 1) // 2 <= sm else (3 if cell == "gru" else 4)
    return {256: 32, 512: 128}.get(H, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_act_batched_vs_fp64(case):
    """T consecutive act_batched steps with the state carried: logits, value, state and log-probabilities of the agents
    in R against the float64 reference, and every pick against the float64 inverse CDF."""
    from dotaclient_b200.policy import Policy
    name, cell, H, L, A = case
    sm = _sm_count()
    A = {"2sm": 2 * sm, "2sm+1": 2 * sm + 1}.get(A, A)
    rows = boundary_rows(A, _tile(cell, H, A, sm))
    d = torch.device("cuda", 0)
    ref32 = make_reference(H, cell, L)
    policy = Policy(hidden_size=H, cell=cell, num_layers=L)
    policy.load_state_dict(ref32.state_dict())
    policy.to(d)
    obs, masks, u, g = pool_inputs(A, rows, 1000 * H + A)
    hidden0 = initial_hidden(L, A, H, cell, g)
    f64, f32 = run_reference(ref32, obs, rows, hidden0, cell)

    idx = torch.tensor(rows, device=d)
    hid = tuple(x.to(d) for x in hidden0) if cell == "lstm" else hidden0.to(d)
    failures, ratios, in_band, differ = [], [], 0, 0
    for t in range(T):
        chosen, logp, logits, value, hid = policy.act_batched(
            hid, {k: v[t].to(d) for k, v in obs.items()}, {k: v.to(d) for k, v in masks[t].items()}, u[t].to(d))
        got = {k: logits[k].index_select(0, idx).cpu() for k in HEADS}
        got["value"] = value.index_select(0, idx).cpu()
        hs, cs = hid if cell == "lstm" else (hid, None)
        got["h"] = hs.index_select(1, idx).cpu()
        if cell == "lstm":
            got["c"] = cs.index_select(1, idx).cpu()
        ch = torch.stack([chosen[k] for k in HEADS], 1).index_select(0, idx).cpu().long()
        for k in HEADS:
            if not torch.isfinite(logits[k]).all():
                failures.append("step %d: %s logits are not finite" % (t, k))
        r, f, b, dif = check_step(got, ch, logp.index_select(0, idx).cpu(), f64[t], f32[t],
                                  {k: v[list(rows)] for k, v in masks[t].items()}, u[t][list(rows)], cell)
        ratios.append(r)
        failures += ["step %d: %s" % (t, s) for s in f]
        in_band += b
        differ += dif
    print("\n%s (A %d, R %s): logits/value %.3g, state %.3g, logp %.3g; picks in a band %d, differing from float64 %d" % (
        (name, A, rows) + summarise(ratios, cell) + (in_band, differ)))
    assert not failures, failures


def _oracle_cumulative(logits, mask):
    """The fp32 total and cumulative masses ``sample_index`` computes for one row: [(index, acc)] over the legal entries."""
    lp = masked_softmax(logits.view(1, 1, -1), mask.view(1, 1, -1)).view(-1)
    probs = torch.exp(lp).clone()
    probs[~mask.view(-1)] = 0.0
    total, acc, out = np.float32(0.0), np.float32(0.0), []
    for p in probs.numpy():
        total = np.float32(total + p)
    for i, p in enumerate(probs.numpy()):
        if bool(mask[i]):
            acc = np.float32(acc + p)
            out.append((i, acc))
    return total, out


@pytest.mark.gpu
def test_select_actions_hard_inputs_vs_fp64():
    """``dc_select_actions`` on 100003 agents with the product's pitches and hard inputs: no illegal pick and no -1 on a
    row with a legal entry, every pick inside the float64 band, logp against float64, and the picks that differ from
    ``sample_index`` counted (all of them inside the band)."""
    from dotaclient_b200 import ops
    A = 100003
    g = torch.Generator().manual_seed(17)
    one_below = float(np.nextafter(np.float32(1), np.float32(0)))
    kind = torch.arange(A) % 8      # 0-2 random, 3 single-entry rows, 4 u = 0, 5 u = 1 - 2^-24, 6-7 u on boundaries
    scale = torch.tensor([0.5, 4.0, 20.0, 60.0])[torch.randint(0, 4, (A,), generator=g)]
    masks, logits = {}, {}
    for k, n in zip(HEADS, SIZES):
        lo = 1 if k == "target_unit" else 0
        m = torch.rand(A, n, generator=g) < 0.5
        m[torch.arange(A), torch.randint(lo, n, (A,), generator=g)] = True
        single = kind == 3
        m[single] = False
        m[single.nonzero()[:, 0], torch.randint(lo, n, (int(single.sum()),), generator=g)] = True
        m[:, 0] = m[:, 0] & (k != "target_unit")
        masks[k] = m
    # rows of kind 7 draw a sub-head: their enum has one legal entry in 1..3
    seven = (kind == 7).nonzero()[:, 0]
    masks["enum"][seven] = False
    masks["enum"][seven, torch.randint(1, 4, (len(seven),), generator=g)] = True
    for k, n in zip(HEADS, SIZES):
        l = (torch.rand(A, n, generator=g) * 2 - 1) * scale[:, None]
        off = torch.where(torch.rand(A, n, generator=g) < 0.5, 1e4, -1e4)
        logits[k] = torch.where(masks[k], l, off)
    u = torch.rand(A, 5, generator=g)
    u[kind == 4] = 0.0
    u[kind == 5] = one_below
    # u on, and one ulp either side of, a cumulative boundary of sample_index: the enum's on kind 6, the sub-heads' on 7
    n_boundary = 0
    for a in (kind >= 6).nonzero()[:, 0].tolist():
        heads = (0,) if kind[a] == 6 else FOLLOW[int(masks["enum"][a].nonzero()[0, 0])]
        for h in heads:
            total, cum = _oracle_cumulative(logits[HEADS[h]][a], masks[HEADS[h]][a])
            if len(cum) < 2:
                continue
            _, acc = cum[int(torch.randint(0, len(cum) - 1, (1,), generator=g))]
            b = np.float32(acc / total)
            b = [np.nextafter(b, np.float32(0)), b, np.nextafter(b, np.float32(1))][(a // 8) % 3]
            u[a, h] = float(min(max(b, np.float32(0)), np.float32(one_below)))
            n_boundary += 1
    assert n_boundary > A // 8

    d = torch.device("cuda", 0)
    packed = torch.zeros(A, ops.PACK_WIDTH)
    for k in ("enum", "x", "y", "ability"):
        c0, c1 = ops.PACK_COLS[k]
        packed[:, c0:c1] = logits[k]
    packed = packed.to(d)
    tu = logits["target_unit"].to(d)
    views = [packed[:, slice(*ops.PACK_COLS[k])] if k != "target_unit" else tu for k in HEADS]
    assert all(v.stride(0) == (40 if k == "target_unit" else 128) for k, v in zip(HEADS, views))
    chosen, logp = ops.select_actions(views, [masks[k].to(d) for k in HEADS], u.to(d))
    chosen, logp = chosen.cpu().long(), logp.cpu()

    failures = []
    allow, exact = {}, {}
    for h, k in enumerate(HEADS):
        allow[h], exact[h] = allowed_picks(logits[k].double(), masks[k], u[:, h], draw_delta(logits[k], masks[k]))
    e = chosen[:, 0]
    sampled = torch.zeros(A, 5, dtype=torch.bool)
    sampled[:, 0] = True
    for h in range(1, 5):
        sampled[:, h] = torch.tensor([h in FOLLOW[v] for v in range(4)])[e.clamp(0, 3)]
    if bool((e < 0).any()):
        failures.append("%d enum picks are -1" % int((e < 0).sum()))
    for h, k in enumerate(HEADS):
        pick = chosen[:, h]
        if bool((pick[~sampled[:, h]] != -1).any()):
            failures.append("%s picked where the enum does not sample it" % k)
        s = sampled[:, h] & (e >= 0)
        p = pick[s]
        if bool(((p < 0) | (p >= SIZES[h])).any()):
            failures.append("%s: %d picks are -1 or out of range on rows with a legal entry" % (k, int(((p < 0) | (p >= SIZES[h])).sum())))
            continue
        rows = s.nonzero()[:, 0]
        if not bool(masks[k][rows, p].all()):
            failures.append("%s: %d illegal picks" % (k, int((~masks[k][rows, p]).sum())))
        out = ~allow[h][rows, p]
        if bool(out.any()):
            failures.append("%s: %d picks outside the float64 band, e.g. row %d" % (k, int(out.sum()), int(rows[out][0])))
        lp64 = masked_log_softmax64(logits[k][rows], masks[k][rows]).gather(1, p[:, None])[:, 0]
        tol = draw_delta(logits[k][rows], masks[k][rows])
        err = (logp[rows, h].double() - lp64).abs()
        if bool((err > tol).any()):
            failures.append("%s: logp off by %.3e (tolerance %.3e)" % (k, float(err.max()), float(tol[err.argmax()])))
        print("\n%s: max |logp - f64| %.3e, max ratio to its tolerance %.3g" % (k, float(err.max()), float((err / tol).max())))

    # the picks that differ from sample_index, on every sampled head of every row
    differ, in_band = {k: 0 for k in HEADS}, {k: 0 for k in HEADS}
    for a in range(A):
        for h in sampled[a].nonzero()[:, 0].tolist():
            k = HEADS[h]
            band = int(allow[h][a].sum()) > 1
            in_band[k] += band
            want = sample_index(logits[k][a], masks[k][a], float(u[a, h]))
            if want != int(chosen[a, h]):
                differ[k] += 1
                if not (band and bool(allow[h][a, want])):
                    failures.append("row %d %s: kernel %d, sample_index %d, outside the band" % (a, k, int(chosen[a, h]), want))
    print("picks in a band: %s; differing from sample_index: %s" % (in_band, differ))
    assert not failures, failures[:20]
