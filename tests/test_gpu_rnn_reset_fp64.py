"""The recurrence with state resets inside a sequence (``ops.rnn_sequence(reset=...)``: the reset rows' h2h GEMM,
``dc_rnn_seq_fwd_reset`` / ``dc_rnn_seq_bwd_reset`` and the dW_hh reset correction of ``ops.RnnSequence.backward``) on
every recurrence design, at the shapes the benchmark runs and at their tile edges, against a float64 reference.

This is what packed training batches (``pack_sequences=True``) run.  The reference is
``test_gpu_packing.segmented_reference``: torch's CPU GRU / LSTM runs every segment of a column on its own, from h0 / c0
or from its reset's table row.  As in ``test_gpu_rnn_fp64``, it runs on a sample R of 8 rows on both sides of the
design's batch-tile, cluster or M-tile edges, once in float64 and once in float32 to calibrate the bound, and the bounds
are that file's: max|gpu - f64| <= k * max|torch32 - f64| + floor * max|f64|, per tensor (K below is the
number of rows of the reset tables, the most resets in one column).

Every sampled row carries its own reset pattern: none, t = 0 only (h0 / c0 never read), t = 1 and S-1, a consecutive
pair mid-sequence, t = S-1 only, every 16th step, a pair early in the sequence and every 16th step at another phase.
Every other column cycles through the same patterns, so every column but the pattern-free ones restarts at least once.
At S = 1 every pattern but the first is a reset at t = 0.  Two more layouts: the packed layout of
``optimizer.pack_layout`` on seeded ragged rollout lengths (R holds the layout's seven most-reset columns and one full
chunk; K reaches 74 at S 512 and 101 at S 1024), and a dense one where one pattern resets at every step t >= 1
(K = S - 1), which makes the reset-row GEMM and the dW_hh correction run over (S - 1) * B rows.  Table states are drawn
at 0.5 N(0, 1).

The bound is shown to catch what it is meant to, once per design: a forward with W_hh rounded to TF32, a forward with
the slot table shifted one step later, and one with the table rows rolled by one column must fail the forward bound, and
a backward without the dW_hh reset correction must fail the bound on weight_hh_l0.  ``test_bound_logic_on_the_cpu``
checks the reference itself against a step-by-step float64 transcription of the cell equations.

Measured on one H100 80GB HBM3 (700 W power limit), the largest ratio max|gpu - f64| / max|torch32 - f64| per group of
cases, forward / state gradients / weight gradients (the weight gradients as max|gpu - f64| / max|f64| in brackets), and
the TF32-rounded forward's ratios last:
    resident  B 256 / 512, S 512                    3.8 /  4.5 / 13  (5.3e-6)   TF32 153-232
    resident  S 1 / S 3                             6.5 /  5.6 / 4.6 (7.5e-7)   TF32 209-585
    cluster   B 512 / 500, S 512                    5.3 / 13   / 20  (1.0e-5)   TF32 122-147
    cluster   B 33, S 1                             3.2 / 12   / 2.3 (1.3e-6)   TF32 175
    step-wise B 512 S 1024 / B 300 S 256            7.1 / 21   / 8.7 (4.7e-6)   TF32 120-143
    step-wise B 129, S 1                            5.0 / 24   / 4.9 (3.1e-6)   TF32 116
    generic   B 256 S 512 / B 5 S 2                 6.6 /  5.6 / 7.0 (3.8e-6)   TF32 224-516
    saturating inputs (H 128 LSTM / H 256 GRU)      3.3 /  9.2 / 7.5 (4.1e-5)
    packed layouts C2 (K 74) / C4 (K 101)           4.6 / 20   / 4.8 (3.9e-6)   TF32 73-136
    dense resets, resident GRU (K 511) /
      step-wise LSTM (K 1023)                       5.2 / 23   / 12  (4.7e-6)   TF32 108-185
They stay within a factor of 1.5 of what ``test_gpu_rnn_fp64`` measures at the same shapes without resets.  The
tightest margins: the state gradients of step-wise B 129 at 24 of the bound's 32 (22 without resets), the saturating
LSTM's weight gradients at 4.1e-5 of the 1e-4 floor, and the superposition residual at 4.8e-6 of max|dW| against 5e-5.
The smallest TF32 ratio, 73 (packed layout C4), clears the forward bound's 16 by a factor of 4.5.  The other mutants
fail by far more: the shifted slot table and the rolled table rows reach forward ratios of 1.8e5 and above, the
backward without the reset correction a weight_hh_l0 ratio of 7.9e4 and above.
"""
import numpy as np
import pytest
import torch

from test_gpu_packing import segmented_reference
from test_gpu_rnn_fp64 import (FORWARD_BOUND, STATE_GRAD_BOUND, SUPERPOSE, WEIGHT_GRAD_BOUND, WEIGHTS, _rows, bound_check,
                               forward_names, make_weights, state_grad_names, tf32_rna)

R256 = (0, 1, 2, 127, 128, 129, 254, 255)
R512 = (0, 127, 128, 255, 256, 383, 384, 511)
# (case id, cell, B, S, H, sampled rows R, saturating inputs, reset layout, sensitivity runs)
CASES = [
    # resident, H 128: 2-sequence tiles (B <= 264) on 128 CTAs; 3-sequence (GRU) / 4-sequence (LSTM) tiles above
    ("resident-b256-gru", "gru", 256, 512, 128, R256, False, "patterns", True),
    ("resident-b256-lstm", "lstm", 256, 512, 128, R256, False, "patterns", True),
    ("resident-b512-gru", "gru", 512, 512, 128, (0, 2, 3, 254, 255, 509, 510, 511), False, "patterns", True),
    ("resident-b512-lstm", "lstm", 512, 512, 128, (0, 3, 4, 255, 256, 259, 508, 511), False, "patterns", True),
    # fewer steps than the kStages = 4 prefetch ring, and resets at t = 0 of a 1-step sequence
    ("resident-s1-gru", "gru", 256, 1, 128, R256, False, "patterns", True),
    ("resident-s1-lstm", "lstm", 256, 1, 128, R256, False, "patterns", True),
    ("resident-s3-gru", "gru", 256, 3, 128, R256, False, "patterns", True),
    ("resident-s3-lstm", "lstm", 256, 3, 128, R256, False, "patterns", True),
    # cluster, H 256: 32 sequences per 8-CTA cluster; 16 clusters, and a last cluster holding 20 of its 32 rows
    ("cluster-b512-gru", "gru", 512, 512, 256, (0, 31, 32, 255, 256, 480, 481, 511), False, "patterns", True),
    ("cluster-b512-lstm", "lstm", 512, 512, 256, (0, 31, 32, 255, 256, 480, 481, 511), False, "patterns", True),
    ("cluster-b500-gru", "gru", 500, 512, 256, (0, 31, 32, 255, 256, 479, 480, 499), False, "patterns", True),
    ("cluster-b33-s1-lstm", "lstm", 33, 1, 256, (0, 1, 30, 31, 32), False, "patterns", True),
    # step-wise, H 512: 128-row M tiles of the per-step split-K GEMM; C4's B 512 x S 1024, a ragged last M tile, and
    # row 128 alone in its tile
    ("stepwise-b512-lstm", "lstm", 512, 1024, 512, R512, False, "patterns", True),
    ("stepwise-b300-gru", "gru", 300, 256, 512, (0, 127, 128, 255, 256, 257, 298, 299), False, "patterns", True),
    ("stepwise-b129-s1-lstm", "lstm", 129, 1, 512, (0, 1, 126, 127, 128), False, "patterns", True),
    # generic, H 192: 4-sequence CTAs
    ("generic-b256-lstm", "lstm", 256, 512, 192, (0, 3, 4, 127, 128, 131, 252, 255), False, "patterns", True),
    ("generic-b5-s2-gru", "gru", 5, 2, 192, (0, 3, 4), False, "patterns", True),
    # saturated gates (|pre-activation| 30..100) and an LSTM forget bias of +5
    ("saturating-h128-lstm", "lstm", 256, 512, 128, R256, True, "patterns", False),
    ("saturating-h256-gru", "gru", 256, 512, 256, (0, 31, 32, 127, 128, 224, 225, 255), True, "patterns", False),
    # the slot tables of packed batches: C2 on the resident design, C4 on the step-wise one
    ("packed-layout-c2", "lstm", 256, 512, 128, R256, False, "packed", True),
    ("packed-layout-c4", "lstm", 512, 1024, 512, R512, False, "packed", True),
    # one pattern resets at every step t >= 1: K = S - 1
    ("dense-resets-resident-gru", "gru", 256, 512, 128, R256, False, "dense", True),
    ("dense-resets-stepwise-lstm", "lstm", 512, 1024, 512, R512, False, "dense", True),
]
PATTERNS = ("none", "t0", "first-last", "pair", "last", "every16", "pair-early", "every16-late")


# ------------------------------------------------------------------------------------------------ reset layouts
def pattern_steps(name, S):
    """The steps at which a column of S steps with pattern ``name`` resets.  Steps past the sequence are dropped, and a
    pattern other than 'none' left with no step resets at t = S-1 instead."""
    ts = {"none": [], "t0": [0], "first-last": [1, S - 1], "pair": [S // 2, S // 2 + 1], "last": [S - 1],
          "every16": range(16, S, 16), "pair-early": [2, 3], "every16-late": range(7, S, 16), "dense": range(1, S)}[name]
    ts = sorted({t for t in ts if t < S})
    return ts if ts or name == "none" else [S - 1]


def packed_slots(S, seed):
    """``reset_slot`` of ``optimizer.pack_layout`` on seeded ragged lengths: a few rollouts longer than S (full chunks and
    long tails), and many short ones whose tails pack dozens to a column."""
    from dotaclient_b200.optimizer import pack_layout
    rng = np.random.default_rng(seed)
    lengths = np.concatenate([rng.integers(S + 1, 3 * S, 4), rng.integers(1, S // 4, 60), rng.integers(1, S // 32, 300)])
    rng.shuffle(lengths)
    return pack_layout(lengths.tolist(), S).reset_slot


def reset_slots(layout, S, B, rows, seed):
    """-> (reset_slot [S, B] int32, K).  'patterns' / 'dense': sampled row i carries pattern i of PATTERNS ('dense'
    replaces the last), every other column b pattern b % 8.  'packed': the sampled rows carry the packed layout's seven
    most-reset columns and one column without resets, every other column b the layout's column b % B'."""
    if layout == "packed":
        lay = packed_slots(S, seed)
        n = (lay >= 0).sum(0)
        order = np.argsort(-n, kind="stable")
        cols = np.arange(B) % lay.shape[1]
        cols[list(rows)] = list(order[:len(rows) - 1]) + [int(np.flatnonzero(n == 0)[0])]
        slot = np.ascontiguousarray(lay[:, cols])
    else:
        names = PATTERNS[:-1] + ("dense",) if layout == "dense" else PATTERNS
        col = [names[b % len(names)] for b in range(B)]
        for i, b in enumerate(rows):
            col[b] = names[i]
        slot = np.full((S, B), -1, dtype=np.int32)
        for b, name in enumerate(col):
            for k, t in enumerate(pattern_steps(name, S)):
                slot[t, b] = k
    return slot, int(slot.max()) + 1


# ------------------------------------------------------------------------------------------------ CPU: the reference itself
def transcription(cell, w, x, h0, c0, slot, h_tab, c_tab, dy, dhn, dcn, drop_correction=False):
    """float64, every column at once, step by step from the cell equations: at a token with ``slot[t, b] = k >= 0`` the
    state entering step t is row (k, b) of the tables.  Outputs and the gradients of <y, dy> + <h_n, dhn> (+ <c_n, dcn>).
    ``drop_correction``: at a reset token W_hh's gradient pairs dgh with the carried state instead of the table row (what
    dW_hh is without the reset correction of ``ops.RnnSequence.backward``) while the value keeps the table row."""
    S, B, H = x.shape
    p = {k: w[k].double().clone().requires_grad_(True) for k in WEIGHTS}
    xr, h0r = x.double().requires_grad_(True), h0.double().requires_grad_(True)
    c0r = c0.double().requires_grad_(True) if cell == "lstm" else None
    w_ih, w_hh, b_ih, b_hh = (p[k] for k in WEIGHTS)
    cols = torch.arange(B)
    h, c, ys = h0r, c0r, []
    for t in range(S):
        reset = torch.from_numpy(slot[t] >= 0)[:, None]
        k = torch.from_numpy(np.maximum(slot[t], 0)).long()
        hp = torch.where(reset, h_tab.double()[k, cols], h)
        gi = xr[t] @ w_ih.t() + b_ih
        gh = hp @ w_hh.t() + b_hh
        if drop_correction:
            stale = h.detach() @ w_hh.t()
            gh = torch.where(reset, hp @ w_hh.detach().t() + b_hh + (stale - stale.detach()), gh)
        if cell == "gru":
            r = torch.sigmoid(gi[:, :H] + gh[:, :H])
            z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
            n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
            h = (1 - z) * n + z * hp
        else:
            cp = torch.where(reset, c_tab.double()[k, cols], c)
            g = gi + gh
            c = torch.sigmoid(g[:, H:2 * H]) * cp + torch.sigmoid(g[:, :H]) * torch.tanh(g[:, 2 * H:3 * H])
            h = torch.sigmoid(g[:, 3 * H:]) * torch.tanh(c)
        ys.append(h)
    y = torch.stack(ys)
    loss = (y * dy.double()).sum() + (h * dhn.double()).sum() + ((c * dcn.double()).sum() if cell == "lstm" else 0.0)
    loss.backward()
    zero = torch.zeros_like(h0r)
    out = {"y": y.detach(), "h_n": h.detach(), "dx": xr.grad, "dh0": zero if h0r.grad is None else h0r.grad}
    if cell == "lstm":
        out.update(c_n=c.detach(), dc0=zero if c0r.grad is None else c0r.grad)
    out.update({k: p[k].grad for k in WEIGHTS})
    return out


@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_bound_logic_on_the_cpu(cell):
    """``segmented_reference`` in float64 equals the step-by-step transcription with resets (every pattern, the dense one
    included); the transcription without the dW_hh reset correction fails the weight-gradient bound on weight_hh_l0 and
    nothing else."""
    S, B, H = 40, 8, 32
    w = make_weights(cell, H, 5, False)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(S, B, H, generator=g)
    h0, c0 = 0.5 * torch.randn(B, H, generator=g), 0.5 * torch.randn(B, H, generator=g)
    slot, K = reset_slots("dense", S, B, tuple(range(B)), 0)
    h_tab, c_tab = 0.5 * torch.randn(K, B, H, generator=g), 0.5 * torch.randn(K, B, H, generator=g)
    dy, dhn, dcn = torch.randn(S, B, H, generator=g), torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
    args = (cell, w, x, h0, c0, slot, h_tab, c_tab, dy, dhn, dcn)
    f64, f32 = segmented_reference(*args, torch.float64), segmented_reference(*args, torch.float32)
    full, dropped = transcription(*args), transcription(*args, drop_correction=True)
    for n in forward_names(cell) + state_grad_names(cell) + WEIGHTS:
        scale = float(f64[n].abs().max())
        assert float((full[n] - f64[n]).abs().max()) <= 1e-12 * scale, n
        if n != "weight_hh_l0":
            assert float((dropped[n] - f64[n]).abs().max()) <= 1e-12 * scale, n
    _, over = bound_check(dropped, f64, f32, WEIGHTS, WEIGHT_GRAD_BOUND)
    assert [o.split(":")[0] for o in over] == ["weight_hh_l0"], over
    assert bool((f64["dh0"][torch.from_numpy(slot[0] >= 0)] == 0).all())


def test_reset_layouts_cover_the_sampled_rows():
    """Every case's layout: the sampled rows carry pairwise different reset steps (where S leaves room for them), every
    column restarts at least once except the pattern-free ones, the dense layout has K = S - 1, and most sampled rows of a
    packed layout restart."""
    for name, _, B, S, _, rows, _, layout, _ in CASES:
        slot, K = reset_slots(layout, S, B, rows, S)
        assert slot.shape == (S, B) and slot.dtype == np.int32 and K >= 1, name
        resets = [tuple(np.flatnonzero(slot[:, b] >= 0)) for b in range(B)]
        for b in range(B):                              # slot k of a column is its k-th reset
            assert list(slot[resets[b], b]) == list(range(len(resets[b]))), (name, b)
        if layout == "packed":
            assert K >= 64 and sum(len(resets[b]) > 0 for b in rows) == len(rows) - 1, name
            continue
        if S >= 32:
            assert len({resets[b] for b in rows}) == len(rows), name
        assert all(len(resets[b]) > 0 for b in range(B) if b not in rows and b % len(PATTERNS)), name
        assert len(resets[rows[0]]) == 0 and all(len(resets[b]) > 0 for b in rows[1:]), name
        if layout == "dense":
            assert K == S - 1 and resets[rows[-1]] == tuple(range(1, S)), name


# ------------------------------------------------------------------------------------------------ GPU
def _gpu_run(cell, wd, x, h0, c0, dy, dhn, dcn, reset):
    """forward + backward of ops.rnn_sequence with ``reset`` on all rows; -> outputs and every gradient."""
    from dotaclient_b200 import ops
    p = [wd[k].clone().requires_grad_(True) for k in WEIGHTS]
    xg = x.detach().requires_grad_(True)
    h0g = h0.detach().requires_grad_(True)
    c0g = c0.detach().requires_grad_(True) if cell == "lstm" else None
    y, hn, cn = ops.rnn_sequence(xg, *p, h0g, c0g, cell, reset)
    outs, grads = [y, hn], [dy, dhn]
    if cell == "lstm":
        outs.append(cn)
        grads.append(dcn)
    torch.autograd.backward(outs, grads)
    r = {"y": y.detach(), "h_n": hn.detach(), "dx": xg.grad, "dh0": h0g.grad}
    if cell == "lstm":
        r.update(c_n=cn.detach(), dc0=c0g.grad)
    r.update({k: t.grad for k, t in zip(WEIGHTS, p)})
    return r


def _forward(cell, wd, x, h0, c0, reset, w_hh=None):
    from dotaclient_b200 import ops
    with torch.no_grad():
        y, hn, cn = ops.rnn_sequence(x, wd["weight_ih_l0"], wd["weight_hh_l0"] if w_hh is None else w_hh, wd["bias_ih_l0"],
                                     wd["bias_hh_l0"], h0, c0, cell, reset)
    return {"y": y, "h_n": hn, "c_n": cn}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_rnn_resets_vs_fp64(case):
    """Forward on R, backward with a dense upstream gradient on R (and exact zeros in dh0 / dc0 of columns reset at t = 0),
    weight gradients with the upstream gradient zero outside R (and exact zeros in every state gradient outside R),
    superposition of the two partial upstream gradients, a bitwise repeat, and the reset entry points with every slot at -1
    bit for bit equal to the plain ones.  The mutants of the module docstring must fail their bounds."""
    name, cell, B, S, H, rows, saturate, layout, sensitivity = case
    from dotaclient_b200 import ops
    d = torch.device("cuda", 0)
    w = make_weights(cell, H, B + S + H, saturate)
    wd = {k: v.to(d) for k, v in w.items()}
    slot, K = reset_slots(layout, S, B, rows, S)
    g = torch.Generator(device=d).manual_seed(B * S + H + 1)
    x = torch.randn(S, B, H, device=d, generator=g)
    h0 = torch.randn(B, H, device=d, generator=g) * 0.5
    c0 = torch.randn(B, H, device=d, generator=g) * 0.5 if cell == "lstm" else None
    h_tab = torch.randn(K, B, H, device=d, generator=g) * 0.5
    c_tab = torch.randn(K, B, H, device=d, generator=g) * 0.5 if cell == "lstm" else None
    dy = torch.randn(S, B, H, device=d, generator=g)
    dhn = torch.randn(B, H, device=d, generator=g)
    dcn = torch.randn(B, H, device=d, generator=g) if cell == "lstm" else None
    slot_d = torch.from_numpy(slot).to(d)
    reset = (slot_d, h_tab, c_tab)
    ridx = torch.tensor(rows, device=d)
    out_r = torch.ones(B, dtype=torch.bool, device=d)
    out_r[ridx] = False

    # the float64 reference and the fp32 calibration, on R only (table rows are column-local: R's columns of the tables)
    def cols(t, dim):
        return None if t is None else t.index_select(dim, ridx).cpu()
    args = (cell, w, cols(x, 1), cols(h0, 0), cols(c0, 0), slot[:, list(rows)], cols(h_tab, 1), cols(c_tab, 1), cols(dy, 1),
            cols(dhn, 0), cols(dcn, 0))
    f64, f32 = segmented_reference(*args, torch.float64), segmented_reference(*args, torch.float32)
    if saturate:
        pre = (args[2].double() @ w["weight_ih_l0"].double().t() + w["bias_ih_l0"].double()).abs().max()
        assert 30 <= float(pre) <= 150, "saturating inputs reach |pre-activation| %.1f" % float(pre)

    failures, ratios = [], {}
    # 1 + 2: forward and the state gradients of a dense upstream gradient, on R
    dense = _gpu_run(cell, wd, x, h0, c0, dy, dhn, dcn, reset)
    names = forward_names(cell) + state_grad_names(cell)
    for n in names:
        if not torch.isfinite(dense[n]).all():
            failures.append("%s is not finite" % n)
    got = _rows(dense, rows, names)
    for kind, bound in ((forward_names(cell), FORWARD_BOUND), (state_grad_names(cell), STATE_GRAD_BOUND)):
        r, over = bound_check(got, f64, f32, kind, bound)
        ratios.update(r)
        failures += over
    first = slot_d[0] >= 0                                 # reset at t = 0: h0 / c0 are never read
    for n in ("dh0", "dc0") if cell == "lstm" else ("dh0",):
        if bool((dense[n][first] != 0).any()):
            failures.append("%s is non-zero on columns reset at t = 0" % n)

    # 5: a repeated forward + backward is bitwise equal
    again = _gpu_run(cell, wd, x, h0, c0, dy, dhn, dcn, reset)
    failures += ["%s differs on a repeat" % n for n in dense if not torch.equal(dense[n], again[n])]
    del again

    # 3: upstream gradient zero outside R -> weight gradients of R alone, and no gradient leaks into other rows
    keep = (~out_r).to(torch.float32)
    only_up = (dy * keep[None, :, None], dhn * keep[:, None], dcn * keep[:, None] if cell == "lstm" else None)
    only = _gpu_run(cell, wd, x, h0, c0, *only_up, reset)
    r, over = bound_check({n: only[n].cpu() for n in WEIGHTS}, f64, f32, WEIGHTS, WEIGHT_GRAD_BOUND)
    ratios.update(r)
    failures += over
    for n in state_grad_names(cell):
        t = only[n][:, out_r] if n == "dx" else only[n][out_r]
        if bool((t != 0).any()):
            failures.append("%s is non-zero outside R (%d elements)" % (n, int((t != 0).sum())))

    # 4: superposition of the dense weight gradients
    drop = out_r.to(torch.float32)
    rest = _gpu_run(cell, wd, x, h0, c0, dy * drop[None, :, None], dhn * drop[:, None],
                    dcn * drop[:, None] if cell == "lstm" else None, reset)
    for n in WEIGHTS:
        if not torch.isfinite(dense[n]).all():
            failures.append("%s is not finite" % n)
        err = float((dense[n].double() - only[n].double() - rest[n].double()).abs().max())
        scale = float(dense[n].abs().max())
        ratios["superpose " + n] = err / scale
        if not err <= SUPERPOSE * scale:
            failures.append("superposition of %s: %.3e of max|dW| %.3e" % (n, err, scale))
    del dense, only, rest

    # 6: every slot at -1: the reset entry points and the correction (all rows weighted 0) are the plain ones bit for bit
    plain = _gpu_run(cell, wd, x, h0, c0, dy, dhn, dcn, None)
    unset = _gpu_run(cell, wd, x, h0, c0, dy, dhn, dcn, (torch.full_like(slot_d, -1), h_tab, c_tab))
    failures += ["%s: the reset path without resets differs from the plain one" % n for n in plain
                 if not torch.equal(plain[n], unset[n])]
    del plain, unset

    if sensitivity:
        shifted = torch.full_like(slot_d, -1)
        shifted[1:] = slot_d[:-1]
        rolled = (slot_d, h_tab.roll(1, dims=1), None if c_tab is None else c_tab.roll(1, dims=1))
        mutants = {"tf32": _forward(cell, wd, x, h0, c0, reset, tf32_rna(wd["weight_hh_l0"])),
                   "shifted": _forward(cell, wd, x, h0, c0, (shifted, h_tab, c_tab)),
                   "rolled": _forward(cell, wd, x, h0, c0, rolled)}
        for m, out in mutants.items():
            r, over = bound_check(_rows(out, rows, forward_names(cell)), f64, f32, forward_names(cell), FORWARD_BOUND)
            ratios.update({"%s %s" % (m, n): v for n, v in r.items() if not n.startswith("rel ")})
            if not over:
                failures.append("the %s mutant passed the forward bound" % m)
        # the dW_hh reset correction dropped: every table row marked unused
        orig_rows = ops._reset_rows

        def unused_rows(s, k):
            tok, used = orig_rows(s, k)
            return tok, torch.zeros_like(used)
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(ops, "_reset_rows", unused_rows)
            nocorr = _gpu_run(cell, wd, x, h0, c0, *only_up, reset)
        r, over = bound_check({"weight_hh_l0": nocorr["weight_hh_l0"].cpu()}, f64, f32, ("weight_hh_l0",), WEIGHT_GRAD_BOUND)
        ratios["no-correction weight_hh_l0"] = r["weight_hh_l0"]
        if not over:
            failures.append("the backward without the dW_hh reset correction passed the bound on weight_hh_l0")
    print("\n%s (K %d) ratios: %s" % (name, K, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert not failures, failures
