"""The recurrence (``ops.rnn_sequence``: i2h GEMM, recurrence kernels, weight-gradient GEMMs) at the shapes the benchmark
runs, against ``torch.nn.GRU`` / ``nn.LSTM`` in float64 on the CPU.

Sequences are independent, so the float64 reference runs only on a sample R of 8 rows: rows 0 and B-1 and the rows on
both sides of a batch-tile, cluster or M-tile boundary of the design under test.  The same weights also run through torch
in fp32 on R; that run calibrates the bound every kernel output must meet, per tensor:

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

The floor is absolute (scaled by the tensor's magnitude, not element-wise): ``dc_tanh`` = 1 - 2/(e^{2x}+1) has an absolute
error of about 6e-8 near 0 by design, which no relative bound on tiny activations would admit.  The bound is shown to see
the error 3xTF32 removes: a forward with W_hh rounded to TF32 (a single-pass TF32 h2h product) must fail it, once per
design.  ``test_bound_logic_on_the_cpu`` checks the same helpers without a GPU.

K and FLOOR differ by kind of tensor.  Measured on one H100 SXM (700 W power limit), the largest ratio
max|gpu - f64| / max|torch32 - f64| per design, forward / state gradients / weight gradients (the weight gradients as
max|gpu - f64| / max|f64| in brackets; re-measured on an H100 80GB HBM3 at 700 W once the weight-gradient GEMM bounded
its accumulation length to 4096 rows, ``kWgFlush`` in gemm_tf32x3.cu -- before, cluster reached 179 (8.0e-5) and step-wise 511 (2.4e-4)):
    resident  (H 128, fp32 FMA)          4.4 /  6.3 /  12  (4.5e-6)
    cluster   (H 256, wgmma 3xTF32)      6.9 / 13   /  21  (1.0e-5)
    step-wise (H 512, split-K 3xTF32)    9.8 / 20   /  9.7 (5.5e-6, C4's 1024 steps)
    generic   (H 192, fp32 FMA)          4.6 /  4.7 /  9.1 (4.1e-6)
    saturating inputs (H 128 / 256)      8.7 /  6.2 /  8.1 (4.6e-4, at a torch fp32 error of 1.1e-4)
The forwards with TF32-rounded W_hh give ratios of 96 to 284, so the forward K of 16 rejects them with a margin of 6.

The edge cases, same columns (the TF32-rounded forward's ratios last):
    resident-b512-gru (3-sequence tiles, ragged last tile)   3.8 / 3.5 / 12 (4.5e-6)   TF32 191-219
    resident S 1 / S 3 (fewer steps than kStages = 4)         5.1 / 5.1 / 4.1 (5.9e-7)  TF32 200-400
    cluster B 1 (S 16) / B 33 (S 1)                           11  / 11  / 8.8 (1.3e-6)  TF32 47-568
    step-wise B 1 (S 16) / B 129 (S 1)                        8.6 / 22  / 11  (3.2e-6)  TF32 125-345
    generic B 5 (S 2)                                         4.7 / 5.1 / 3.8 (7.5e-7)  TF32 233-319
The smallest TF32 ratio, 47 (cluster B 1, c_n), still clears the forward K by a factor of 3.
The weight-gradient floor, 1e-4, is twice what the saturating LSTM at H 128 needs (its bias gradients: 9.3e-5 of
max|f64| at 8.1 times torch's error); the step-wise design at C4's 1024 steps needs 3.2e-6.  It was 5e-4 while the
weight-gradient GEMM's error grew with the tokens it summed.  The superposition residual reaches 1.1e-5 of max|dW| (it was
3.0e-4 at the step-wise design's 524288 tokens).
"""
import pytest
import torch

# (K, FLOOR) per kind of tensor: allowed multiple of torch fp32's own error against float64, and the absolute floor as a
# fraction of max|f64| of the tensor
FORWARD_BOUND = (16.0, 1e-6)       # y, h_n, c_n
STATE_GRAD_BOUND = (32.0, 1e-6)    # dx, dh0, dc0
WEIGHT_GRAD_BOUND = (4.0, 1e-4)    # dW_ih, dW_hh, db_ih, db_hh: sums over thousands of tokens
SUPERPOSE = 5e-5                   # dense == R-only + complement weight gradients, as a fraction of max|dW|

# (case id, cell, B, S, H, sampled rows R, saturating inputs, TF32 sensitivity run)
CASES = [
    # resident, H 128: 2-sequence tiles (B <= 264) on 128 CTAs; 3-sequence (GRU) / 4-sequence (LSTM) tiles above
    ("resident-b256-gru", "gru", 256, 512, 128, (0, 1, 2, 127, 128, 129, 254, 255), False, True),
    ("resident-b256-lstm", "lstm", 256, 512, 128, (0, 1, 2, 127, 128, 129, 254, 255), False, True),
    ("resident-b512-lstm", "lstm", 512, 512, 128, (0, 3, 4, 255, 256, 259, 508, 511), False, False),
    # 3-sequence GRU tiles (B > 2 * SMs): 170 full tiles and a last tile holding rows 510 and 511
    ("resident-b512-gru", "gru", 512, 512, 128, (0, 2, 3, 254, 255, 509, 510, 511), False, True),
    # fewer steps than the kStages = 4 prefetch ring: the prologue and refill guards
    ("resident-s1-gru", "gru", 256, 1, 128, (0, 1, 2, 127, 128, 129, 254, 255), False, True),
    ("resident-s1-lstm", "lstm", 256, 1, 128, (0, 1, 2, 127, 128, 129, 254, 255), False, True),
    ("resident-s3-gru", "gru", 256, 3, 128, (0, 1, 2, 127, 128, 129, 254, 255), False, True),
    ("resident-s3-lstm", "lstm", 256, 3, 128, (0, 1, 2, 127, 128, 129, 254, 255), False, True),
    # cluster, H 256: 32 sequences per 8-CTA cluster; 16 clusters, and a last cluster holding 20 of its 32 rows
    ("cluster-b512-gru", "gru", 512, 512, 256, (0, 31, 32, 255, 256, 480, 481, 511), False, True),
    ("cluster-b512-lstm", "lstm", 512, 512, 256, (0, 31, 32, 255, 256, 480, 481, 511), False, True),
    ("cluster-b500-gru", "gru", 500, 512, 256, (0, 31, 32, 255, 256, 479, 480, 499), False, False),
    ("cluster-b500-lstm", "lstm", 500, 512, 256, (0, 31, 32, 255, 256, 479, 480, 499), False, False),
    # one live row in a cluster, one row past a cluster at a single step
    ("cluster-b1-lstm", "lstm", 1, 16, 256, (0,), False, True),
    ("cluster-b33-s1-gru", "gru", 33, 1, 256, (0, 1, 30, 31, 32), False, True),
    # step-wise, H 512: 128-row M tiles of the per-step split-K GEMM; C4's B 512 x S 1024, and a ragged last M tile
    ("stepwise-b512-lstm", "lstm", 512, 1024, 512, (0, 127, 128, 255, 256, 383, 384, 511), False, True),
    ("stepwise-b300-gru", "gru", 300, 256, 512, (0, 127, 128, 255, 256, 257, 298, 299), False, True),
    # one live row in an M tile, one row past an M tile at a single step
    ("stepwise-b1-gru", "gru", 1, 16, 512, (0,), False, True),
    ("stepwise-b129-s1-lstm", "lstm", 129, 1, 512, (0, 1, 126, 127, 128), False, True),
    # generic, H 192: 4-sequence CTAs
    ("generic-b256-lstm", "lstm", 256, 512, 192, (0, 3, 4, 127, 128, 131, 252, 255), False, True),
    ("generic-b5-s2-gru", "gru", 5, 2, 192, (0, 3, 4), False, True),
    # saturated gates (|pre-activation| 30..100) and an LSTM forget bias of +5
    ("saturating-h128-gru", "gru", 256, 512, 128, (0, 1, 2, 127, 128, 129, 254, 255), True, False),
    ("saturating-h128-lstm", "lstm", 256, 512, 128, (0, 1, 2, 127, 128, 129, 254, 255), True, False),
    ("saturating-h256-gru", "gru", 256, 512, 256, (0, 31, 32, 127, 128, 224, 225, 255), True, False),
    ("saturating-h256-lstm", "lstm", 256, 512, 256, (0, 31, 32, 127, 128, 224, 225, 255), True, False),
]
WEIGHTS = ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0")


# ------------------------------------------------------------------------------------------------ helpers
def tf32_rna(t):
    """fp32 -> TF32 (10 mantissa bits), round to nearest with ties away from zero: the hi half of the kernels' 3xTF32 split."""
    bits = t.to(torch.float32).contiguous().view(torch.int32)
    return ((bits + 0x1000) & -0x2000).view(torch.float32)


def make_weights(cell, H, seed, saturate):
    """torch's default initialisation; with ``saturate`` the i2h rows of every fourth unit are scaled so those gates see
    pre-activations of 30..100, and the LSTM forget gate gets a bias of +5 (cell states build up over hundreds of steps)."""
    torch.manual_seed(seed)
    m = (torch.nn.GRU if cell == "gru" else torch.nn.LSTM)(H, H)
    w = {k: getattr(m, k).detach().clone() for k in WEIGHTS}
    if saturate:
        G = 3 if cell == "gru" else 4
        rows = (torch.arange(G * H) % H) % 4 == 0
        w["weight_ih_l0"][rows] *= 40.0
        if cell == "lstm":
            w["bias_ih_l0"][H:2 * H] += 5.0         # gate order i, f, g, o
    return w


def reference(cell, w, x, h0, c0, dy, dhn, dcn, dtype, w_hh=None):
    """torch's CPU GRU / LSTM in ``dtype`` on the rows given ([S, R, H] time-major): outputs and the gradients of
    <y, dy> + <h_n, dhn> (+ <c_n, dcn>).  ``w_hh`` replaces the h2h weight when given."""
    H = h0.shape[-1]
    m = (torch.nn.GRU if cell == "gru" else torch.nn.LSTM)(H, H).to(dtype)
    with torch.no_grad():
        for k in WEIGHTS:
            getattr(m, k).copy_(w_hh if (k == "weight_hh_l0" and w_hh is not None) else w[k])
    xr = x.to(dtype, copy=True).requires_grad_(True)
    h0r = h0.to(dtype, copy=True).unsqueeze(0).requires_grad_(True)
    if cell == "lstm":
        c0r = c0.to(dtype, copy=True).unsqueeze(0).requires_grad_(True)
        y, (hn, cn) = m(xr, (h0r, c0r))
        loss = (y * dy.to(dtype)).sum() + (hn[0] * dhn.to(dtype)).sum() + (cn[0] * dcn.to(dtype)).sum()
    else:
        y, hn = m(xr, h0r)
        cn = None
        loss = (y * dy.to(dtype)).sum() + (hn[0] * dhn.to(dtype)).sum()
    loss.backward()
    out = {"y": y.detach(), "h_n": hn[0].detach(), "dx": xr.grad, "dh0": h0r.grad[0]}
    if cell == "lstm":
        out.update(c_n=cn[0].detach(), dc0=c0r.grad[0])
    out.update({k: getattr(m, k).grad for k in WEIGHTS})
    return out


def bound_check(got, f64, f32, names, bound):
    """-> ({name: max|got - f64| / max|f32 - f64|}, [the tensors over the bound K * max|f32 - f64| + FLOOR * max|f64|])."""
    k, floor = bound
    ratios, over = {}, []
    for n in names:
        ref = f64[n]
        err = float((got[n].double() - ref).abs().max())
        cal = float((f32[n].double() - ref).abs().max())
        ratios[n] = err / cal if cal > 0 else (0.0 if err == 0 else float("inf"))
        if not err <= k * cal + floor * float(ref.abs().max()):
            over.append("%s: max|err| %.3e, torch fp32 %.3e, max|f64| %.3e" % (n, err, cal, float(ref.abs().max())))
        ratios["rel " + n] = err / max(float(ref.abs().max()), 1e-30)
    return ratios, over


def forward_names(cell):
    return ("y", "h_n", "c_n") if cell == "lstm" else ("y", "h_n")


def state_grad_names(cell):
    return ("dx", "dh0", "dc0") if cell == "lstm" else ("dx", "dh0")


def loop_fp32(cell, w, x, h0, c0):
    """A step-by-step fp32 GRU / LSTM written out from the cell equations: an fp32 implementation independent of torch's."""
    H = h0.shape[-1]
    w_ih, w_hh, b_ih, b_hh = (w[k].float() for k in WEIGHTS)
    h, c, ys = h0.float(), None if c0 is None else c0.float(), []
    for t in range(x.shape[0]):
        gi = x[t].float() @ w_ih.t() + b_ih
        gh = h @ w_hh.t() + b_hh
        if cell == "gru":
            r = torch.sigmoid(gi[:, :H] + gh[:, :H])
            z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
            n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
            h = (1 - z) * n + z * h
        else:
            g = gi + gh
            i, f = torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H])
            c = f * c + i * torch.tanh(g[:, 2 * H:3 * H])
            h = torch.sigmoid(g[:, 3 * H:]) * torch.tanh(c)
        ys.append(h)
    out = {"y": torch.stack(ys), "h_n": h}
    if cell == "lstm":
        out["c_n"] = c
    return out


# ------------------------------------------------------------------------------------------------ CPU: the bound itself
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_bound_logic_on_the_cpu(cell):
    """An independent fp32 implementation passes the forward bound; torch fp32 with W_hh rounded to TF32 fails it."""
    S, R, H = 96, 8, 64
    w = make_weights(cell, H, 7, False)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(S, R, H, generator=g)
    h0, c0 = torch.randn(R, H, generator=g) * 0.5, torch.randn(R, H, generator=g) * 0.5
    dy, dhn, dcn = torch.randn(S, R, H, generator=g), torch.randn(R, H, generator=g), torch.randn(R, H, generator=g)
    c0 = c0 if cell == "lstm" else None
    f64 = reference(cell, w, x, h0, c0, dy, dhn, dcn, torch.float64)
    f32 = reference(cell, w, x, h0, c0, dy, dhn, dcn, torch.float32)
    _, over = bound_check(loop_fp32(cell, w, x, h0, c0), f64, f32, forward_names(cell), FORWARD_BOUND)
    assert not over, over
    rounded = reference(cell, w, x, h0, c0, dy, dhn, dcn, torch.float32, w_hh=tf32_rna(w["weight_hh_l0"]))
    _, over = bound_check(rounded, f64, f32, forward_names(cell), FORWARD_BOUND)
    assert over, "a TF32 h2h product passed the forward bound"


def test_tf32_rna_rounding():
    """Round to nearest, ties away from zero, at the 13th bit (the kernels' dc_tf32_rna)."""
    one_ulp = 2.0 ** -10                                 # TF32 spacing in [1, 2)
    x = torch.tensor([1.0, 1.0 + one_ulp / 2, -(1.0 + one_ulp / 2), 1.0 + one_ulp / 2 - 2.0 ** -23, 3.0 + 2.0 ** -23])
    want = torch.tensor([1.0, 1.0 + one_ulp, -(1.0 + one_ulp), 1.0, 3.0])
    assert torch.equal(tf32_rna(x), want)
    y = tf32_rna(torch.randn(1000))
    assert torch.equal(tf32_rna(y), y) and bool(((y.view(torch.int32) & 0x1FFF) == 0).all())


# ------------------------------------------------------------------------------------------------ GPU
def _gpu_run(cell, wd, x, h0, c0, dy, dhn, dcn):
    """forward + backward of ops.rnn_sequence on all rows; -> outputs and every gradient."""
    from dotaclient_b200 import ops
    p = [wd[k].clone().requires_grad_(True) for k in WEIGHTS]
    xg = x.detach().requires_grad_(True)
    h0g = h0.detach().requires_grad_(True)
    c0g = c0.detach().requires_grad_(True) if cell == "lstm" else None
    y, hn, cn = ops.rnn_sequence(xg, *p, h0g, c0g, cell)
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


def _rows(r, rows, names):
    """The sampled rows of the per-sequence tensors, on the CPU."""
    idx = torch.tensor(rows, device=r["y"].device)
    return {n: (r[n].index_select(1, idx) if n in ("y", "dx") else r[n].index_select(0, idx)).cpu() for n in names}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_rnn_production_shape_vs_fp64(case):
    """Forward on R, backward with a dense upstream gradient on R, weight gradients with the upstream gradient zero outside
    R (and exact zeros in every state gradient outside R), superposition of the two partial upstream gradients, and a
    bitwise repeat.  TF32-rounded W_hh must fail the forward bound."""
    _, cell, B, S, H, rows, saturate, sensitivity = case
    d = torch.device("cuda", 0)
    w = make_weights(cell, H, B + S + H, saturate)
    wd = {k: v.to(d) for k, v in w.items()}
    g = torch.Generator(device=d).manual_seed(B * S + H)
    x = torch.randn(S, B, H, device=d, generator=g)
    h0 = torch.randn(B, H, device=d, generator=g) * 0.5
    c0 = torch.randn(B, H, device=d, generator=g) * 0.5 if cell == "lstm" else None
    dy = torch.randn(S, B, H, device=d, generator=g)
    dhn = torch.randn(B, H, device=d, generator=g)
    dcn = torch.randn(B, H, device=d, generator=g) if cell == "lstm" else None
    ridx = torch.tensor(rows, device=d)
    out_r = torch.ones(B, dtype=torch.bool, device=d)
    out_r[ridx] = False

    # the float64 reference and the fp32 calibration, on R only
    xs, h0s = x[:, ridx].cpu(), h0[ridx].cpu()
    c0s = c0[ridx].cpu() if cell == "lstm" else None
    dys, dhns = dy[:, ridx].cpu(), dhn[ridx].cpu()
    dcns = dcn[ridx].cpu() if cell == "lstm" else None
    f64 = reference(cell, w, xs, h0s, c0s, dys, dhns, dcns, torch.float64)
    f32 = reference(cell, w, xs, h0s, c0s, dys, dhns, dcns, torch.float32)
    if saturate:
        pre = (xs.double() @ w["weight_ih_l0"].double().t() + w["bias_ih_l0"].double()).abs().max()
        assert 30 <= float(pre) <= 150, "saturating inputs reach |pre-activation| %.1f" % float(pre)

    failures, ratios = [], {}
    # 1 + 2: forward and the state gradients of a dense upstream gradient, on R
    dense = _gpu_run(cell, wd, x, h0, c0, dy, dhn, dcn)
    names = forward_names(cell) + state_grad_names(cell)
    got = _rows(dense, rows, names)
    for n in names:
        if not torch.isfinite(dense[n]).all():
            failures.append("%s is not finite" % n)
    for kind, bound in ((forward_names(cell), FORWARD_BOUND), (state_grad_names(cell), STATE_GRAD_BOUND)):
        r, over = bound_check(got, f64, f32, kind, bound)
        ratios.update(r)
        failures += over

    # 5: a repeated forward + backward is bitwise equal (no recurrence kernel uses atomics)
    again = _gpu_run(cell, wd, x, h0, c0, dy, dhn, dcn)
    failures += ["%s differs on a repeat" % n for n in dense if not torch.equal(dense[n], again[n])]
    del again

    # 3: upstream gradient zero outside R -> weight gradients of R alone, and no gradient leaks into other rows
    keep = (~out_r).to(torch.float32)
    only = _gpu_run(cell, wd, x, h0, c0, dy * keep[None, :, None], dhn * keep[:, None],
                    dcn * keep[:, None] if cell == "lstm" else None)
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
                    dcn * drop[:, None] if cell == "lstm" else None)
    for n in WEIGHTS:
        if not torch.isfinite(dense[n]).all():
            failures.append("%s is not finite" % n)
        err = float((dense[n].double() - only[n].double() - rest[n].double()).abs().max())
        scale = float(dense[n].abs().max())
        ratios["superpose " + n] = err / scale
        if not err <= SUPERPOSE * scale:
            failures.append("superposition of %s: %.3e of max|dW| %.3e" % (n, err, scale))
    del dense, only, rest

    # sensitivity: a single-pass TF32 h2h product (W_hh rounded to TF32) must fail the forward bound
    if sensitivity:
        from dotaclient_b200 import ops
        with torch.no_grad():
            y, hn, cn = ops.rnn_sequence(x, wd["weight_ih_l0"], tf32_rna(wd["weight_hh_l0"]), wd["bias_ih_l0"], wd["bias_hh_l0"],
                                         h0, c0, cell)
        rounded = _rows({"y": y, "h_n": hn, "c_n": cn}, rows, forward_names(cell))
        r, over = bound_check(rounded, f64, f32, forward_names(cell), FORWARD_BOUND)
        ratios.update({"tf32 " + n: v for n, v in r.items()})
        if not over:
            failures.append("the TF32-rounded W_hh passed the forward bound")
    print("\n%s ratios: %s" % (case[0], ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert not failures, failures
