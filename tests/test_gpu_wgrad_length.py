"""Weight-gradient GEMM (``gemm_wgrad_kernel``: ``dc_gemm_wgrad_tf32x3`` and ``dc_unit_wgrad_routed``) at the accumulation
lengths the benchmark runs, against float64.

The kernel splits the tokens over ``nsplit = max(1, SMs / tiles)`` CTAs per output tile, so one CTA sums about
``T * tiles / SMs`` rows.  Cases: the pre-RNN ``[H, 896]`` and ``W_ih`` / ``W_hh`` ``[4H, H]`` weight gradients and the
routed 5- and 16-unit groups (real arg-max routing of a max-pool) at c2's, c3's and c4's token counts, and a synthetic
``[2048, 1152]`` product whose 144 output tiles leave one split, so that one CTA sums all T rows (16k to 1M).  Two
operand kinds: zero-mean normal, and coherent (X = ReLU(normal), dY = normal + 0.5), where the partial sums grow like T
rather than sqrt(T) -- what ReLU activations look like, and the worst case for a biased accumulator.

Reference: float64 on the CPU over a sample of output rows o (both sides of the 128-row tile boundaries) and input
columns i (both consumer warpgroups' halves, i = 63 / 64, and the tile boundaries); every sampled entry is exact.  The
same product in fp32 on the CPU calibrates the bound (``bound``):

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

Also checked per case: db against the float64 column sum (within 1e-6 of max_o sum_t |dY|), a bitwise repeat, and
(plain cases) accumulation into a row slice of a larger gradient.  Sensitivity: single-pass TF32 with exact accumulation
(operands rounded by ``tf32_rna``, the product in float64) must fail the bound on zero-mean operands.  On coherent ones it
cannot: its rounding errors are unbiased and average out over T, to 3e-6 .. 3e-5 of max|f64|, below the error of any
kernel that accumulates in fp32, so there it is reported only.  ``test_bound_logic_on_the_cpu`` shows the bound accepting
an independent fp32 product and rejecting that TF32 mutant and a 3xTF32 product that drops one k-step's lo*hi term.
Growth (``test_error_does_not_grow_with_length``): on the single-split product, max|err| / max|f64| at 1M tokens is at
most 1.5x its value at 16k, for both operand kinds.  ``test_unit_dgrad_dwb_length`` holds the unit encoder's dW_b and db_b
within 4e-5 of max|f64| at c2's and c4's token counts, and dW_b to the same growth criterion between them.

Measured on one H100 80GB HBM3 (700 W power limit): the ratio max|gpu - f64| / max|torch32 - f64| and max|err| / max|f64|
of this kernel (every accumulator flushed after 4096 rows, ``kWgFlush`` = 128), the same two for the kernel before it
flushed (one accumulator over the CTA's whole token share), and single-pass TF32's max|err| / max|f64| and its multiple of
the bound:

    case         kind      now           before             TF32
    pre-c2       normal    54.8  2.7e-05      124  6.0e-05   3.7e-04   6.9
    pre-c2       coherent 180.4  2.6e-05      362  5.2e-05   1.1e-05   0.2
    pre-c3       normal    71.8  2.6e-05      575  2.1e-04   2.9e-04   5.6
    pre-c3       coherent 112.0  2.8e-05      785  2.0e-04   8.9e-06   0.2
    pre-c4       normal    62.5  3.4e-05     2135  1.1e-03   4.0e-04   7.3
    pre-c4       coherent 109.2  2.8e-05     2330  6.1e-04   4.3e-06   0.1
    ih-c2        normal    91.1  3.1e-05       91  3.1e-05   2.5e-04   4.8
    ih-c2        coherent 155.5  2.8e-05      156  2.8e-05   1.0e-05   0.2
    ih-c3        normal    64.6  2.6e-05      472  1.9e-04   3.0e-04   5.6
    ih-c3        coherent 138.9  2.9e-05     1039  2.1e-04   5.9e-06   0.1
    ih-c4        normal    59.3  2.6e-05     3766  1.6e-03   2.6e-04   4.9
    ih-c4        coherent 101.2  2.8e-05     3453  9.7e-04   5.3e-06   0.1
    unit5-c2     normal    71.0  2.0e-05      108  3.1e-05   2.2e-04   4.1
    unit5-c2     coherent  87.0  1.4e-05      137  2.3e-05   4.9e-06   0.1
    unit5-c4     normal    58.9  3.5e-05      287  1.7e-04   3.8e-04   6.9
    unit5-c4     coherent  42.9  1.7e-05      220  8.5e-05   4.2e-06   0.1
    unit16-c2    normal    22.5  1.3e-05       75  4.2e-05   3.1e-04   5.7
    unit16-c2    coherent  23.5  7.2e-06       99  3.0e-05   4.6e-06   0.1
    unit16-c4    normal     9.6  1.2e-05      176  2.1e-04   3.4e-04   5.7
    unit16-c4    coherent  20.8  7.5e-06      320  1.2e-04   2.9e-06   0.1
    single-16k   normal    69.3  2.9e-05      313  1.3e-04   2.7e-04   5.0
    single-16k   coherent 161.5  2.9e-05      631  1.1e-04   2.6e-05   0.5
    single-64k   normal    96.8  3.1e-05     1566  5.1e-04   2.3e-04   4.4
    single-64k   coherent 178.9  2.8e-05     2371  3.8e-04   1.5e-05   0.3
    single-256k  normal    61.9  2.7e-05     4930  2.1e-03   2.6e-04   4.8
    single-256k  coherent 134.7  2.9e-05     4570  9.7e-04   7.6e-06   0.1
    single-1024k normal    63.3  2.9e-05    14496  6.6e-03   2.7e-04   5.0
    single-1024k coherent  75.7  2.9e-05     8637  3.3e-03   4.3e-06   0.1

FLOOR = 5e-5 leaves this kernel a margin of 1.56 (largest share of its bound used: 0.64, unit5-c4 normal) and single-pass
TF32 one of at least 4.1 on zero-mean operands; ``kWgFlush`` in gemm_tf32x3.cu records how the interval was chosen.  The
kernel before the flush fails the bound in the c3, c4 and single-split cases and passes it in the six c2 cases of W_ih
and the unit groups, whose CTAs sum only 4k to 16k rows: at c2 only the pre-RNN cases tell the two apart.  Its growth
also failed for both kinds: on the single split, normal 1.3e-4 / 5.1e-4 / 2.1e-3 / 6.6e-3 at 16k / 64k / 256k / 1M (50x),
coherent 1.1e-4 / 3.8e-4 / 9.7e-4 / 3.3e-3 (29x).  Now: normal 2.92e-5 / 3.15e-5 / 2.65e-5 / 2.86e-5 (0.98x), coherent
2.87e-5 / 2.84e-5 / 2.85e-5 / 2.88e-5 (1.00x).  db reaches 9.4e-8 of max sum|dY| (before its Kahan-compensated column
sums: 1.5e-5 at the single split's 1M).  The unit encoder's dW_b / db_b (``test_unit_dgrad_dwb_length``, flushed every
``kDgFlush`` = 32 tiles), max|err| / max|f64| at 131072 / 524288 tokens: normal 1.1e-5, 8.7e-6 / 1.1e-5, 1.0e-5,
coherent 1.8e-5, 1.4e-5 / 1.8e-5, 1.4e-5; before its flush, dW_b 4.1e-5 / 2.4e-4 and 8.5e-5 / 3.5e-4, db_b 2.7e-5 / 1.5e-4
and 6.4e-5 / 2.3e-4.  The file runs in about 20 s.
"""
import functools
import zlib

import numpy as np
import pytest
import torch

from test_gpu_rnn_fp64 import tf32_rna

DEV = torch.device("cuda", 0)
BOUND = (8.0, 5e-5)                # K, FLOOR (see the module docstring)
DB_BOUND = 1e-6                    # db: max|err| <= DB_BOUND * max_o sum_t |dY[t, o]| (the producers' fp32 column sums)
GROWTH = 1.5
DGRAD_FLOOR = 4e-5                 # dW_b / db_b of the unit encoder: max|err| <= DGRAD_FLOOR * max|f64|
SYN_T = (16384, 65536, 262144, 1048576)
KINDS = ("normal", "coherent")

# (case id, form, No, Ni (plain) or units per token (routed), T (plain) or tokens (routed))
CASES = [
    ("pre-c2", "plain", 128, 896, 131072), ("pre-c3", "plain", 256, 896, 262144), ("pre-c4", "plain", 512, 896, 524288),
    ("ih-c2", "plain", 512, 128, 131072), ("ih-c3", "plain", 1024, 256, 262144), ("ih-c4", "plain", 2048, 512, 524288),
    ("unit5-c2", "routed", 128, 5, 131072), ("unit5-c4", "routed", 128, 5, 524288),
    ("unit16-c2", "routed", 128, 16, 131072), ("unit16-c4", "routed", 128, 16, 524288),
] + [("single-%dk" % (t // 1024), "plain", 2048, 1152, t) for t in SYN_T]
CASE = {c[0]: c for c in CASES}


def _sample(n, count, seed):
    """Indices in [0, n): both sides of every 128 boundary (up to 512), the warpgroup halves 63 / 64, the last one, and
    seeded random ones up to `count`."""
    fixed = {0, 63, 64, 127, 128, 191, 255, 256, 383, 384, 511, 512, n // 2 - 1, n // 2, n - 1}
    idx = sorted(i for i in fixed if 0 <= i < n)
    g = np.random.default_rng(seed)
    rest = [i for i in g.permutation(n).tolist() if i not in fixed]
    return torch.tensor(sorted(idx + rest[:max(0, count - len(idx))]), dtype=torch.long)


def operands(kind, rows, cols, g):
    """kind "normal": N(0, 1); "x": ReLU(N(0, 1)); "y": N(0, 1) + 0.5."""
    if kind == "normal":
        return torch.randn(rows, cols, generator=g, device=DEV)
    if kind == "x":
        return torch.relu(torch.randn(rows, cols, generator=g, device=DEV))
    return torch.randn(rows, cols, generator=g, device=DEV) + 0.5


def bound(cal, ref):
    """-> K * max|torch32 - f64| + FLOOR * max|f64|, the largest max|gpu - f64| allowed."""
    return BOUND[0] * cal + BOUND[1] * ref


def reference(dys, xs):
    """Sampled dY [T, n_o] and X [T, n_i] (fp32, CPU) -> (float64, torch fp32, single-pass TF32 exact-sum) products [n_o, n_i]."""
    f64 = dys.double().t() @ xs.double()
    f32 = (dys.t() @ xs).double()
    tf = tf32_rna(dys).double().t() @ tf32_rna(xs).double()
    return f64, f32, tf


def _stats(got, f64, f32, tf):
    ref = float(f64.abs().max())
    return dict(err=float((got.double() - f64).abs().max()), cal=float((f32 - f64).abs().max()), ref=ref,
                tf32=float((tf - f64).abs().max()))


def colsum64(y, rows=65536):
    """-> (float64 column sums of y, max over columns of the float64 sum of |y|), in row chunks: no float64 copy of y."""
    s = torch.zeros(y.shape[1], dtype=torch.float64, device=y.device)
    a = torch.zeros_like(s)
    for r0 in range(0, y.shape[0], rows):
        c = y[r0:r0 + rows].double()
        s += c.sum(0)
        a += c.abs().sum(0)
    return s, float(a.max())


@functools.lru_cache(maxsize=None)
def measure(case_id, kind):
    """Runs one case; -> dict of errors (see _stats), the db error and scale, the repeat / slice results."""
    from dotaclient_b200 import _lib, ops
    _, form, No, Ni_or_nu, T = CASE[case_id]
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(("%s/%s" % (case_id, kind)).encode()))
    x_kind, y_kind = ("normal", "normal") if kind == "normal" else ("x", "y")
    out = {}
    if form == "plain":
        Ni = Ni_or_nu
        dy, x = operands(y_kind, T, No, g), operands(x_kind, T, Ni, g)
        o_idx, i_idx = _sample(No, 12, 1), _sample(Ni, 40, 2)
        dw, db = ops.gemm_wgrad_tf32x3(dy, x)
        dw2, db2 = ops.gemm_wgrad_tf32x3(dy, x)
        out["repeat"] = bool(torch.equal(dw, dw2) and torch.equal(db, db2))
        # accumulation into rows [64, 64 + No) of a larger gradient: the rows outside stay untouched
        base = torch.randn(No + 128, Ni, generator=g, device=DEV)
        base_b = torch.randn(No + 128, generator=g, device=DEV)
        acc, acc_b = base.clone(), base_b.clone()
        ops.gemm_wgrad_tf32x3(dy, x, dw_out=acc[64:64 + No], db_out=acc_b[64:64 + No], accumulate=True)
        out["slice_outside"] = bool(torch.equal(acc[:64], base[:64]) and torch.equal(acc[64 + No:], base[64 + No:])
                                    and torch.equal(acc_b[:64], base_b[:64]) and torch.equal(acc_b[64 + No:], base_b[64 + No:]))
        dys, xs = dy[:, o_idx.to(DEV)].cpu(), x[:, i_idx.to(DEV)].cpu()
        db64, db_scale = colsum64(dy)
        slice_got = (acc[64:64 + No] - base[64:64 + No]).index_select(0, o_idx.to(DEV)).index_select(1, i_idx.to(DEV)).cpu()
        del dy, x, dw2, db2
    else:
        n_u, N = Ni_or_nu, T
        d = operands(y_kind, N, 128, g)
        basic = operands(x_kind, N * n_u, 128, g)
        w_g = torch.randn(128, 128, generator=g, device=DEV) / 128 ** 0.5
        am = (basic @ w_g.t()).view(N, n_u, 128).argmax(1).to(torch.uint8).contiguous()     # the max-pool's arg-max
        lib, st = _lib.load(), _lib.stream_ptr()
        ws = torch.empty(int(lib.dc_gemm_wgrad_workspace_bytes(128, 128)), dtype=torch.uint8, device=DEV)
        res = []
        for _ in range(2):
            dw, db = torch.full((128, 128), 7.0, device=DEV), torch.full((128,), 7.0, device=DEV)
            _lib.check(lib.dc_unit_wgrad_routed(d.data_ptr(), None, 128, am.data_ptr(), basic.data_ptr(), N, n_u, dw.data_ptr(),
                                                db.data_ptr(), ws.data_ptr(), st), "dc_unit_wgrad_routed")
            res.append((dw, db))
        (dw, db), (dw2, db2) = res
        out["repeat"] = bool(torch.equal(dw, dw2) and torch.equal(db, db2))
        o_idx, i_idx = _sample(128, 6, 1), _sample(128, 12, 2)
        od = o_idx.to(DEV)
        r = torch.where(am[:, od].long().unsqueeze(1) == torch.arange(n_u, device=DEV).view(1, n_u, 1), d[:, od].unsqueeze(1), 0.0)
        dys, xs = r.reshape(N * n_u, len(o_idx)).cpu(), basic[:, i_idx.to(DEV)].cpu()
        db64, db_scale = colsum64(d)             # every token routes each channel to exactly one unit
        slice_got = None
        del d, basic, am, r, dw2, db2
    f64, f32, tf = reference(dys, xs)
    got = dw.index_select(0, o_idx.to(DEV)).index_select(1, i_idx.to(DEV)).cpu()
    out.update(_stats(got, f64, f32, tf))
    out["db_err"] = float((db.double() - db64).abs().max())
    out["db_scale"] = db_scale
    if slice_got is not None:
        out["slice_err"] = float((slice_got.double() - f64).abs().max())
    del dw, db, db64, dys, xs
    torch.cuda.empty_cache()
    return out


def report(case_id, kind):
    m = measure(case_id, kind)
    return ("%-12s %-8s  ratio to fp32 %7.2f  max|err|/max|f64| %.2e  tf32 %.2e (%.1fx its bound)  db %.2e of max sum|dY|"
            % (case_id, kind, m["err"] / m["cal"], m["err"] / m["ref"], m["tf32"] / m["ref"],
               m["tf32"] / bound(m["cal"], m["ref"]), m["db_err"] / m["db_scale"]))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case_id", [c[0] for c in CASES])
def test_wgrad_against_float64(case_id, kind):
    m = measure(case_id, kind)
    print(report(case_id, kind))
    assert m["repeat"], "not bitwise repeatable"
    assert m["err"] <= bound(m["cal"], m["ref"]), report(case_id, kind)
    assert m["db_err"] <= DB_BOUND * m["db_scale"], report(case_id, kind)
    if kind == "normal":
        assert m["tf32"] > bound(m["cal"], m["ref"]), "single-pass TF32 passes: " + report(case_id, kind)
    if "slice_err" in m:
        assert m["slice_outside"], "accumulation into a row slice wrote outside it"
        assert m["slice_err"] <= bound(m["cal"], m["ref"]) + 1e-6 * m["ref"], report(case_id, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_error_does_not_grow_with_length(kind):
    rel = {t: measure("single-%dk" % (t // 1024), kind)["err"] / measure("single-%dk" % (t // 1024), kind)["ref"] for t in SYN_T}
    print(kind, {t: "%.2e" % v for t, v in rel.items()})
    assert rel[SYN_T[-1]] <= GROWTH * rel[SYN_T[0]], rel


def _three_tf32(dys, xs, drop_kstep=None):
    """float64 emulation of the kernel's 3xTF32 product (hi*lo + lo*hi + hi*hi, exact sums); with drop_kstep, the lo(X) *
    hi(dY) term of the 8 tokens of that k-step is left out."""
    yh, xh = tf32_rna(dys).double(), tf32_rna(xs).double()
    yl, xl = dys.double() - yh, xs.double() - xh
    lo_hi = xl.clone()
    if drop_kstep is not None:
        lo_hi[8 * drop_kstep:8 * drop_kstep + 8] = 0.0
    return yl.t() @ xh + yh.t() @ lo_hi + yh.t() @ xh


@pytest.mark.parametrize("kind", KINDS)
def test_bound_logic_on_the_cpu(kind):
    """An independent fp32 product (numpy) passes the bound; single-pass TF32 with exact accumulation and a 3xTF32 product
    without one k-step's lo*hi term fail it."""
    g = torch.Generator().manual_seed(5)
    T, No, Ni = 96, 24, 40
    if kind == "normal":
        dys, xs = torch.randn(T, No, generator=g), torch.randn(T, Ni, generator=g)
    else:
        dys, xs = torch.randn(T, No, generator=g) + 0.5, torch.relu(torch.randn(T, Ni, generator=g))
    f64, f32, tf = reference(dys, xs)
    cal, ref = float((f32 - f64).abs().max()), float(f64.abs().max())
    lim = bound(cal, ref)
    indep = torch.from_numpy(dys.numpy().T.astype(np.float32) @ xs.numpy().astype(np.float32)).double()
    assert float((indep - f64).abs().max()) <= lim
    assert float((_three_tf32(dys, xs) - f64).abs().max()) <= lim
    assert float((tf - f64).abs().max()) > lim
    assert float((_three_tf32(dys, xs, drop_kstep=5) - f64).abs().max()) > lim


def dgrad_rel_error(N, kind):
    """dc_unit_dgrad_fused_mask's dW_b and db_b of the routed 16-unit group at N tokens (each CTA sums N * 16 / SMs rows)
    -> (max|err| / max|f64| of dW_b [128, 12], the same of db_b [128]), the float64 chain on the device as reference."""
    import test_gpu_unit_relu_mask as RM
    from dotaclient_b200 import _lib
    lib, n_u, C = _lib.load(), 16, RM.C
    t = RM._inputs(N, n_u, 17 + N)
    if kind == "coherent":                   # G^T units with G and units of one sign: the partial sums grow like T
        t["dx"] += 0.5
        t["units"] = t["units"].abs()
        t["W"] = t["W"].abs()
    wt = t["W"].t().contiguous()
    ws = torch.empty(int(lib.dc_unit_basic_bwd_workspace_bytes()), dtype=torch.uint8, device=DEV)
    mask = RM._stored_mask(lib, _lib, t, N, n_u)
    dwb, dbb = torch.empty(C, RM.F, device=DEV), torch.empty(C, device=DEV)
    RM._dgrad(lib, _lib, t, N, n_u, mask, True, False, False, 0, dwb, dbb, ws, wt)
    ref = torch.zeros(C, RM.F, dtype=torch.float64, device=DEV)
    ref_b = torch.zeros(C, dtype=torch.float64, device=DEV)
    W64, wb64, bb64 = t["W"].double(), t["w_b"].double(), t["b_b"].double()
    for n0 in range(0, N, 8192):
        n1 = min(N, n0 + 8192)
        u = t["units"][n0 * n_u:n1 * n_u].double()
        basic = torch.relu(u @ wb64.t() + bb64)
        d_emb = torch.zeros(n1 - n0, n_u, C, dtype=torch.float64, device=DEV)
        d_emb.scatter_(1, t["am"][n0:n1].long().unsqueeze(1), t["dx"][n0:n1, 2 * C:3 * C].double().unsqueeze(1))
        gm = (d_emb.reshape(-1, C) @ W64) * (basic > 0)
        ref += gm.t() @ u
        ref_b += gm.sum(0)
    return (float((dwb.double() - ref).abs().max() / ref.abs().max()),
            float((dbb.double() - ref_b).abs().max() / ref_b.abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_unit_dgrad_dwb_length(kind):
    """The unit-encoder data gradient's dW_b and db_b (``unit_dgrad_kernel``, accumulated in registers over a CTA's tiles
    and flushed every kDgFlush tiles) within DGRAD_FLOOR of max|f64| at c2's and c4's token counts, and dW_b's error at
    c4 at most GROWTH times c2's."""
    rel = {n: dgrad_rel_error(n, kind) for n in (131072, 524288)}
    print("dW_b, db_b", kind, {n: "%.2e, %.2e" % v for n, v in rel.items()})
    for n, (w, b) in rel.items():
        assert w <= DGRAD_FLOOR and b <= DGRAD_FLOOR, (n, rel)
    assert rel[524288][0] <= GROWTH * rel[131072][0], rel
