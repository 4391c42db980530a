"""GPU tests of the row-list kernels of the target-unit head (``TargetUnitRows``) on their own, at the count and tile edges:
``dc_target_rows``, ``dc_rows_zero_inactive``, ``dc_gemm_tf32x3_rows``, ``dc_gemm_wgrad_tf32x3_rows`` and
``dc_target_unit_q_fwd_rows`` / ``_bwd_rows``, then the whole branch at every token active, at more widths, and replayed from
one captured graph at counts that rise and fall.

The count of a row list lives on the device and the kernels clamp to it, so the checks are arranged around it:
  * bit for bit: rows i < count equal the plain entry point on the gathered / scattered operands (the GEMMs at M = count,
    the weight gradient at T = count, the head on a dense q / dlogits), on every row;
  * float64 (on the GPU) with the bounds of the plain kernels' own tests: test_gpu_gemm.py (3e-6 of max |A||B|^T; dW
    3e-6 of max |dY|^T|X| and db 1e-6 of max sum|dY|), test_gpu_wgrad_length.py's FLOOR past 100k tokens, and
    test_gpu_unit_embed_fused.py for the head;
  * canaries: every output row or column a kernel must not write is filled with a signalling-NaN bit pattern and must
    keep it (compared as int32); every input row it must not read is NaN.  Entries of a row list past the count point at
    a spare row appended to each operand, so that a kernel that read past the count reads a NaN or writes a canary row,
    never out of bounds;
  * a second call gives the same bits.
Each kind of check is shown able to fail on the host: the bitwise checks reject the kernel's result at count - 1, the
canary checks an output with one extra row written, and the float64 bounds the same product on operands rounded by
``tf32_rna`` (single-pass TF32).

Measured on one H100 80GB HBM3 (700 W power limit), the largest max|err| / bound over each test's counts and row lists:
    GEMM, M 5000      att K = H 64 / 128 / 192 / 256 / 512: 0.135 / 0.183 / 0.208 / 0.271 / 0.358 (ReLU, C or C_rows
                      alone: the same to 0.01); q_c 0.185; d_att_c (K 896) 0.528; dy N 128 / 192: 0.181 / 0.177
    GEMM, M 131072    att H 128 / 512: 0.181 / 0.413; q_c 0.182; d_att_c 0.598; dy N 192: 0.180
    weight gradient   Ni 128 / 192 / 512, T 5000: dW 0.094 / 0.099 / 0.090, db 0.092 / 0.089 / 0.053;
                      T 131072 (FLOOR at count T): dW 0.157 / 0.302 / 0.577, db 0.057 / 0.090 / 0.064
    head              N 3001: forward 0.008, backward 0.405; N 131072: forward 0.011, backward 0.448
The file runs in about 20 s.
"""
import numpy as np
import pytest
import torch

from test_gpu_rnn_fp64 import tf32_rna
from test_gpu_target_unit_active import FLOOR, _policy, _obs, _s_f64
from test_gpu_target_unit_active import test_compact_matches_dense as _compact_matches_dense
from test_gpu_unit_embed_fused import C, OFFSETS, UNITS, _head_inputs, _basic64

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
CANARY = 0x7F8DEAD1                 # a signalling NaN: no kernel writes it
GEMM_BOUND = 3e-6                   # max|err| <= GEMM_BOUND * max(|A||B|^T)           (test_gpu_gemm.py)
DB_BOUND = 1e-6                     # db: max|err| <= DB_BOUND * max sum|dY| + 1e-6    (test_gpu_gemm.py)
LONG_T = 100000                     # longest token count test_gpu_gemm.py bounds with GEMM_BOUND; past it, FLOOR
HEAD_FWD_BOUND = 1e-5               # logits: |err| <= HEAD_FWD_BOUND * (sum |basic q| + 1)   (test_gpu_unit_embed_fused.py)
HEAD_BWD_BOUND = 2e-6               # s:      |err| <= HEAD_BWD_BOUND * (sum |dl basic| + 1)
QW = 7 * C


def _lib():
    from dotaclient_b200 import _lib as lib_mod
    return lib_mod, lib_mod.load()


def _canary(*shape):
    return torch.full(shape, CANARY, dtype=torch.int32, device=DEV).view(torch.float32)


def _same(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _untouched(t):
    return bool((t.view(torch.int32) == CANARY).all())


def _count(n):
    return torch.tensor([n], dtype=torch.int32, device=DEV)


def _row_list(M, count, order, seed):
    """-> (rows [M] int32 on the GPU, n = min(count, M)): n distinct rows of range(M), ascending (as dc_target_rows lists
    them) or shuffled, then the spare row M."""
    n = min(count, M)
    pick = torch.randperm(M, generator=torch.Generator().manual_seed(seed))[:n]
    if order == "ascending":
        pick = pick.sort().values
    rows = torch.full((M,), M, dtype=torch.int32)
    rows[:n] = pick.to(torch.int32)
    return rows.to(DEV), n


def _listed(rows, n, size):
    """Bool [size]: the rows rows[:n]."""
    m = torch.zeros(size, dtype=torch.bool, device=DEV)
    m[rows[:n].long()] = True
    return m


# ---------------------------------------------------------------------------------------------------------- dc_target_rows
def _patterns(N, rng):
    """(name, mask, action) [N, 40] uint8 patterns at the 1024-token block edges of target_rows_kernel."""
    z = lambda: np.zeros((N, 40), np.uint8)                        # noqa: E731
    tok = np.arange(N)
    out = [("none", z(), z()), ("all", np.ones((N, 40), np.uint8), np.ones((N, 40), np.uint8))]
    m = z(); m[0, 5] = 1; out.append(("first only", m, z()))
    a = z(); a[N - 1, 0] = 1; out.append(("last only", z(), a))
    edges = [t for k in range(1024, N, 1024) for t in (k - 1, k)] + [N - 1]
    m = z(); m[edges, 17] = 1; out.append(("block edges", m, z()))
    for parity in (0, 1):
        m = z(); m[(tok // 1024) % 2 == parity, 3] = 1; out.append(("blocks %d" % parity, m, z()))
    m, a = z(), z()
    m[rng.random(N) < 0.3, 39] = 1                                 # byte 39 only: the last uint2 row_any reads
    m[N - 1, 39] = 1
    a[rng.random(N) < 0.3, 39] = 1
    out.append(("byte 39", m, a))
    kind = rng.integers(0, 4, N)                                   # none, mask only, action only, both
    col = rng.integers(0, 40, N)
    m, a = z(), z()
    m[tok[kind & 1 == 1], col[kind & 1 == 1]] = 1
    a[tok[kind & 2 == 2], col[kind & 2 == 2]] = 1
    out.append(("mask / action only", m, a))
    return out


@pytest.mark.parametrize("N", [1, 3, 1023, 1024, 1025, 4097, 131075])
def test_target_rows_at_block_edges(N):
    """rows[:count], count and flags against numpy, on a view at the start of its allocation and on one 40 bytes in; the
    rows around the view hold 0xff, so a read outside it would add a token; rows past the count keep their canary."""
    lib_mod, lib = _lib()
    rng = np.random.default_rng(N)
    ws = torch.empty(int(lib.dc_target_rows_workspace_bytes(N)), dtype=torch.uint8, device=DEV)
    for name, m, a in _patterns(N, rng):
        want_flags = (m | a).any(1)
        want_rows = np.nonzero(want_flags)[0].astype(np.int32)
        for off in (0, 1):
            bufs = []
            for src in (m, a):
                buf = torch.full(((N + 1) * 40,), 0xFF, dtype=torch.uint8)
                buf[off * 40:(off + N) * 40] = torch.from_numpy(src.reshape(-1))
                bufs.append(buf.to(DEV))
            mv, av = (b[off * 40:(off + N) * 40] for b in bufs)
            results = []
            for _ in range(2):
                rows = torch.full((N,), CANARY, dtype=torch.int32, device=DEV)
                count = torch.full((1,), -5, dtype=torch.int32, device=DEV)
                flags = torch.full((N,), 0xAB, dtype=torch.uint8, device=DEV)
                lib_mod.check(lib.dc_target_rows(mv.data_ptr(), av.data_ptr(), N, rows.data_ptr(), count.data_ptr(),
                                                 flags.data_ptr(), ws.data_ptr(), lib_mod.stream_ptr()), "dc_target_rows")
                results.append((rows.cpu(), count.cpu(), flags.cpu()))
            rows, count, flags = results[0]
            n = int(count)
            what = "%s, offset %d" % (name, off)
            assert n == want_rows.size, what
            assert np.array_equal(rows[:n].numpy(), want_rows), what
            assert (rows[n:] == CANARY).all(), what
            assert np.array_equal(flags.numpy(), want_flags.astype(np.uint8)), what
            assert all(torch.equal(x, y) for x, y in zip(results[0], results[1])), what


# --------------------------------------------------------------------------------------------------- dc_rows_zero_inactive
@pytest.mark.parametrize("N", [1, 31, 33, 131075])
@pytest.mark.parametrize("width,ld", [(40, 40), (192, 192), (128, 896)])
def test_rows_zero_inactive(N, width, ld):
    """Only the first `width` columns of the rows whose flag is 0 become +0.0; active rows and the columns past `width`
    keep their canary."""
    lib_mod, lib = _lib()
    g = torch.Generator().manual_seed(N + width)
    for flags in ((torch.rand(N, generator=g) < 0.5), torch.zeros(N, dtype=torch.bool), torch.ones(N, dtype=torch.bool)):
        f = flags.to(torch.uint8).to(DEV)
        dst = _canary(N, ld)
        lib_mod.check(lib.dc_rows_zero_inactive(f.data_ptr(), N, dst.data_ptr(), ld, width, lib_mod.stream_ptr()),
                      "dc_rows_zero_inactive")
        want = torch.full((N, ld), CANARY, dtype=torch.int32, device=DEV)
        want[~flags.to(DEV), :width] = 0
        assert torch.equal(dst.view(torch.int32), want)


# ----------------------------------------------------------------------------------------------------- dc_gemm_tf32x3_rows
# (K, N, gather, bias, relu, outputs, pitch padding): the four GEMMs of TargetUnitRows -- att_c / att (K = H, gather, C and
# C_rows), q_c (K = 128, N = 896), d_att_c (K = 896), dy (N = H, scatter only) -- and variants of the first.  K <= 128 runs
# the weight-stationary kernel (64-row tiles), K > 128 the streaming kernel (128-row tiles).
GEMM_SHAPES = {
    "att-h64": (64, 128, True, True, False, "both", 0),
    "att-h128": (128, 128, True, True, False, "both", 0),
    "att-h192": (192, 128, True, True, False, "both", 0),
    "att-h256": (256, 128, True, True, False, "both", 0),
    "att-h512": (512, 128, True, True, False, "both", 0),
    "att-h64-relu": (64, 128, True, True, True, "both", 0),
    "att-h256-relu": (256, 128, True, True, True, "both", 0),
    "att-h128-C": (128, 128, True, True, False, "C", 32),
    "att-h128-Crows": (128, 128, True, True, False, "C_rows", 32),
    "att-h256-C": (256, 128, True, False, False, "C", 32),
    "att-h256-Crows": (256, 128, True, False, False, "C_rows", 32),
    "q_c": (128, 896, False, False, False, "C", 0),
    "d_att_c": (896, 128, False, False, False, "C", 0),
    "dy-h128": (128, 128, False, False, False, "C_rows", 0),
    "dy-h192": (128, 192, False, False, False, "C_rows", 0),
}
GEMM_M = 5000
GEMM_COUNTS = (0, 1, 63, 64, 65, 127, 128, 129, GEMM_M - 1, GEMM_M, GEMM_M + 7)


def _gemm_operands(shape, M, seed):
    K, N, gather, has_bias = GEMM_SHAPES[shape][:4]
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M + 1 if gather else M, K, generator=g, device=DEV)
    b = torch.randn(N, K, generator=g, device=DEV) * 0.3
    bias = torch.randn(N, generator=g, device=DEV) if has_bias else None
    return a, b, bias


def _gemm_rows(shape, a, b, bias, rows, count, M):
    """One dc_gemm_tf32x3_rows call into fresh canary outputs -> (C [M, ld] or None, C_rows [M + 1, ld] or None)."""
    K, N, gather, _, relu, outs, pad = GEMM_SHAPES[shape]
    lib_mod, lib = _lib()
    ld = N + pad
    c = _canary(M, ld) if outs != "C_rows" else None
    c_rows = _canary(M + 1, ld) if outs != "C" else None
    lib_mod.check(lib.dc_gemm_tf32x3_rows(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), lib_mod.ptr(bias), lib_mod.ptr(c),
                                          lib_mod.ptr(c_rows), ld, M, count.data_ptr(), rows.data_ptr(), 1 if gather else 0, N, K,
                                          1 if relu else 0, lib_mod.stream_ptr()), "dc_gemm_tf32x3_rows")
    return c, c_rows


def _f64_product(a, b, bias, relu):
    out = a.double() @ b.double().t()
    if bias is not None:
        out = out + bias.double()
    return out.clamp_min(0) if relu else out


def _gemm_failures(shape, outs, rows, n, ref):
    """What is wrong with the outputs (C, C_rows) of n listed rows against `ref` (the plain GEMM on the gathered rows)."""
    N = GEMM_SHAPES[shape][1]
    bad = []
    for name, out in zip(("C", "C_rows"), outs):
        if out is None:
            continue
        written = torch.zeros(out.shape[0], dtype=torch.bool, device=DEV)
        if name == "C":
            written[:n] = True
        else:
            written[rows[:n].long()] = True
        got = out[:n] if name == "C" else out[rows[:n].long()]
        if n and not _same(got[:, :N], ref):
            bad.append("%s differs from dc_gemm_tf32x3 on the listed rows" % name)
        if not _untouched(out[~written]):
            bad.append("%s: a row that is not listed was written" % name)
        if not _untouched(out[written][:, N:]):
            bad.append("%s: a column past N was written" % name)
    return bad


def _gemm_case(shape, M, count, order, seed, controls=False):
    """-> max|err| / bound against float64 (0 at count 0)."""
    from dotaclient_b200 import ops
    _, N, gather, _, relu = GEMM_SHAPES[shape][:5]
    a0, b, bias = _gemm_operands(shape, M, seed)
    rows, n = _row_list(M, count, order, seed + count)
    a = a0.clone()
    if gather:
        a[~_listed(rows, n, M + 1)] = float("nan")                 # rows not listed (the spare row M included)
    else:
        a[n:] = float("nan")                                       # rows past the count
    cnt = _count(count)
    got = _gemm_rows(shape, a, b, bias, rows, cnt, M)
    again = _gemm_rows(shape, a, b, bias, rows, cnt, M)
    what = "%s M %d count %d %s" % (shape, M, count, order)
    assert all(x is None or _same(x, y) for x, y in zip(got, again)), what + ": not repeatable"
    ac = (a0[rows[:n].long()] if gather else a0[:n]).contiguous()
    ref = ops.gemm_tf32x3(ac, b, bias, relu=relu) if n else None
    assert not _gemm_failures(shape, got, rows, n, ref), (what, _gemm_failures(shape, got, rows, n, ref))
    if n == 0:
        return 0.0
    compact = got[0][:n, :N] if got[0] is not None else got[1][rows[:n].long(), :N]
    f64 = _f64_product(ac, b, bias, relu)
    lim = GEMM_BOUND * float((ac.double().abs() @ b.double().abs().t()).max())
    err = float((compact.double() - f64).abs().max())
    assert err <= lim, (what, err, lim)
    if controls:
        # the result at count - 1 fails the bitwise checks, one extra row fails the canaries, single-pass TF32 the bound
        short = _gemm_rows(shape, a, b, bias, rows, _count(n - 1), M)
        assert _gemm_failures(shape, short, rows, n, ref), what + ": the result at count - 1 passed"
        extra = [None if x is None else x.clone() for x in got]
        spare = M if extra[1] is not None else n                   # C_rows: the spare row; C: the row at the count
        (extra[1] if extra[1] is not None else extra[0])[spare] = 0.0
        assert _gemm_failures(shape, extra, rows, n, ref), what + ": an extra row passed the canaries"
        tf = _f64_product(tf32_rna(ac), tf32_rna(b), bias, relu)
        assert float((tf - f64).abs().max()) > lim, what + ": single-pass TF32 passed the float64 bound"
    return err / lim


@pytest.mark.parametrize("shape", list(GEMM_SHAPES))
def test_gemm_rows_at_tile_edges(shape):
    worst = max(_gemm_case(shape, GEMM_M, c, order, 1000 + i, controls=(c == 65))
                for i, c in enumerate(GEMM_COUNTS) for order in ("ascending", "shuffled"))
    print("\n%s: max|err| / bound %.3f" % (shape, worst))


@pytest.mark.parametrize("shape", ["att-h128", "att-h512", "q_c", "d_att_c", "dy-h192"])
def test_gemm_rows_every_token_at_benchmark_rows(shape):
    """c2's 131,072 tokens, all of them listed."""
    M = 131072
    worst = max(_gemm_case(shape, M, M, order, 7) for order in ("ascending", "shuffled"))
    print("\n%s M %d: max|err| / bound %.3f" % (shape, M, worst))


# ----------------------------------------------------------------------------------------------- dc_gemm_wgrad_tf32x3_rows
WGRAD_COUNTS = (0, 1, 31, 32, 33, 4095, 4096, 4097)


def _wgrad_rows(dy, x, x_rows, count, dw, db, accumulate):
    from dotaclient_b200 import ops
    ops.gemm_wgrad_tf32x3(dy, x, dw_out=dw, db_out=db, accumulate=accumulate, t_dev=_count(count), x_rows=x_rows)
    return dw, db


def _wgrad_case(dy0, x0, T, count, order, seed, controls=False):
    """-> (max|err| / bound of dW, of db) against float64 ((0, 0) at count 0)."""
    from dotaclient_b200 import ops
    No, Ni = dy0.shape[1], x0.shape[1]
    what = "No %d Ni %d T %d count %d %s" % (No, Ni, T, count, order)
    if order == "identity":                                        # x_rows NULL: token t reads X row t
        rows, n = None, min(count, T)
        x = x0[:T].clone()
        x[n:] = float("nan")
        xg = x0[:n]
    else:
        rows, n = _row_list(T, count, order, seed)
        x = x0.clone()
        x[~_listed(rows, n, T + 1)] = float("nan")
        xg = x0[rows[:n].long()]
    dy = dy0.clone()
    dy[n:] = float("nan")
    base_w = torch.randn(No, Ni, device=DEV)
    base_b = torch.randn(No, device=DEV)
    dw, db = _wgrad_rows(dy, x, rows, count, _canary(No, Ni), _canary(No), False)
    dw2, db2 = _wgrad_rows(dy, x, rows, count, _canary(No, Ni), _canary(No), False)
    assert _same(dw, dw2) and _same(db, db2), what + ": not repeatable"
    acc_w, acc_b = _wgrad_rows(dy, x, rows, count, base_w.clone(), base_b.clone(), True)
    if n == 0:
        assert not dw.view(torch.int32).any() and not db.view(torch.int32).any(), what + ": dW / db not +0.0"
        assert _same(acc_w, base_w) and _same(acc_b, base_b), what + ": accumulate changed the gradient"
        return 0.0, 0.0
    ref_w, ref_b = ops.gemm_wgrad_tf32x3(dy0[:n].contiguous(), xg.contiguous())
    assert _same(dw, ref_w) and _same(db, ref_b), what + ": differs from dc_gemm_wgrad_tf32x3 at T = count"
    dense_w, dense_b = ops.gemm_wgrad_tf32x3(dy0[:n].contiguous(), xg.contiguous(), dw_out=base_w.clone(), db_out=base_b.clone(),
                                             accumulate=True)
    assert _same(acc_w, dense_w) and _same(acc_b, dense_b), what + ": accumulation differs from dc_gemm_wgrad_tf32x3"
    d64, x64 = dy0[:n].double(), xg.double()
    f64 = d64.t() @ x64
    lim = FLOOR * float(f64.abs().max()) if n > LONG_T else GEMM_BOUND * float((d64.abs().t() @ x64.abs()).max())
    err = float((dw.double() - f64).abs().max())
    assert err <= lim, (what, err, lim)
    lim_b = DB_BOUND * float(d64.abs().sum(0).max()) + 1e-6
    err_b = float((db.double() - d64.sum(0)).abs().max())
    assert err_b <= lim_b, (what, err_b, lim_b)
    if controls:
        short = _wgrad_rows(dy, x, rows, n - 1, _canary(No, Ni), _canary(No), False)
        assert not (_same(short[0], ref_w) and _same(short[1], ref_b)), what + ": the result at count - 1 passed"
        tf = tf32_rna(dy0[:n]).double().t() @ tf32_rna(xg).double()
        assert float((tf - f64).abs().max()) > lim, what + ": single-pass TF32 passed the float64 bound"
    return err / lim, err_b / lim_b


@pytest.mark.parametrize("T", [5000, 131072])
@pytest.mark.parametrize("Ni", [128, 192, 512])
def test_wgrad_rows_at_chunk_edges(T, Ni):
    """dW / db of the tokens t < count (X row x_rows[t]): counts at the 32-row chunks and the 4096-row accumulator flush,
    T and T + 7 (clamped); X through an ascending, a shuffled and no row list."""
    g = torch.Generator(device=DEV).manual_seed(T + Ni)
    dy0 = torch.randn(T, 128, generator=g, device=DEV)
    x0 = torch.randn(T + 1, Ni, generator=g, device=DEV)
    worst_w = worst_b = 0.0
    for i, count in enumerate(WGRAD_COUNTS + (T, T + 7)):
        for order in ("ascending", "shuffled", "identity"):
            rw, rb = _wgrad_case(dy0, x0, T, count, order, 2000 + i, controls=(order == "shuffled" and count in (33, T)))
            worst_w, worst_b = max(worst_w, rw), max(worst_b, rb)
    print("\nwgrad Ni %d T %d: max|err| / bound dW %.3f db %.3f" % (Ni, T, worst_w, worst_b))


# --------------------------------------------------------------------------------- dc_target_unit_q_fwd_rows / _bwd_rows
HEAD_COUNTS = (0, 1, 7, 8, 9)


def _head_call(fwd, src, units, w_b, b_b, out, N, rows, count):
    lib_mod, lib = _lib()
    ptrs = (lib_mod._c.c_void_p * 6)(*[u.data_ptr() for u in units])
    if rows is None:
        if fwd:
            rc = lib.dc_target_unit_q_fwd(src.data_ptr(), QW, ptrs, w_b.data_ptr(), b_b.data_ptr(), out.data_ptr(), N,
                                          lib_mod.stream_ptr())
        else:
            rc = lib.dc_target_unit_q_bwd(src.data_ptr(), ptrs, w_b.data_ptr(), b_b.data_ptr(), out.data_ptr(), QW, N,
                                          lib_mod.stream_ptr())
    elif fwd:
        rc = lib.dc_target_unit_q_fwd_rows(src.data_ptr(), QW, ptrs, w_b.data_ptr(), b_b.data_ptr(), out.data_ptr(), N,
                                           rows.data_ptr(), count.data_ptr(), lib_mod.stream_ptr())
    else:
        rc = lib.dc_target_unit_q_bwd_rows(src.data_ptr(), ptrs, w_b.data_ptr(), b_b.data_ptr(), out.data_ptr(), QW, N,
                                           rows.data_ptr(), count.data_ptr(), lib_mod.stream_ptr())
    lib_mod.check(rc, "target-unit head")
    return out


def _sample_items(n, seed, extra=192):
    fixed = {0, 1, 7, 8, 9, n // 2, n - 1}
    pick = torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:extra].tolist()
    return torch.tensor(sorted(i for i in fixed | set(pick) if 0 <= i < n), dtype=torch.long, device=DEV)


def _head_fwd64(units, w_b, b_b, q, tokens):
    """-> (float64 logits [s, 40] of `tokens` from q rows [s, 896], the scale sum |basic q| + 1)."""
    ref = torch.zeros(tokens.numel(), 40, dtype=torch.float64, device=DEV)
    scale = torch.ones_like(ref)
    q64 = q.double()
    for gi, (nu, off) in enumerate(zip(UNITS, OFFSETS)):
        u = units[gi].view(-1, nu, 12)[tokens].reshape(-1, 12)
        b = _basic64([u], w_b, b_b)[0].view(-1, nu, C)
        qg = q64[:, gi * C:(gi + 1) * C]
        ref[:, off:off + nu] = torch.einsum("nuc,nc->nu", b, qg) + q64[:, 6 * C + gi:6 * C + gi + 1]
        scale[:, off:off + nu] += torch.einsum("nuc,nc->nu", b, qg.abs())
    return ref, scale


def _head_case(N, base, count, order, seed, controls=False):
    """-> (max over the sampled items of |err| / bound, forward and backward) against float64."""
    units0, w_b, b_b, q0, dl0 = base
    rows, n = _row_list(N, count, order, seed)
    what = "head N %d count %d %s" % (N, count, order)
    listed = _listed(rows, n, N + 1)
    units = [u.clone() for u in units0]
    for u, nu in zip(units, UNITS):
        u.view(N + 1, nu, 12)[~listed] = float("nan")              # tokens not listed, the spare token N included
    sel = rows[:n].long()
    cnt = _count(count)
    # forward: item i reads q_c row i, writes logits row rows[i]
    q_c = q0[:N].clone()
    q_c[n:] = float("nan")
    lg = _head_call(True, q_c, units, w_b, b_b, _canary(N + 1, 40), N, rows, cnt)
    lg2 = _head_call(True, q_c, units, w_b, b_b, _canary(N + 1, 40), N, rows, cnt)
    assert _same(lg, lg2), what + ": forward not repeatable"
    q_d = torch.full((N + 1, QW), float("nan"), device=DEV)
    q_d[sel] = q0[:n]
    dense = _head_call(True, q_d, units, w_b, b_b, torch.empty(N + 1, 40, device=DEV), N + 1, None, None)

    def fwd_failures(out):
        bad = []
        if not _same(out[sel], dense[sel]):
            bad.append("logits differ from dc_target_unit_q_fwd on the listed tokens")
        if not _untouched(out[~listed]):
            bad.append("a logit row of a token that is not listed was written")
        return bad

    assert not fwd_failures(lg), (what, fwd_failures(lg))
    # backward: item i reads dlogits row rows[i], writes s row i; a listed token whose dlogits are zero gets a zero row
    dl = dl0.clone()
    dl[~listed] = float("nan")
    s = _head_call(False, dl, units, w_b, b_b, _canary(N, QW), N, rows, cnt)
    s2 = _head_call(False, dl, units, w_b, b_b, _canary(N, QW), N, rows, cnt)
    assert _same(s, s2), what + ": backward not repeatable"
    s_d = _head_call(False, dl, units, w_b, b_b, _canary(N + 1, QW), N + 1, None, None)

    def bwd_failures(out):
        bad = []
        if not _same(out[:n], s_d[sel]):
            bad.append("s differs from dc_target_unit_q_bwd on the listed tokens")
        if not _untouched(out[n:]):
            bad.append("an s row past the count was written")
        return bad

    assert not bwd_failures(s), (what, bwd_failures(s))
    zero = (dl0[sel] == 0).all(1)
    assert not s[:n][zero].view(torch.int32).any(), what + ": a listed token with zero dlogits has no +0.0 row"
    if n == 0:
        return 0.0, 0.0
    items = _sample_items(n, seed)
    tokens = sel[items]
    f64, scale = _head_fwd64(units0, w_b, b_b, q0[:n][items], tokens)
    rf = float(((lg[tokens].double() - f64).abs() / (HEAD_FWD_BOUND * scale)).max())
    assert rf <= 1.0, (what, rf)
    link = {"units": units0, "w_b": w_b, "b_b": b_b}
    s64 = _s_f64(link, dl0, tokens)
    s_scale = _s_f64(link, dl0.abs(), tokens) + 1.0
    rb = float(((s[items].double() - s64).abs() / (HEAD_BWD_BOUND * s_scale)).max())
    assert rb <= 1.0, (what, rb)
    if controls:
        short = _head_call(True, q_c, units, w_b, b_b, _canary(N + 1, 40), N, rows, _count(n - 1))
        assert fwd_failures(short), what + ": the forward at count - 1 passed"
        short = _head_call(False, dl, units, w_b, b_b, _canary(N, QW), N, rows, _count(n - 1))
        assert bwd_failures(short), what + ": the backward at count - 1 passed"
        extra = lg.clone()
        extra[N] = 0.0                                             # the spare token's row
        assert fwd_failures(extra), what + ": an extra logit row passed the canaries"
        extra = s.clone()
        extra[n] = 0.0                                             # the row at the count
        assert bwd_failures(extra), what + ": an extra s row passed the canaries"
        tf, _ = _head_fwd64(units0, w_b, b_b, tf32_rna(q0[:n][items]), tokens)
        assert float(((tf - f64).abs() / (HEAD_FWD_BOUND * scale)).max()) > 1.0, what + ": TF32 q passed the bound"
        tfs = _s_f64(link, tf32_rna(dl0), tokens)
        assert float(((tfs - s64).abs() / (HEAD_BWD_BOUND * s_scale)).max()) > 1.0, what + ": TF32 dlogits passed the bound"
    return rf, rb


@pytest.mark.parametrize("N", [3001, 131072])
def test_head_rows_at_warp_edges(N):
    """Counts at the 8-warp block edges and every token; at 131,072 the grid is capped and the loop over listed tokens wraps."""
    _, units, w_b, b_b, q = _head_inputs(N, N + 1)
    dl = torch.randn(N + 1, 40, generator=torch.Generator().manual_seed(N)).to(DEV)
    dl[::3] = 0.0                                                  # tokens whose dlogits are all zero
    dl[1::3, :20] = 0.0                                            # ... and partly zero
    base = (units, w_b, b_b, q, dl)
    worst_f = worst_b = 0.0
    for i, count in enumerate(HEAD_COUNTS + (N,)):
        for order in ("ascending", "shuffled"):
            rf, rb = _head_case(N, base, count, order, 3000 + i, controls=(count == 9 and order == "shuffled"))
            worst_f, worst_b = max(worst_f, rf), max(worst_b, rb)
    print("\nhead N %d: max|err| / bound forward %.3f backward %.3f" % (N, worst_f, worst_b))


# ------------------------------------------------------------------------------------------------ the whole TargetUnitRows
@pytest.mark.parametrize("H,cell,S,B,frac", [(128, "lstm", 64, 64, 1.0), (64, "gru", 64, 64, 0.5), (192, "lstm", 64, 32, 0.25),
                                             (512, "gru", 32, 64, 0.5), (512, "lstm", 32, 32, 1.0)])
def test_compact_matches_dense_every_token_and_widths(H, cell, S, B, frac):
    """test_compact_matches_dense's checks with every token active (count = N) and at H = 64 (att GEMM K = 64, 2 k-chunks),
    192 (dy at a ragged N = 192) and 512 (att on the streaming kernel)."""
    _compact_matches_dense(H, cell, S, B, frac)


def _masks_count(S, B, n, seed):
    """target_unit (mask, action) rows [S, B, 40] on the GPU with exactly n active tokens; an active token has a mask row,
    an action row or both."""
    g = torch.Generator().manual_seed(seed)
    act = torch.zeros(S * B, dtype=torch.bool)
    act[torch.randperm(S * B, generator=g)[:n]] = True
    act = act.view(S, B, 1)
    col = torch.randint(0, 40, (S, B, 1), generator=g)
    hit = torch.zeros(S, B, 40, dtype=torch.bool).scatter_(2, col, True) & act
    side = torch.rand(S, B, 1, generator=g)
    return (hit & (side < 0.7)).cuda(), (hit & (side > 0.3)).cuda()


@pytest.mark.parametrize("H", [128, 192])
def test_graph_replay_rising_and_falling_counts(H):
    """One captured forward + backward of the compact branch, replayed at counts N, 1, 0, 129, N/2, N: each replay equals an
    eager run on the same inputs bit for bit, so no row of an earlier, larger count survives into a later one."""
    pol = _policy(H, "lstm")
    S, B = 64, 64
    N = S * B
    obs = _obs(S, B, 9)
    link = dict(pol._encode(obs['env'], [obs[k] for k in pol.INPUT_KEYS[1:]])[1])
    y = (torch.randn(S, B, H, generator=torch.Generator().manual_seed(3)) * 0.5).cuda()
    counts = (N, 1, 0, 129, N // 2, N)
    inputs = [_masks_count(S, B, c, 40 + i) for i, c in enumerate(counts)]
    dls = [torch.randn(S, B, 40, generator=torch.Generator().manual_seed(50 + i)).cuda() * (m | a).any(-1, keepdim=True)
           for i, (m, a) in enumerate(inputs)]
    w, b = pol.affine_unit_attention.weight, pol.affine_unit_attention.bias
    from dotaclient_b200 import encoder_ops

    def step(mask, action, dl):
        w.grad = b.grad = None
        yy = y.detach().requires_grad_(True)
        rows, count, flags = encoder_ops.target_rows(mask, action)
        lg = encoder_ops.target_unit_rows(yy, w, b, link, rows, count, flags)
        lg.backward(dl)
        link.pop("pending", None)
        return lg.detach().clone(), yy.grad.clone(), w.grad.clone(), b.grad.clone(), count.clone()

    eager = [step(m, a, d) for (m, a), d in zip(inputs, dls)]
    assert [int(e[4]) for e in eager] == list(counts)
    sm, sa, sd = (t.clone() for t in (*inputs[0], dls[0]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(sm, sa, sd)                                           # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step(sm, sa, sd)
    for c, (m, a), d, want in zip(counts, inputs, dls, eager):
        sm.copy_(m), sa.copy_(a), sd.copy_(d)
        graph.replay()
        torch.cuda.synchronize()
        for name, got, exp in zip(("logits", "dy", "dW_att", "db_att", "count"), out, want):
            assert _same(got, exp), "count %d: %s differs from the eager run" % (c, name)
