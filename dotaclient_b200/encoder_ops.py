"""Autograd wrappers of the unit encoder and the target-unit head (``policy.py:99-136,144-153``).

Forward and backward are explicit chains of C-ABI kernels -- the fp32-accurate tensor-core GEMMs of
``csrc/gemm_tf32x3.cu`` for the 128x128 unit embeddings and the bandwidth kernels of ``csrc/encoder.cu`` around them --
neither pass materialises the [N, 40, 128] unit embedding or its gradient: forward has the max-pool in the embedding GEMM's
epilogue and the target-unit head through ``att W_g``; backward generates the max-pool routing inside the weight- and
data-gradient kernels and takes the head's rank-1 share through token-level products.
"""
import torch

from . import _lib
from .ops import PROFILE, _f32c, _need_cuda, _u8, gemm_tf32x3, gemm_wgrad_supported, gemm_wgrad_tf32x3

UNITS = (1, 5, 16, 16, 1, 1)              # allied/enemy heroes, allied/enemy non-heroes, allied/enemy towers
OFFSETS = (0, 1, 6, 22, 38, 39)
MAX_UNITS = 40
C = 128
XCAT = 7 * C                               # pre-rnn input row: env encoding + six group maxima (policy.py:129-136)

_basic_ws = {}


def _basic_workspace(device):
    ws = _basic_ws.get(device)
    if ws is None:
        ws = torch.empty(int(_lib.load().dc_unit_basic_bwd_workspace_bytes()), dtype=torch.uint8, device=device)
        _basic_ws[device] = ws
    return ws


_env_ws = {}


def _env_workspace(device):
    ws = _env_ws.get(device)
    if ws is None:
        ws = torch.empty(int(_lib.load().dc_env_bwd_workspace_bytes()), dtype=torch.uint8, device=device)
        _env_ws[device] = ws
    return ws


_wgrad_ws = {}


def _wgrad_workspace(No, Ni, device):
    key = (No, Ni, device)
    ws = _wgrad_ws.get(key)
    if ws is None:
        ws = torch.empty(int(_lib.load().dc_gemm_wgrad_workspace_bytes(No, Ni)), dtype=torch.uint8, device=device)
        _wgrad_ws[key] = ws
    return ws


# The unit embedding [N, 40, 128] (policy.py:130-131) is never materialised in the forward pass, and the basic layer
# basic = relu(units W_b^T + b_b) that feeds it is rebuilt from the 12 raw features of a unit wherever it is read.  The consumers are
#   * the max-pool: one launch per group (dc_unit_embed_fwd) whose producers generate `basic` into the embedding GEMM's operand
#     ring and whose epilogue keeps max + arg-max per token and channel; for the 1-unit groups the plain epilogue writes the
#     group's slot of the pre-rnn row.  The enemy-tower group runs nothing in forward because policy.py:127 takes that slot's
#     maximum from the enemy non-heroes.  `basic` of groups 0-4 and its ReLU mask (16 bytes per unit row) are stored by the same
#     launch only when a backward may follow: the weight gradients below read `basic`, the data gradient the mask;
#   * the target-unit head, which is linear in it: logits[n,u] = <att[n] W_g, basic[n,u]> + <att[n], b_g>  (TargetUnit below,
#     `basic` regenerated from the raw features in the head kernels).
# In backward the embedding's gradient d_emb[n,u,:] has two sources -- the head (rank 1: dlogits[n,u] * att[n,:], arrives first) and the
# max-pool routing R (d_xmax[n,:] to the arg-max unit of every channel; arrives with the pre-rnn gradient, after the recurrence).
# TargetUnit parks (dlogits, att, s) in the `link` cell the two Functions of one graph share; UnitEncoder.backward then needs no
# dense [N, 40, 128] tensor at all:
#   dW_g  = R^T basic_g  (dc_unit_wgrad_routed: R generated in the dY^T producer)  +  att^T s_g   (one token-level GEMM for all groups,
#           s_g = sum_u dlogits_u basic_u from dc_target_unit_q_bwd; its bias block gives the head's share of db_g)
#   dW_b += (relu'(.) (R + dlogits x att) W_g)^T units   (dc_unit_dgrad_fused_mask: d_emb generated in the producers, the ReLU mask
#           the forward stored -- recomputed for the enemy towers, which have no forward launch -- and dW_b as a second tensor-core
#           product from the masked accumulator) -- d_basic never exists either.


def _ptr(t, float_offset=0):
    return t.data_ptr() + 4 * float_offset


def _ptr6(tensors):
    return (_lib._c.c_void_p * 6)(*[t.data_ptr() for t in tensors])


class UnitEncoder(torch.autograd.Function):
    """(env, w_e, b_e, w_b, b_b, units x6, W_g x6, b_g x6) -> the pre-rnn input row ``[..., 896]`` = relu(affine_env(env))
    followed by the six group maxima, written in place by the kernels (no cat, no ``[N, 40, 128]`` embedding).

    maxima slot 5 (enemy towers) is a copy of slot 3 (enemy non-heroes): the reference's ``policy.py:127``.
    ``link`` (a dict) receives the raw unit features, the basic layer's and the embedding weights for the target-unit head.
    ``wait``: see ``unit_encoder``.  ``need_grad``: a backward may follow, so the basic activations of groups 0-4 are stored
    for the weight gradients and their ReLU masks for the data gradient (without it nothing of the basic layer reaches HBM).
    """

    @staticmethod
    def forward(ctx, link, wait, need_grad, env, w_e, b_e, w_b, b_b, *rest):
        units, weights, biases = rest[:6], rest[6:12], rest[12:18]
        ctx.link = link
        _need_cuda(env, w_b, *units)
        lib = _lib.load()
        st = _lib.stream_ptr()
        lead = units[0].shape[:-2]
        N = 1
        for d in lead:
            N *= d
        dev = units[0].device
        w_b, b_b = _f32c(w_b.detach()), _f32c(b_b.detach())
        units = [_f32c(u.detach()).reshape(N * n, 12) for u, n in zip(units, UNITS)]
        units = [u if u.data_ptr() % 16 == 0 else u.clone() for u in units]   # the backward kernels read whole rows as 3 x 16 bytes
        weights = [_f32c(w.detach()) for w in weights]
        biases = [_f32c(b.detach()) for b in biases]
        xcat = torch.empty((N, XCAT), dtype=torch.float32, device=dev)
        argmax = torch.zeros((5, N, C), dtype=torch.uint8, device=dev)         # 1-unit groups: the maximum is unit 0
        env2 = _f32c(env.detach()).reshape(N, 3)
        w_e, b_e = _f32c(w_e.detach()), _f32c(b_e.detach())
        if wait is not None:
            wait(env2)
        with PROFILE.span("env_fwd", 1, 4 * N * (3 + C)):
            _lib.check(lib.dc_env_fwd(env2.data_ptr(), w_e.data_ptr(), b_e.data_ptr(), xcat.data_ptr(), XCAT, N, st), "dc_env_fwd")
        basics, masks = [], []
        for g, n_u in enumerate(UNITS):
            R = N * n_u
            if wait is not None:                      # this group's observations may still be in flight over PCIe
                wait(units[g])
            if g == 5:                                # policy.py:127: the enemy-tower maximum is never used
                continue
            # basic layer + embedding GEMM in one launch: the max-pool epilogue, or for one unit the embedding IS the maximum
            # and goes straight into its slot
            basic = torch.empty((R, C), dtype=torch.float32, device=dev) if need_grad else None
            mask = torch.empty((R, 4), dtype=torch.int32, device=dev) if need_grad else None     # bit j/4 of word j%4 of row r: basic[r, j] > 0
            copy = _ptr(xcat, 6 * C) if g == 3 else None
            am = argmax[g].data_ptr() if n_u > 1 else None
            nbytes = 4 * (R * 12 + (R * C + R * 4 if need_grad else 0) + C * C + N * C) + (N * C if n_u > 1 else 0)
            with PROFILE.span("gemm_unit_max" if n_u > 1 else "gemm_tf32x3", 1, nbytes):
                _lib.check(lib.dc_unit_embed_fwd_mask(units[g].data_ptr(), w_b.data_ptr(), b_b.data_ptr(), _lib.ptr(basic), _lib.ptr(mask),
                                                      weights[g].data_ptr(), biases[g].data_ptr(), _ptr(xcat, (g + 1) * C), copy, XCAT,
                                                      am, N, n_u, st), "dc_unit_embed_fwd_mask")
            basics.append(basic)
            masks.append(mask)
        link["units"], link["w_b"], link["b_b"] = units, w_b, b_b
        link["weights"], link["biases"] = weights, biases
        ctx.N = N
        ctx.lead = lead
        ctx.save_for_backward(argmax, *units, *basics, *weights, env2, xcat, w_b, b_b, *masks)
        return xcat.view(*lead, XCAT)

    @staticmethod
    def backward(ctx, d_xcat):
        saved = ctx.saved_tensors
        argmax, units, basics, weights, env2, xcat = saved[0], saved[1:7], saved[7:12], saved[12:18], saved[18], saved[19]
        w_b, b_b, masks = saved[20], saved[21], saved[22:27]
        N = ctx.N
        lib = _lib.load()
        st = _lib.stream_ptr()
        dev = argmax.device
        pending = ctx.link.pop("pending", None)
        d_xcat = _f32c(d_xcat).reshape(N, XCAT)
        dw_e = torch.empty((C, 3), dtype=torch.float32, device=dev)
        db_e = torch.empty(C, dtype=torch.float32, device=dev)
        with PROFILE.span("env_bwd", 2, 4 * N * (2 * C + 3)):
            _lib.check(lib.dc_env_bwd(d_xcat.data_ptr(), xcat.data_ptr(), XCAT, env2.data_ptr(), dw_e.data_ptr(), db_e.data_ptr(),
                                      N, _env_workspace(dev).data_ptr(), st), "dc_env_bwd")
        dl = att = s_head = att_head = count = None
        if pending is not None:
            dl, att, s_head, att_head, count = pending     # att_head / s_head: compact rows when count is set (TargetUnitRows)
        dw_b = torch.empty((C, 12), dtype=torch.float32, device=dev)
        db_b = torch.empty(C, dtype=torch.float32, device=dev)
        dw_all = torch.zeros((6, C, C), dtype=torch.float32, device=dev)     # zeros: the enemy-tower layer has no max-pool path
        db_all = torch.zeros((6, C), dtype=torch.float32, device=dev)
        ws_w = _wgrad_workspace(C, C, dev)
        ws_b = _basic_workspace(dev)
        for g, (n_u, off) in enumerate(zip(UNITS, OFFSETS)):
            R = N * n_u
            routed = g < 5                                 # policy.py:127: enemy towers never reach the maxima
            dx = _ptr(d_xcat, (g + 1) * C) if routed else None
            dx2 = _ptr(d_xcat, 6 * C) if g == 3 else None  # ... their slot was fed from the enemy non-hero maximum
            if routed and n_u > 1:
                with PROFILE.span("gemm_wgrad", 2, 4 * (R * C + C * C + N * C) + N * C):   # dW_g = R^T basic_g, db_g = colsum(R)
                    _lib.check(lib.dc_unit_wgrad_routed(dx, dx2, XCAT, argmax[g].data_ptr(), basics[g].data_ptr(), N, n_u,
                                                        dw_all[g].data_ptr(), db_all[g].data_ptr(), ws_w.data_ptr(), st),
                               "dc_unit_wgrad_routed")
            elif routed:                                   # one unit: the routing is the gradient of the maximum itself
                with PROFILE.span("gemm_wgrad", 2, 4 * (2 * R * C + C * C)):
                    _lib.check(lib.dc_gemm_wgrad_tf32x3(dx, XCAT, basics[g].data_ptr(), C, R, C, C, dw_all[g].data_ptr(), C,
                                                        db_all[g].data_ptr(), 0, ws_w.data_ptr(), st), "dc_gemm_wgrad_tf32x3")
            wt = weights[g].t().contiguous()
            mask = masks[g] if routed else None           # the enemy towers have no forward launch: their mask is recomputed
            with PROFILE.span("unit_dgrad_fused", 2, N * (4 * C + C) * (1 if routed else 0) + 4 * R * 12 + (16 * R if routed else 0)
                              + (4 * N * (C + n_u) if dl is not None else 0)):
                _lib.check(lib.dc_unit_dgrad_fused_mask(dx, dx2, XCAT, argmax[g].data_ptr() if (routed and n_u > 1) else None,
                                                        None if dl is None else _ptr(dl, off), MAX_UNITS, None if att is None else att.data_ptr(),
                                                        wt.data_ptr(), units[g].data_ptr(), _lib.ptr(mask), w_b.data_ptr(), b_b.data_ptr(),
                                                        N, n_u, dw_b.data_ptr(), db_b.data_ptr(), 1 if g > 0 else 0, ws_b.data_ptr(), st),
                           "dc_unit_dgrad_fused_mask")
        if dl is not None:
            # the head's share of every dW_g and db_g in ONE token-level product: att^T [s_0 | ... | s_5 | sum_u dlogits]
            dw_head, _ = gemm_wgrad_tf32x3(att_head, s_head, want_bias=False, t_dev=count, t_host=ctx.link.get("n_active"))
            dw_all += dw_head[:, :6 * C].reshape(C, 6, C).permute(1, 0, 2)
            db_all += dw_head[:, 6 * C:6 * C + 6].t()
        dws, dbs = list(dw_all.unbind(0)), list(db_all.unbind(0))
        return (None, None, None, None, dw_e, db_e, dw_b, db_b) + (None,) * 6 + tuple(dws) + tuple(dbs)


QW = 7 * C     # width of the head's token-level operands: six groups x 128 channels + one block carrying the six bias dots


class TargetUnit(torch.autograd.Function):
    """``logits[..., u] = <attention, unit_embedding[..., u, :]>`` (``policy.py:152-153``) WITHOUT the embedding:
    ``<att, W_g basic_u + b_g> = <att W_g, basic_u> + <att, b_g>``.  One GEMM over tokens produces ``q = att [W_0|..|W_5|b]``
    ``[N, 896]``, a kernel dots it with the ``basic`` rows it rebuilds from the raw unit features.  Backward: ``s_g = sum_u
    dlogits_u basic_u`` (same kernel shape), ``d_att = s [W_0|..|W_5|b]^T`` (one GEMM); the gradient towards the embedding
    weights and the basic layer is finished by ``UnitEncoder.backward`` from (dlogits, att, s) parked in ``link``."""

    @staticmethod
    def forward(ctx, att, link):
        _need_cuda(att)
        units, w_b, b_b = link["units"], link["w_b"], link["b_b"]
        lead = att.shape[:-1]
        N = att.numel() // C
        att2 = _f32c(att.detach()).reshape(N, C)
        dev = att2.device
        bm = _head_matrix(link)
        q = gemm_tf32x3(att2, bm.t().contiguous())                           # [N, 896] = att [W_0 | ... | W_5 | b]
        logits = torch.empty((N, MAX_UNITS), dtype=torch.float32, device=dev)
        with PROFILE.span("target_unit_fwd", 1, 4 * N * (MAX_UNITS * 12 + QW + MAX_UNITS)):
            _lib.check(_lib.load().dc_target_unit_q_fwd(q.data_ptr(), QW, _ptr6(units), w_b.data_ptr(), b_b.data_ptr(),
                                                        logits.data_ptr(), N, _lib.stream_ptr()), "dc_target_unit_q_fwd")
        ctx.save_for_backward(att2, bm, w_b, b_b, *units)
        ctx.link = link
        ctx.att_shape = att.shape
        return logits.view(*lead, MAX_UNITS)

    @staticmethod
    def backward(ctx, dlogits):
        att2, bm, w_b, b_b = ctx.saved_tensors[:4]
        units = ctx.saved_tensors[4:]
        N = att2.shape[0]
        dl = _f32c(dlogits).reshape(N, MAX_UNITS)
        s = torch.empty((N, QW), dtype=torch.float32, device=att2.device)
        with PROFILE.span("target_unit_bwd", 1):       # bytes depend on how many tokens used the head (others are skipped)
            _lib.check(_lib.load().dc_target_unit_q_bwd(dl.data_ptr(), _ptr6(units), w_b.data_ptr(), b_b.data_ptr(), s.data_ptr(),
                                                        QW, N, _lib.stream_ptr()), "dc_target_unit_q_bwd")
        d_att = gemm_tf32x3(s, bm)                                          # [N, 128] = s [W_0 | ... | W_5 | b]^T
        ctx.link["pending"] = (dl, att2, s, att2, None)                      # consumed by UnitEncoder.backward
        return d_att.view(ctx.att_shape), None


def _head_matrix(link):
    """[128, 896]: bm[c, g*128+j] = W_g[c,j], bm[c, 768+g] = b_g[c], zeros in the rest of the bias block."""
    bias_block = torch.zeros((C, C), dtype=torch.float32, device=link["w_b"].device)
    bias_block[:, :6] = torch.stack(link["biases"], dim=1)
    return torch.cat(list(link["weights"]) + [bias_block], dim=1)


_rows_ws = {}


def target_rows(mask, action):
    """-> (rows int32 [N], count int32 [1], flags uint8 [N]), all on the device: the tokens, ascending, whose target-unit
    ``mask`` or ``action`` row (``[..., 40]`` bool) has an entry set -- the rows the PPO loss reads (``dc_target_rows``) --
    and a 0/1 flag per token.  Entries of ``rows`` past the count are unspecified."""
    _need_cuda(mask, action)
    m, a = _u8(mask).reshape(-1, MAX_UNITS), _u8(action).reshape(-1, MAX_UNITS)
    N = m.shape[0]
    dev = m.device
    ws = _rows_ws.get((N, dev))
    if ws is None:
        ws = _rows_ws[(N, dev)] = torch.empty(int(_lib.load().dc_target_rows_workspace_bytes(N)), dtype=torch.uint8, device=dev)
    rows = torch.empty(N, dtype=torch.int32, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    flags = torch.empty(N, dtype=torch.uint8, device=dev)
    with PROFILE.span("target_rows", 2, 2 * N * MAX_UNITS + 2 * N + 4 * N):
        _lib.check(_lib.load().dc_target_rows(m.data_ptr(), a.data_ptr(), N, rows.data_ptr(), count.data_ptr(), flags.data_ptr(),
                                              ws.data_ptr(), _lib.stream_ptr()), "dc_target_rows")
    return rows, count, flags


def _gemm_rows(a, b, rows, count, n_host, bias=None, gather=False, out=None, out_rows=None):
    """Rows i < count of ``a' b^T (+ bias)``, a' row i = ``a[rows[i]]`` when ``gather`` else ``a[i]``, into ``out[i]`` and / or
    ``out_rows[rows[i]]`` (``dc_gemm_tf32x3_rows``).  ``n_host``: the count when known, for the profile's bytes only."""
    M = rows.numel()
    K, N = a.shape[1], b.shape[0]
    ld = (out if out is not None else out_rows).stride(0)
    n = M if n_host is None else n_host
    with PROFILE.span("gemm_tf32x3", 1, 4 * (n * K + N * K + n * N * ((out is not None) + (out_rows is not None)))):
        _lib.check(_lib.load().dc_gemm_tf32x3_rows(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), _lib.ptr(bias), _lib.ptr(out),
                                                   _lib.ptr(out_rows), ld, M, count.data_ptr(), rows.data_ptr(), 1 if gather else 0,
                                                   N, K, 0, _lib.stream_ptr()), "dc_gemm_tf32x3_rows")


def _zero_inactive(flags, dst, n_host):
    """Zero rows of ``dst`` at the tokens whose flag is 0 (``dc_rows_zero_inactive``)."""
    N, width = dst.shape
    n = 0 if n_host is None else N - n_host
    with PROFILE.span("rows_zero", 1, N + 4 * n * width):
        _lib.check(_lib.load().dc_rows_zero_inactive(flags.data_ptr(), N, dst.data_ptr(), dst.stride(0), width, _lib.stream_ptr()),
                   "dc_rows_zero_inactive")


class TargetUnitRows(torch.autograd.Function):
    """The attention layer and the target-unit head (``TargetUnit``) on the active tokens only: ``rows[:count]`` and the
    per-token ``flags`` from ``target_rows``, all on the device, so that the training step stays one graph whatever the count.
    Logits of the active rows are those of ``affine_unit_attention`` + ``TargetUnit`` bit for bit; the other rows are zero,
    which the loss never reads.  No row is copied: the GEMMs read y through the row list and write their dense outputs at
    rows[i] themselves; dense outputs get their inactive rows zeroed, which writes nothing when every token is active.
      forward:  att_c = y[rows] W_att^T + b_att (compact, and dense ``att`` for ``UnitEncoder.backward``), q_c = att_c bm,
                logits[rows] from q_c;
      backward: s_c, d_att_c = s_c bm^T, dy[rows] = d_att_c W_att, dW_att = d_att_c^T y[rows], and (dl, att, s_c, att_c) for
                the encoder's backward (the head's share of dW_g = att_c^T s_c)."""

    @staticmethod
    def forward(ctx, y, w_att, b_att, link, rows, count, flags):
        _need_cuda(y, rows, count)
        units, w_b, b_b = link["units"], link["w_b"], link["b_b"]
        H = y.shape[-1]
        lead = y.shape[:-1]
        N = y.numel() // H
        dev = y.device
        n_act = int(count.item()) if PROFILE.enabled else None     # exact bytes for the profile only: a host sync
        link["n_active"] = n_act
        y2 = _f32c(y.detach()).reshape(N, H)
        w_att, b_att = _f32c(w_att.detach()), _f32c(b_att.detach())
        att_c = torch.empty((N, C), dtype=torch.float32, device=dev)
        att = torch.empty((N, C), dtype=torch.float32, device=dev)
        _gemm_rows(y2, w_att, rows, count, n_act, bias=b_att, gather=True, out=att_c, out_rows=att)
        _zero_inactive(flags, att, n_act)
        bm = _head_matrix(link)
        q_c = torch.empty((N, QW), dtype=torch.float32, device=dev)
        _gemm_rows(att_c, bm.t().contiguous(), rows, count, n_act, out=q_c)
        logits = torch.empty((N, MAX_UNITS), dtype=torch.float32, device=dev)
        _zero_inactive(flags, logits, n_act)
        nb = N if n_act is None else n_act
        with PROFILE.span("target_unit_fwd", 1, 4 * nb * (MAX_UNITS * 12 + QW + MAX_UNITS)):
            _lib.check(_lib.load().dc_target_unit_q_fwd_rows(q_c.data_ptr(), QW, _ptr6(units), w_b.data_ptr(), b_b.data_ptr(),
                                                             logits.data_ptr(), N, rows.data_ptr(), count.data_ptr(),
                                                             _lib.stream_ptr()), "dc_target_unit_q_fwd_rows")
        ctx.save_for_backward(y2, att_c, att, w_att, bm, w_b, b_b, rows, count, flags, *units)
        ctx.link = link
        ctx.n_act = n_act
        ctx.y_shape = y.shape
        return logits.view(*lead, MAX_UNITS)

    @staticmethod
    def backward(ctx, dlogits):
        y2, att_c, att, w_att, bm, w_b, b_b, rows, count, flags = ctx.saved_tensors[:10]
        units = ctx.saved_tensors[10:]
        N, H = y2.shape
        n_act = ctx.n_act
        nb = N if n_act is None else n_act
        dev = y2.device
        dl = _f32c(dlogits).reshape(N, MAX_UNITS)
        s_c = torch.empty((N, QW), dtype=torch.float32, device=dev)
        with PROFILE.span("target_unit_bwd", 1, 4 * nb * (MAX_UNITS * 12 + MAX_UNITS + QW)):
            _lib.check(_lib.load().dc_target_unit_q_bwd_rows(dl.data_ptr(), _ptr6(units), w_b.data_ptr(), b_b.data_ptr(),
                                                             s_c.data_ptr(), QW, N, rows.data_ptr(), count.data_ptr(),
                                                             _lib.stream_ptr()), "dc_target_unit_q_bwd_rows")
        d_att_c = torch.empty((N, C), dtype=torch.float32, device=dev)
        _gemm_rows(s_c, bm, rows, count, n_act, out=d_att_c)                       # [N, 128] = s_c bm^T, rows < count
        dy = dw = db = None
        if ctx.needs_input_grad[0]:
            dy = torch.empty((N, H), dtype=torch.float32, device=dev)
            _gemm_rows(d_att_c, w_att.t().contiguous(), rows, count, n_act, out_rows=dy)
            _zero_inactive(flags, dy, n_act)
            dy = dy.view(ctx.y_shape)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dw, db = gemm_wgrad_tf32x3(d_att_c, y2, want_bias=True, t_dev=count, t_host=n_act, x_rows=rows)
        ctx.link["pending"] = (dl, att, s_c, att_c, count)                       # consumed by UnitEncoder.backward
        return dy, dw, db, None, None, None, None


def unit_encoder(env, w_e, b_e, w_b, b_b, units, weights, biases, wait=None):
    """-> (``link``: the handle ``target_unit`` needs, pre-rnn input ``[..., 896]``).  ``wait(tensor)``, when given, makes
    the current stream wait for an input still being uploaded: it is called for ``env`` and for each unit group right
    before their first kernel, so the upload of group g+1 overlaps the kernels of group g."""
    link = {}
    tensors = (env, w_e, b_e, w_b, b_b, *units, *weights, *biases)
    need_grad = torch.is_grad_enabled() and any(t.requires_grad for t in tensors)
    xcat = UnitEncoder.apply(link, wait, need_grad, *tensors)
    return link, xcat


def target_unit(att, link):
    return TargetUnit.apply(att, link)


def target_unit_rows(y, w_att, b_att, link, rows, count, flags):
    """Target-unit logits ``[..., 40]`` from the core output ``y`` through the attention layer, on the tokens
    ``rows[:count]`` of ``target_rows`` only (``TargetUnitRows``); zero rows elsewhere."""
    return TargetUnitRows.apply(y, w_att, b_att, link, rows, count, flags)


__all__ = ["unit_encoder", "target_unit", "target_unit_rows", "target_rows", "gemm_wgrad_supported"]
