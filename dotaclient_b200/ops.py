"""Torch-facing wrappers of the C-ABI kernels (device memory + stream plumbing only).

Every function here requires CUDA tensors and enqueues hand-written sm_90a kernels from
``libdotaclient_b200.so`` on torch's current stream.  No CPU path exists: CPU tensors raise.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib

CELL_ID = {"gru": 0, "lstm": 1}
HEAD_KEYS = ("enum", "x", "y", "target_unit", "ability")     # policy.py:46
HEAD_SIZES = (4, 9, 9, 40, 3)
GATES = {"gru": 3, "lstm": 4}


class _Profile:
    """Optional per-kernel CUDA-event timing on the launching stream + a count of OUR kernel launches.

    Used by bench.py (roofline) -- events are recorded around each C-ABI call on torch's current stream.
    """

    def __init__(self):
        self.reset(False)

    def reset(self, enabled=False):
        self.enabled = enabled
        self.pairs = []
        self.launches = 0
        self.bytes = {}            # name -> algorithmic HBM bytes of the timed calls (inputs read once + outputs written once)

    class _Span:
        def __init__(self, prof, name, n_launches, nbytes=0):
            self.prof, self.name, self.n, self.nbytes = prof, name, n_launches, nbytes

        def __enter__(self):
            if self.prof.enabled:
                self.e0 = torch.cuda.Event(enable_timing=True)
                self.e1 = torch.cuda.Event(enable_timing=True)
                self.e0.record()
            return self

        def __exit__(self, *exc):
            if self.prof.enabled:
                self.e1.record()
                self.prof.pairs.append((self.name, self.e0, self.e1))
                self.prof.launches += self.n
                self.prof.bytes[self.name] = self.prof.bytes.get(self.name, 0) + self.nbytes
            return False

    def span(self, name, n_launches, nbytes=0):
        return _Profile._Span(self, name, n_launches, nbytes)

    def totals(self):
        torch.cuda.synchronize()
        out = {}
        for name, e0, e1 in self.pairs:
            out[name] = out.get(name, 0.0) + e0.elapsed_time(e1)
        return out

    def summary(self, steps=None):
        """ms per kernel name, averaged per step when ``steps`` is given (else per call)."""
        tot = self.totals()
        if steps:
            return {k: v / steps for k, v in tot.items()}
        counts = {}
        for name, _, _ in self.pairs:
            counts[name] = counts.get(name, 0) + 1
        return {k: v / counts[k] for k, v in tot.items()}


PROFILE = _Profile()


def _need_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("dotaclient_b200 kernels need CUDA tensors (no CPU fallback); got %s" % t.device)


def _f32c(t):
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.to(torch.float32).contiguous()
    return t


def _u8(t):
    """bool/uint8 tensor -> contiguous byte view (0/1)."""
    t = t.contiguous()
    if t.dtype == torch.bool:
        return t.view(torch.uint8)
    if t.dtype != torch.uint8:
        t = (t != 0).view(torch.uint8)
    return t


# --------------------------------------------------------------------------------------------- GAE
def gae_scan(rewards, values, seg_off, gamma=0.98, lam=0.97, boot_value=None, boot_reward=None):
    """GAE advantages + rewards-to-go for many rollouts (``optimizer.py:53-64,397,417-421``).

    rewards [n_rows] or [n_rows, n_sub] fp32; values [n_rows]; seg_off int64 [n_seg+1] (device).
    """
    _need_cuda(rewards, values, seg_off)
    rewards, values = _f32c(rewards), _f32c(values)
    n_sub = 1 if rewards.dim() == 1 else rewards.shape[1]
    n_rows = values.numel()
    assert rewards.numel() == n_rows * n_sub
    seg_off = seg_off.to(torch.int64).contiguous()
    adv = torch.empty(n_rows, dtype=torch.float32, device=values.device)
    ret = torch.empty_like(adv)
    lib = _lib.load()
    with PROFILE.span("gae_scan", 1):
        _lib.check(lib.dc_gae_scan(rewards.data_ptr(), n_sub, values.data_ptr(), seg_off.data_ptr(),
                                   seg_off.numel() - 1, _lib.ptr(boot_value), _lib.ptr(boot_reward), float(gamma),
                                   float(lam), adv.data_ptr(), ret.data_ptr(), _lib.stream_ptr()), "dc_gae_scan")
    return adv, ret


def _heads_args(group, gammas, K):
    """The host group map (int32 [n_sub]) and discounts (float64 [K]) of the multi-head scans, as ctypes arrays."""
    group = np.ascontiguousarray(group, dtype=np.int32)
    gammas = np.ascontiguousarray(gammas, dtype=np.float64)
    if gammas.shape != (K,):
        raise ValueError("gammas must hold one discount per value head (%d), got %s" % (K, gammas.shape))
    return (ctypes.c_int32 * group.size)(*group.tolist()), (ctypes.c_double * K)(*gammas.tolist()), group.size


def _heads_boot(boot, n_seg, K):
    if boot is None:
        return None
    boot = _f32c(boot)
    if boot.numel() != n_seg * K:
        raise ValueError("bootstraps must be [n_seg=%d, K=%d], got %s" % (n_seg, K, tuple(boot.shape)))
    return boot


def gae_scan_heads(rewards, values, seg_off, group, gammas, lam, boot_value=None, boot_reward=None):
    """GAE with one value head per reward group (``dc_gae_scan_heads``): ``rewards`` [n_rows, n_sub] fp32, ``values``
    [n_rows, K], ``seg_off`` int64 [n_seg + 1] (device); ``group`` the host int32 [n_sub] group of every reward column,
    ``gammas`` the K discounts; ``boot_value`` / ``boot_reward`` [n_seg, K] or None (0).  Returns ``(adv [n_rows], ret
    [n_rows, K])``: the advantage summed over the heads, and every head's return."""
    _need_cuda(rewards, values, seg_off, boot_value, boot_reward)
    rewards, values = _f32c(rewards), _f32c(values)
    n_rows, K = values.shape
    g, gm, n_sub = _heads_args(group, gammas, K)
    if rewards.numel() != n_rows * n_sub:
        raise ValueError("rewards have %d elements for %d rows of %d sub-rewards" % (rewards.numel(), n_rows, n_sub))
    seg_off = seg_off.to(torch.int64).contiguous()
    n_seg = seg_off.numel() - 1
    boot_value, boot_reward = _heads_boot(boot_value, n_seg, K), _heads_boot(boot_reward, n_seg, K)
    adv = torch.empty(n_rows, dtype=torch.float32, device=values.device)
    ret = torch.empty((n_rows, K), dtype=torch.float32, device=values.device)
    with PROFILE.span("gae_scan_heads", 1):
        _lib.check(_lib.load().dc_gae_scan_heads(rewards.data_ptr(), n_sub, g, K, values.data_ptr(), seg_off.data_ptr(),
                                                 n_seg, _lib.ptr(boot_value), _lib.ptr(boot_reward), gm, float(lam),
                                                 adv.data_ptr(), ret.data_ptr(), _lib.stream_ptr()), "dc_gae_scan_heads")
    return adv, ret


def gae_scan_heads_indexed(rewards, values, tok, seg_off, adv, ret, group, gammas, lam, boot_value=None,
                           boot_reward=None):
    """``gae_scan_heads`` in ``gae_scan_indexed``'s token layout (``dc_gae_scan_heads_indexed``): ``values`` [..., K] may be
    a view whose rows of K lie at one stride (the packed head output's value columns); row r reads the K values of token
    ``tok[r]`` and writes ``adv`` [n_tokens] and ``ret`` [n_tokens, K] (contiguous fp32) there, in place; rows with
    ``tok[r] < 0`` read 0 and write nothing."""
    _need_cuda(rewards, values, tok, seg_off, adv, ret, boot_value, boot_reward)
    rewards = _f32c(rewards)
    K = values.shape[-1]
    rows = values.detach().reshape(-1, K)
    if rows.dtype != torch.float32 or rows.stride(1) != 1:
        raise ValueError("values must be fp32 rows of K contiguous elements")
    ld = rows.stride(0) if rows.shape[0] > 1 else K
    if tok.dtype != torch.int64 or tok.dim() != 1 or not tok.is_contiguous():
        raise ValueError("tok must be a contiguous 1-D int64 tensor")
    g, gm, n_sub = _heads_args(group, gammas, K)
    if rewards.numel() != tok.numel() * n_sub:
        raise ValueError("rewards have %d elements for %d rows of %d sub-rewards" % (rewards.numel(), tok.numel(), n_sub))
    n_tok = rows.shape[0]
    for o, n in ((adv, n_tok), (ret, n_tok * K)):
        if o.dtype != torch.float32 or not o.is_contiguous() or o.numel() != n:
            raise ValueError("adv / ret must be contiguous fp32 tensors of %d / %d elements" % (n_tok, n_tok * K))
    seg_off = seg_off.to(torch.int64).contiguous()
    n_seg = seg_off.numel() - 1
    boot_value, boot_reward = _heads_boot(boot_value, n_seg, K), _heads_boot(boot_reward, n_seg, K)
    with PROFILE.span("gae_scan_heads_indexed", 1):
        _lib.check(_lib.load().dc_gae_scan_heads_indexed(
            rewards.data_ptr(), n_sub, g, K, rows.data_ptr(), ld, tok.data_ptr(), seg_off.data_ptr(), n_seg,
            _lib.ptr(boot_value), _lib.ptr(boot_reward), gm, float(lam), adv.data_ptr(), ret.data_ptr(),
            _lib.stream_ptr()), "dc_gae_scan_heads_indexed")
    return adv, ret


def vtrace_scan(rewards, values, logp_target, logp_behaviour, seg_off, gamma, lam, rho_clip, c_clip, boot_value=None,
                valid_len=None, stats=False):
    """V-trace value targets and policy-gradient advantages for many rollouts (``dc_vtrace_scan``).

    rewards [n_rows] or [n_rows, n_sub] fp32; values [n_rows]; logp_target / logp_behaviour [n_rows, 5] (0 where a head
    took no action); seg_off int64 [n_seg+1]; boot_value [n_seg] fp32 or None (0); valid_len int64 [n_seg] or None: the
    real steps of each segment, the only rows the statistics cover.  Returns ``(pg_adv, vs)``, and with ``stats`` also the
    per-segment sums ``[n_seg, _lib.VTRACE_STATS_SLOTS]`` fp64 (token count, sum log rho, sum clipped rho, rows with
    rho > rho_clip, rows with rho > c_clip).
    """
    _need_cuda(rewards, values, logp_target, logp_behaviour, seg_off, boot_value, valid_len)
    rewards, values = _f32c(rewards), _f32c(values)
    logp_target, logp_behaviour = _f32c(logp_target), _f32c(logp_behaviour)
    n_sub = 1 if rewards.dim() == 1 else rewards.shape[1]
    n_rows = values.numel()
    assert rewards.numel() == n_rows * n_sub
    assert logp_target.numel() == n_rows * 5 and logp_behaviour.numel() == n_rows * 5
    seg_off = seg_off.to(torch.int64).contiguous()
    n_seg = seg_off.numel() - 1
    if boot_value is not None:
        boot_value = _f32c(boot_value)
        assert boot_value.numel() == n_seg
    if valid_len is not None:
        valid_len = valid_len.to(torch.int64).contiguous()
        assert valid_len.numel() == n_seg
    pg_adv = torch.empty(n_rows, dtype=torch.float32, device=values.device)
    vs = torch.empty_like(pg_adv)
    seg_stats = torch.empty((n_seg, _lib.VTRACE_STATS_SLOTS), dtype=torch.float64, device=values.device) if stats else None
    lib = _lib.load()
    with PROFILE.span("vtrace_scan", 1):
        _lib.check(lib.dc_vtrace_scan(rewards.data_ptr(), n_sub, values.data_ptr(), logp_target.data_ptr(),
                                      logp_behaviour.data_ptr(), seg_off.data_ptr(), n_seg, _lib.ptr(valid_len),
                                      _lib.ptr(boot_value), float(gamma), float(lam), float(rho_clip), float(c_clip),
                                      pg_adv.data_ptr(), vs.data_ptr(), _lib.ptr(seg_stats), _lib.stream_ptr()),
                   "dc_vtrace_scan")
    return (pg_adv, vs, seg_stats) if stats else (pg_adv, vs)


def _indexed_args(rewards, values, tok, seg_off, out_a, out_b, boot_value):
    """Checks and normalises the operands of the indexed scans: ``values`` (any shape) as a flat strided view and its
    stride, the rollout-major ``rewards`` [n_rows(, n_sub)], ``tok`` [n_rows] int64, and the two contiguous fp32 outputs
    of the token layout, written in place."""
    _need_cuda(rewards, values, tok, seg_off, out_a, out_b, boot_value)
    rewards = _f32c(rewards)
    flat = values.detach().reshape(-1)
    if flat.dtype != torch.float32:
        raise ValueError("values must be fp32, got %s" % flat.dtype)
    ld = flat.stride(0) if flat.numel() > 1 else 1
    if tok.dtype != torch.int64 or tok.dim() != 1 or not tok.is_contiguous():
        raise ValueError("tok must be a contiguous 1-D int64 tensor")
    n_rows = tok.numel()
    n_sub = 1 if rewards.dim() == 1 else rewards.shape[1]
    if rewards.numel() != n_rows * n_sub:
        raise ValueError("rewards have %d elements for %d rows of %d sub-rewards" % (rewards.numel(), n_rows, n_sub))
    for o in (out_a, out_b):
        if o.dtype != torch.float32 or not o.is_contiguous() or o.numel() != flat.numel():
            raise ValueError("the outputs must be contiguous fp32 tensors of one element per value")
    seg_off = seg_off.to(torch.int64).contiguous()
    if boot_value is not None:
        boot_value = _f32c(boot_value)
        assert boot_value.numel() == seg_off.numel() - 1
    return rewards, n_sub, flat, ld, seg_off, boot_value


def gae_scan_indexed(rewards, values, tok, seg_off, adv, ret, gamma, lam, boot_value=None, boot_reward=None):
    """``gae_scan`` over rollout-major rows whose values and outputs live in a token layout of their own
    (``dc_gae_scan_indexed``): row r reads ``values.reshape(-1)[tok[r]]`` -- ``values`` may be a strided view whose
    elements lie at one stride, such as the value column of the packed head output -- and writes ``adv`` / ``ret``
    (contiguous fp32, one element per value) at ``tok[r]``, in place; rows with ``tok[r] < 0`` read a value of 0 and write
    nothing.  ``rewards`` [n_rows(, n_sub)], ``seg_off``, ``boot_value`` and ``boot_reward`` are as ``gae_scan``'s.
    ``tok`` (int64 [n_rows], device) must index ``values`` and name no token twice: the kernel cannot check it."""
    rewards, n_sub, flat, ld, seg_off, boot_value = _indexed_args(rewards, values, tok, seg_off, adv, ret, boot_value)
    if boot_reward is not None:
        boot_reward = _f32c(boot_reward)
    with PROFILE.span("gae_scan_indexed", 1):
        _lib.check(_lib.load().dc_gae_scan_indexed(rewards.data_ptr(), n_sub, flat.data_ptr(), ld, tok.data_ptr(),
                                                   seg_off.data_ptr(), seg_off.numel() - 1, _lib.ptr(boot_value),
                                                   _lib.ptr(boot_reward), float(gamma), float(lam), adv.data_ptr(),
                                                   ret.data_ptr(), _lib.stream_ptr()), "dc_gae_scan_indexed")
    return adv, ret


def vtrace_scan_indexed(rewards, values, logp_target, logp_behaviour, tok, seg_off, pg_adv, vs, gamma, lam, rho_clip,
                        c_clip, boot_value=None, valid_len=None):
    """``vtrace_scan`` with ``gae_scan_indexed``'s token layout (``dc_vtrace_scan_indexed``): row r reads its value and its
    target log-probs ``logp_target`` [n_tokens, 5] at token ``tok[r]`` and writes ``pg_adv`` / ``vs`` there, in place;
    ``logp_behaviour`` [n_rows, 5], ``valid_len`` and the rest stay rollout-major.  The per-segment statistics are not
    computed."""
    rewards, n_sub, flat, ld, seg_off, boot_value = _indexed_args(rewards, values, tok, seg_off, pg_adv, vs, boot_value)
    _need_cuda(logp_target, logp_behaviour, valid_len)
    logp_target, logp_behaviour = _f32c(logp_target), _f32c(logp_behaviour)
    if logp_target.numel() != flat.numel() * 5 or logp_behaviour.numel() != tok.numel() * 5:
        raise ValueError("logp_target must be [n_tokens, 5] and logp_behaviour [n_rows, 5]")
    if valid_len is not None:
        valid_len = valid_len.to(torch.int64).contiguous()
    with PROFILE.span("vtrace_scan_indexed", 1):
        _lib.check(_lib.load().dc_vtrace_scan_indexed(
            rewards.data_ptr(), n_sub, flat.data_ptr(), ld, logp_target.data_ptr(), logp_behaviour.data_ptr(),
            tok.data_ptr(), seg_off.data_ptr(), seg_off.numel() - 1, _lib.ptr(valid_len), _lib.ptr(boot_value),
            float(gamma), float(lam), float(rho_clip), float(c_clip), pg_adv.data_ptr(), vs.data_ptr(), None,
            _lib.stream_ptr()), "dc_vtrace_scan_indexed")
    return pg_adv, vs


def _upgo_logp(logp_target, logp_behaviour, n_target, n_rows):
    """The log-prob operands of the UPGO scans: both None (GAE) or both given (V-trace), as fp32 [n, 5]."""
    if (logp_target is None) != (logp_behaviour is None):
        raise ValueError("give both logp_target and logp_behaviour (V-trace) or neither (GAE)")
    if logp_target is None:
        return None, None
    logp_target, logp_behaviour = _f32c(logp_target), _f32c(logp_behaviour)
    if logp_target.numel() != n_target * 5 or logp_behaviour.numel() != n_rows * 5:
        raise ValueError("logp_target must be [%d, 5] and logp_behaviour [%d, 5]" % (n_target, n_rows))
    return logp_target, logp_behaviour


def upgo_scan(rewards, values, seg_off, adv, gamma, coef, boot_value=None, logp_target=None, logp_behaviour=None,
              rho_clip=1.0, valid_len=None, stats=False):
    """Adds ``coef`` times the UPGO advantage A^U into ``adv`` in place (``dc_upgo_scan``; DESIGN.md section 4.2):
    G_t = r_t + gamma G_{t+1} while the next step's TD error is >= 0, r_t + gamma V_{t+1} after a worse one, and
    A^U_t = rhob_t (G_t - V_t).  ``rewards``, ``values``, ``seg_off``, ``boot_value`` and ``valid_len`` are as
    ``vtrace_scan``'s; ``adv`` [n_rows] contiguous fp32, the advantages the base scan wrote.  Without log-probs rhob = 1
    (GAE); with ``logp_target`` / ``logp_behaviour`` [n_rows, 5] it is V-trace's min(rho_clip, rho).  Returns ``adv``, and
    with ``stats`` also the per-segment sums ``[n_seg, _lib.UPGO_STATS_SLOTS]`` fp64 (row count, rows that went through
    to the next step's return, sum of A^U) over the real steps."""
    _need_cuda(rewards, values, seg_off, adv, boot_value, valid_len, logp_target, logp_behaviour)
    rewards, values = _f32c(rewards), _f32c(values)
    n_sub = 1 if rewards.dim() == 1 else rewards.shape[1]
    n_rows = values.numel()
    if rewards.numel() != n_rows * n_sub:
        raise ValueError("rewards have %d elements for %d rows of %d sub-rewards" % (rewards.numel(), n_rows, n_sub))
    if adv.dtype != torch.float32 or not adv.is_contiguous() or adv.numel() != n_rows:
        raise ValueError("adv must be a contiguous fp32 tensor of %d elements" % n_rows)
    logp_target, logp_behaviour = _upgo_logp(logp_target, logp_behaviour, n_rows, n_rows)
    seg_off = seg_off.to(torch.int64).contiguous()
    n_seg = seg_off.numel() - 1
    if boot_value is not None:
        boot_value = _f32c(boot_value)
        assert boot_value.numel() == n_seg
    if valid_len is not None:
        valid_len = valid_len.to(torch.int64).contiguous()
        assert valid_len.numel() == n_seg
    seg_stats = torch.empty((n_seg, _lib.UPGO_STATS_SLOTS), dtype=torch.float64, device=values.device) if stats else None
    with PROFILE.span("upgo_scan", 1):
        _lib.check(_lib.load().dc_upgo_scan(rewards.data_ptr(), n_sub, values.data_ptr(), _lib.ptr(logp_target),
                                            _lib.ptr(logp_behaviour), seg_off.data_ptr(), n_seg, _lib.ptr(valid_len),
                                            _lib.ptr(boot_value), float(gamma), float(rho_clip), float(coef),
                                            adv.data_ptr(), _lib.ptr(seg_stats), _lib.stream_ptr()), "dc_upgo_scan")
    return (adv, seg_stats) if stats else adv


def upgo_scan_indexed(rewards, values, tok, seg_off, adv, gamma, coef, boot_value=None, logp_target=None,
                      logp_behaviour=None, rho_clip=1.0):
    """``upgo_scan`` with ``vtrace_scan_indexed``'s token layout (``dc_upgo_scan_indexed``): row r reads its value (and
    target log-probs ``logp_target`` [n_tokens, 5]) at token ``tok[r]`` and adds into ``adv`` there, in place; rows with
    ``tok[r] < 0`` read 0 and write nothing.  ``logp_behaviour`` [n_rows, 5] stays rollout-major.  The per-segment
    statistics are not computed."""
    rewards, n_sub, flat, ld, seg_off, boot_value = _indexed_args(rewards, values, tok, seg_off, adv, adv, boot_value)
    _need_cuda(logp_target, logp_behaviour)
    logp_target, logp_behaviour = _upgo_logp(logp_target, logp_behaviour, flat.numel(), tok.numel())
    with PROFILE.span("upgo_scan_indexed", 1):
        _lib.check(_lib.load().dc_upgo_scan_indexed(
            rewards.data_ptr(), n_sub, flat.data_ptr(), ld, _lib.ptr(logp_target), _lib.ptr(logp_behaviour),
            tok.data_ptr(), seg_off.data_ptr(), seg_off.numel() - 1, None, _lib.ptr(boot_value), float(gamma),
            float(rho_clip), float(coef), adv.data_ptr(), None, _lib.stream_ptr()), "dc_upgo_scan_indexed")
    return adv


# --------------------------------------------------------------------------------------------- minibatch gather
_index_staging = {}     # device -> (pinned int64 buffer, event recorded after the last upload from it)


def _upload_index(idx, device):
    """Asynchronous upload of a host index through a cached pinned buffer: a copy from pageable memory may wait for the
    stream, which would stall the host behind the GPU at every minibatch."""
    buf, ev = _index_staging.get(device, (None, None))
    if ev is not None:
        ev.synchronize()                     # the previous upload has left the buffer
    if buf is None or buf.numel() < idx.size:
        buf = torch.empty(max(idx.size, 4096), dtype=torch.int64).pin_memory()
    buf.numpy()[:idx.size] = idx
    out = buf[:idx.size].to(device, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    _index_staging[device] = (buf, ev)
    return out


def gather_columns(pairs, index):
    """``dst.copy_(src.index_select(1, index))`` for every ``(src, dst)`` pair, in one ``dc_gather_columns`` launch per
    ``_lib.GATHER_MAX_TENSORS`` pairs.

    Every ``src`` is a contiguous CUDA tensor of at least 2 dims; its ``dst`` is contiguous, on the same device, of the same
    dtype, and of shape ``(src.shape[0], len(index)) + src.shape[2:]``.  ``index`` is a 1-D integer array or tensor on the
    HOST (a CUDA tensor is read back first): it is checked there -- every value in ``[0, src.shape[1])`` -- and uploaded,
    because the kernel cannot check a device index.  Raises ``ValueError`` before any launch.
    """
    if isinstance(index, torch.Tensor):
        index = index.cpu().numpy()
    idx = np.asarray(index)
    if idx.ndim != 1 or idx.dtype.kind not in "iu":
        raise ValueError("gather_columns: index must be a 1-D integer array, got %s %s" % (idx.dtype, idx.shape))
    lo, hi = (int(idx.min()), int(idx.max())) if idx.size else (0, -1)
    descs, device = [], None
    for src, dst in pairs:
        if src.dim() < 2 or not src.is_contiguous() or not dst.is_contiguous():
            raise ValueError("gather_columns: tensors must be contiguous with at least 2 dims, got %s" % (tuple(src.shape),))
        shape = src.shape
        if lo < 0 or hi >= shape[1]:
            raise ValueError("gather_columns: index values %d..%d outside [0, %d)" % (lo, hi, shape[1]))
        _need_cuda(src, dst)
        if dst.shape != (shape[0], idx.size) + shape[2:] or dst.dtype != src.dtype or dst.device != src.device:
            raise ValueError("gather_columns: dst %s %s does not match src %s %s gathered at %d columns"
                             % (dst.dtype, tuple(dst.shape), src.dtype, tuple(shape), idx.size))
        if device is not None and src.device != device:
            raise ValueError("gather_columns: all tensors must be on one device")
        device = src.device
        row_bytes = math.prod(shape[2:]) * src.element_size()
        if row_bytes and shape[0]:               # an empty tensor has nothing to copy
            descs.append(_lib.GatherDesc(src.data_ptr(), dst.data_ptr(), shape[0], shape[1], row_bytes))
    if not descs or idx.size == 0:
        return
    index_dev = _upload_index(idx, device)
    lib = _lib.load()
    n_max = _lib.GATHER_MAX_TENSORS
    for k in range(0, len(descs), n_max):
        chunk = descs[k:k + n_max]
        with PROFILE.span("gather_columns", 1):
            _lib.check(lib.dc_gather_columns((_lib.GatherDesc * len(chunk))(*chunk), len(chunk), index_dev.data_ptr(),
                                             idx.size, _lib.stream_ptr()), "dc_gather_columns")


def gather_columns_fill(pairs, index):
    """``gather_columns`` with a DEVICE index in which -1 writes zeros (``dc_gather_columns_fill``): column j of every
    ``dst`` is column ``index[j]`` of its ``src``, or zeros where ``index[j] < 0``.  ``src`` / ``dst`` are as
    ``gather_columns``'; ``index`` is a contiguous 1-D int64 CUDA tensor.  The caller guarantees ``-1 <= index <
    src.shape[1]``: the kernel cannot check a device index, so it is built and checked on the host where it is made
    (``state_refresh_layout``).  Raises ``ValueError`` for malformed operands before any launch."""
    if not isinstance(index, torch.Tensor) or index.dtype != torch.int64 or index.dim() != 1 \
            or not index.is_contiguous():
        raise ValueError("gather_columns_fill: index must be a contiguous 1-D int64 tensor")
    _need_cuda(index)
    n = index.numel()
    descs = []
    for src, dst in pairs:
        if src.dim() < 2 or not src.is_contiguous() or not dst.is_contiguous():
            raise ValueError("gather_columns_fill: tensors must be contiguous with at least 2 dims, got %s"
                             % (tuple(src.shape),))
        _need_cuda(src, dst)
        shape = src.shape
        if dst.shape != (shape[0], n) + shape[2:] or dst.dtype != src.dtype or dst.device != index.device \
                or src.device != index.device:
            raise ValueError("gather_columns_fill: dst %s %s does not match src %s %s gathered at %d columns"
                             % (dst.dtype, tuple(dst.shape), src.dtype, tuple(shape), n))
        row_bytes = math.prod(shape[2:]) * src.element_size()
        if row_bytes and shape[0]:
            descs.append(_lib.GatherDesc(src.data_ptr(), dst.data_ptr(), shape[0], shape[1], row_bytes))
    if not descs or n == 0:
        return
    lib = _lib.load()
    n_max = _lib.GATHER_MAX_TENSORS
    for k in range(0, len(descs), n_max):
        chunk = descs[k:k + n_max]
        with PROFILE.span("gather_columns_fill", 1):
            _lib.check(lib.dc_gather_columns_fill((_lib.GatherDesc * len(chunk))(*chunk), len(chunk), index.data_ptr(), n,
                                                  _lib.stream_ptr()), "dc_gather_columns_fill")


def gather_rows_fill(srcs, index):
    """``src[index]`` (zeros where ``index < 0``) for every contiguous ``src`` ``[N, ...]`` with a device ``index`` (one
    ``dc_gather_columns_fill`` launch on ``[1, N, ...]`` views).  Returns the new ``[len(index), ...]`` tensors."""
    n = index.numel()
    outs = [torch.empty((n,) + tuple(s.shape[1:]), dtype=s.dtype, device=s.device) for s in srcs]
    gather_columns_fill([(s.view((1,) + tuple(s.shape)), o.view((1,) + tuple(o.shape))) for s, o in zip(srcs, outs)],
                        index)
    return outs


def refresh_states(ybufs, cbufs, t0, step, rollout, slot, h0, c0, reset_h, reset_c, acc):
    """Writes the recomputed recurrent states of one time block into a training batch, in place, and adds the drift sums
    to ``acc`` (``dc_refresh_states``): for every destination d, every layer l's state ``ybufs[l][step[d] - t0,
    rollout[d]]`` (``[T + 1, R, H]`` state buffers of ``rnn_stack_forward_states``; ``cbufs`` too for the LSTM) goes to
    ``h0[l, slot[d]]`` (``[L, B, H]``) for ``slot[d] < B``, else to the H-wide slice l of row ``slot[d] - B`` of the
    ``[K, B, L*H]`` reset tables; ``acc`` (float64 [2], device) += (sum (new - old)^2, sum old^2).  ``step``, ``rollout``
    and ``slot`` are int64 device tensors of one length that the caller built and checked on the host.  ``c0``,
    ``reset_c`` and ``cbufs``: None for the GRU; ``reset_h`` / ``reset_c`` None without resets."""
    n_layers = len(ybufs)
    lstm = c0 is not None
    _need_cuda(h0, c0, reset_h, reset_c, acc, step, rollout, slot, *ybufs)
    L, B, H = h0.shape
    T1, R = ybufs[0].shape[:2]
    if L != n_layers or not 1 <= n_layers <= _lib.REFRESH_MAX_LAYERS:
        raise ValueError("refresh_states: %d state buffers for h0 of %d layers (1 to %d)"
                         % (n_layers, L, _lib.REFRESH_MAX_LAYERS))
    if acc.dtype != torch.float64 or acc.numel() != 2:
        raise ValueError("refresh_states: acc must be float64 [2]")
    bufs = list(ybufs) + (list(cbufs) if lstm else [])
    if lstm and len(cbufs) != n_layers:
        raise ValueError("refresh_states: the LSTM needs one c buffer per layer")
    for b in bufs:
        if b.dtype != torch.float32 or b.shape != (T1, R, H) or not b.is_contiguous():
            raise ValueError("refresh_states: state buffers must be contiguous fp32 [%d, %d, %d]" % (T1, R, H))
    tabs = [h0] + ([c0] if lstm else [])
    K = 0
    if reset_h is not None:
        K = reset_h.shape[0]
        tabs += [reset_h] + ([reset_c] if lstm else [])
        for t in tabs[2 if lstm else 1:]:
            if t.shape != (K, B, L * H):
                raise ValueError("refresh_states: reset tables must be [K, %d, %d]" % (B, L * H))
    if lstm and (c0.shape != h0.shape):
        raise ValueError("refresh_states: c0 must match h0")
    for t in tabs:
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("refresh_states: the batch's states must be contiguous fp32")
    n = step.numel()
    for t in (step, rollout, slot):
        if t.dtype != torch.int64 or t.dim() != 1 or t.numel() != n or not t.is_contiguous():
            raise ValueError("refresh_states: step, rollout and slot must be contiguous int64 [n]")
    partial = torch.empty((max(n, 1) * n_layers, 2), dtype=torch.float64, device=h0.device)
    ptrs = ctypes.c_void_p * n_layers
    hp = ptrs(*[b.data_ptr() for b in ybufs])
    cp = ptrs(*[b.data_ptr() for b in cbufs]) if lstm else None
    with PROFILE.span("refresh_states", 2, 12 * n * n_layers * H * (2 if lstm else 1)):
        _lib.check(_lib.load().dc_refresh_states(n_layers, H, hp, cp, R, int(t0), step.data_ptr(), rollout.data_ptr(),
                                                 slot.data_ptr(), n, B, K, h0.data_ptr(), _lib.ptr(c0), _lib.ptr(reset_h),
                                                 _lib.ptr(reset_c), partial.data_ptr(), acc.data_ptr(),
                                                 _lib.stream_ptr()), "dc_refresh_states")


# --------------------------------------------------------------------------------------------- RNN
_workspaces = {}


def _rnn_workspace(cell, B, H, device):
    key = (cell, H, device)
    nbytes = max(int(_lib.load().dc_rnn_workspace_bytes(CELL_ID[cell], B, H)), 16)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def _check_reset(reset, S, B, H, cell, device):
    """``reset`` of ``rnn_sequence`` -> ``(slot [S, B] int32, h_tab [K, B, H], prev_tab [K, B, H])`` (prev: h for the GRU, c
    for the LSTM), all contiguous; None when there is nothing to reset (None, or K = 0)."""
    if reset is None:
        return None
    slot, h_tab, c_tab = reset
    _need_cuda(slot, h_tab, c_tab)
    K = h_tab.shape[0]
    if slot.shape != (S, B) or slot.dtype != torch.int32:
        raise ValueError("reset slot must be int32 [%d, %d], got %s %s" % (S, B, slot.dtype, tuple(slot.shape)))
    if h_tab.shape != (K, B, H) or (cell == "lstm") != (c_tab is not None) or (c_tab is not None and c_tab.shape != (K, B, H)):
        raise ValueError("reset states must be [K, %d, %d] (h, and c for the LSTM only), got %s / %s"
                         % (B, H, tuple(h_tab.shape), None if c_tab is None else tuple(c_tab.shape)))
    if K == 0:
        return None
    h_tab = _f32c(h_tab.detach())
    return slot.contiguous(), h_tab, (h_tab if c_tab is None else _f32c(c_tab.detach()))


def _rnn_forward_impl(x, w_ih, w_hh, b_ih, b_hh, h0, c0, cell, reset=None):
    """i2h GEMM (wgmma 3xTF32, ``dc_gemm_tf32x3``) + recurrence kernel.  Returns (x2, w_ih, w_hh, gates, ybuf, cbuf).
    ``reset``: the checked operands of ``_check_reset`` or None; the reset rows' h2h pre-activations are computed here, one
    GEMM of K*B rows, and the recurrence runs through ``dc_rnn_seq_fwd_reset``."""
    _need_cuda(x, w_ih, w_hh, b_ih, b_hh, h0, c0)
    S, B, Hin = x.shape
    H = w_hh.shape[1]
    N = S * B
    x2 = _f32c(x.detach()).view(N, Hin)
    w_ih, w_hh, b_ih, b_hh = _f32c(w_ih.detach()), _f32c(w_hh.detach()), _f32c(b_ih.detach()), _f32c(b_hh.detach())
    # [N, G*H] = x W_ih^T + b_ih on wgmma (3xTF32); shapes outside the kernel's (G*H % 32, Hin % 32) raise DC_EUNSUPPORTED
    gates = gemm_tf32x3(x2, w_ih, b_ih)
    ybuf = torch.empty((S + 1, B, H), dtype=torch.float32, device=x.device)
    cbuf = torch.empty((S + 1, B, H), dtype=torch.float32, device=x.device)
    ybuf[0].copy_(h0.detach().reshape(B, H))
    if cell == "lstm":
        cbuf[0].copy_(c0.detach().reshape(B, H))
    ws = _rnn_workspace(cell, B, H, x.device)
    lib = _lib.load()
    if reset is not None:
        slot, h_tab, prev_tab = reset
        K = h_tab.shape[0]
        pre = gemm_tf32x3(h_tab.view(K * B, H), w_hh, b_hh)                  # h_reset W_hh^T + b_hh [K*B, G*H]
        with PROFILE.span("rnn_fwd", 1, 4 * S * B * ((4 if cell == "lstm" else 3) + 1) * H):
            _lib.check(lib.dc_rnn_seq_fwd_reset(CELL_ID[cell], gates.data_ptr(), w_hh.data_ptr(), b_hh.data_ptr(),
                                                ybuf.data_ptr(), cbuf.data_ptr(), slot.data_ptr(), prev_tab.data_ptr(),
                                                pre.data_ptr(), K, B, S, H, ws.data_ptr(), _lib.stream_ptr()),
                       "dc_rnn_seq_fwd_reset")
        return x2, w_ih, w_hh, gates, ybuf, cbuf
    with PROFILE.span("rnn_fwd", 1, 4 * S * B * ((4 if cell == "lstm" else 3) + 1) * H):      # SURVEY.md 8(d)
        _lib.check(lib.dc_rnn_seq_fwd(CELL_ID[cell], gates.data_ptr(), w_hh.data_ptr(), b_hh.data_ptr(),
                                      ybuf.data_ptr(), cbuf.data_ptr(), B, S, H, ws.data_ptr(), _lib.stream_ptr()),
                   "dc_rnn_seq_fwd")
    return x2, w_ih, w_hh, gates, ybuf, cbuf


def rnn_forward_states(x_tm, w_ih, w_hh, b_ih, b_hh, h0, c0, cell):
    """No-grad forward returning the full state buffers: ybuf [S+1,B,H] (slot 0 = h0, slot t+1 = h_t) and
    cbuf [S+1,B,H] (LSTM cell states).  Used by experience prep to read the hidden state at chunk boundaries."""
    with torch.no_grad():
        _, _, _, _, ybuf, cbuf = _rnn_forward_impl(x_tm, w_ih, w_hh, b_ih, b_hh, h0, c0, cell)
    return ybuf, cbuf


def rnn_stack_forward_states(x_tm, layers, h0, c0, cell):
    """``rnn_forward_states`` through a stack of layers: ``layers`` = [(w_ih, w_hh, b_ih, b_hh)] per layer, h0 / c0
    ``[L, B, H]`` (c0 None for the GRU).  Layer k reads layer k-1's ``ybuf[1:]`` view.  Returns the per-layer lists of
    ybuf and cbuf ``[S+1, B, H]``: the hidden state entering step t of layer k is ``ybufs[k][t]``."""
    ybufs, cbufs, x = [], [], x_tm
    for k, (w_ih, w_hh, b_ih, b_hh) in enumerate(layers):
        ybuf, cbuf = rnn_forward_states(x, w_ih, w_hh, b_ih, b_hh, h0[k], None if c0 is None else c0[k], cell)
        ybufs.append(ybuf)
        cbufs.append(cbuf)
        x = ybuf[1:]
    return ybufs, cbufs


def stack_layers(states):
    """Per-layer ``[B, H]`` states -> torch's ``[L, B, H]`` (a view, no copy, for a single layer)."""
    return states[0].unsqueeze(0) if len(states) == 1 else torch.stack(states)


def _reset_rows(slot, K):
    """For every row ``k*B + b`` of a ``[K, B, ...]`` reset table: the token ``t*B + b`` whose ``slot[t, b]`` is k
    (int64 ``[K*B]``, 0 for unused rows) and whether the row is used (fp32 ``[K*B, 1]``, 1 / 0).  On the device, no sync."""
    S, B = slot.shape
    dev = slot.device
    s = slot.long()
    b = torch.arange(B, device=dev).expand(S, B)
    row = torch.where(s >= 0, s * B + b, K * B).reshape(-1)               # carried tokens all land on a spare row K*B
    tok = torch.arange(S * B, device=dev)
    idx = torch.zeros(K * B + 1, dtype=torch.int64, device=dev).scatter_(0, row, tok)
    used = torch.zeros(K * B + 1, dtype=torch.float32, device=dev).scatter_(0, row, torch.ones(S * B, device=dev))
    return idx[:K * B], used[:K * B].unsqueeze(1)


def _gather_rows(srcs, index):
    """``src[index]`` for every 2-D contiguous ``src`` with a DEVICE int64 ``index`` (one ``dc_gather_columns`` launch on
    ``[1, N, row]`` views).  The caller guarantees ``0 <= index < N``: the index is made on the device from checked data."""
    n = index.numel()
    outs = [torch.empty((n, src.shape[1]), dtype=src.dtype, device=src.device) for src in srcs]
    descs = [_lib.GatherDesc(src.data_ptr(), out.data_ptr(), 1, src.shape[0], src.shape[1] * src.element_size())
             for src, out in zip(srcs, outs)]
    with PROFILE.span("gather_columns", 1):
        _lib.check(_lib.load().dc_gather_columns((_lib.GatherDesc * len(descs))(*descs), len(descs), index.data_ptr(), n,
                                                 _lib.stream_ptr()), "dc_gather_columns")
    return outs


class RnnSequence(torch.autograd.Function):
    """Time-major GRU/LSTM layer: i2h GEMM (wgmma 3xTF32) + hand-written recurrence kernels.

    forward(x [S,B,Hin], w_ih [G*H,Hin], w_hh [G*H,H], b_ih, b_hh, h0 [B,H], c0 [B,H]|None, cell, reset=None)
      -> y [S,B,H], h_n [B,H], c_n [B,H] (zeros-size-0 tensor for GRU)
    Semantics of ``torch.nn.GRU/LSTM(batch_first=...)`` as used in ``policy.py:66,141``.
    ``reset``: None, or ``(slot [S, B] int32, h [K, B, H], c [K, B, H] | None)``: at a token with ``slot[t, b] = k >= 0``
    the state entering step t of sequence b is replaced by row (k, b) of the tables (``dc_rnn_seq_fwd_reset``).  The
    tables are data: they get no gradient, like ``h0`` of a training batch.
    """

    @staticmethod
    def forward(ctx, x, w_ih, w_hh, b_ih, b_hh, h0, c0, cell, reset=None):
        S, B, Hin = x.shape
        H = w_hh.shape[1]
        reset = _check_reset(reset, S, B, H, cell, x.device)
        x2, w_ih, w_hh, gates, ybuf, cbuf = _rnn_forward_impl(x, w_ih, w_hh, b_ih, b_hh, h0, c0, cell, reset)
        ctx.cell, ctx.dims = cell, (S, B, Hin, H, GATES[cell])
        ctx.reset = reset
        ctx.save_for_backward(x2, w_ih, w_hh, gates, ybuf, cbuf)
        y = ybuf[1:]
        h_n = ybuf[S].clone()
        if cell == "lstm":
            c_n = cbuf[S].clone()
        else:
            c_n = ybuf.new_empty(0)
            ctx.mark_non_differentiable(c_n)
        return y, h_n, c_n

    @staticmethod
    def backward(ctx, dy, dhn, dcn):
        x2, w_ih, w_hh, gates, ybuf, cbuf = ctx.saved_tensors
        cell = ctx.cell
        S, B, Hin, H, G = ctx.dims
        N = S * B
        if getattr(ctx, "_consumed", False):
            raise RuntimeError("RnnSequence backward ran twice: the saved gate buffer is consumed in place")
        ctx._consumed = True
        dy = _f32c(dy) if dy is not None else torch.zeros((S, B, H), dtype=torch.float32, device=x2.device)
        dhn = _f32c(dhn) if dhn is not None else None
        dcn = _f32c(dcn) if (dcn is not None and cell == "lstm" and dcn.numel()) else None
        dh0 = torch.empty((B, H), dtype=torch.float32, device=x2.device)
        dc0 = torch.empty((B, H), dtype=torch.float32, device=x2.device) if cell == "lstm" else None
        ws = _rnn_workspace(cell, B, H, x2.device)
        lib = _lib.load()
        reset = ctx.reset
        with PROFILE.span("rnn_bwd", 1, 8 * S * B * ((4 if cell == "lstm" else 3) + 1) * H):
            if reset is None:
                _lib.check(lib.dc_rnn_seq_bwd(CELL_ID[cell], gates.data_ptr(), w_hh.data_ptr(), ybuf.data_ptr(),
                                              cbuf.data_ptr(), dy.data_ptr(), _lib.ptr(dhn), _lib.ptr(dcn), dh0.data_ptr(),
                                              _lib.ptr(dc0), B, S, H, ws.data_ptr(), _lib.stream_ptr()), "dc_rnn_seq_bwd")
            else:
                slot, h_tab, prev_tab = reset
                _lib.check(lib.dc_rnn_seq_bwd_reset(CELL_ID[cell], gates.data_ptr(), w_hh.data_ptr(), ybuf.data_ptr(),
                                                    cbuf.data_ptr(), dy.data_ptr(), _lib.ptr(dhn), _lib.ptr(dcn),
                                                    dh0.data_ptr(), _lib.ptr(dc0), slot.data_ptr(), prev_tab.data_ptr(),
                                                    h_tab.shape[0], B, S, H, ws.data_ptr(), _lib.stream_ptr()),
                           "dc_rnn_seq_bwd_reset")
        dgi = gates                                   # [N, G*H], overwritten in place by the kernel
        hprev = ybuf[:S].view(N, H)                   # h_{t-1} for every token (slot t)
        dx = gemm_tf32x3(dgi, w_ih.t().contiguous()).view(S, B, Hin) if ctx.needs_input_grad[0] else None   # dx = dgi W_ih
        dw_ih, db_ih = gemm_wgrad_tf32x3(dgi, x2)                              # dW_ih = dgi^T x, db_ih = colsum(dgi)
        if cell == "lstm":
            dw_hh = gemm_wgrad_tf32x3(dgi, hprev, want_bias=False)[0]
            db_hh = db_ih
        else:
            dghn = cbuf[1:].view(N, H)                # n-gate part of dgh (= dgi_n * r)
            dw_hh = torch.empty_like(w_hh)
            gemm_wgrad_tf32x3(dgi[:, :2 * H], hprev, want_bias=False, dw_out=dw_hh[:2 * H])
            _, db_n = gemm_wgrad_tf32x3(dghn, hprev, dw_out=dw_hh[2 * H:])
            db_hh = torch.cat([db_ih[:2 * H], db_n])
        if reset is not None:
            # dW_hh above paired each token's dgh with ybuf[t]; a reset token's step used h_reset: add
            # dgh_t^T (h_reset - ybuf[t]) over the reset tokens (K*B gathered rows, unused ones weighted 0)
            slot, h_tab, _ = reset
            K = h_tab.shape[0]
            tok, used = _reset_rows(slot, K)
            srcs = [dgi, hprev] + ([] if cell == "lstm" else [cbuf[1:].view(N, H)])
            rows = _gather_rows(srcs, tok)
            diff = (h_tab.view(K * B, H) - rows[1]) * used
            if cell == "lstm":
                gemm_wgrad_tf32x3(rows[0], diff, want_bias=False, dw_out=dw_hh, accumulate=True)
            else:
                gemm_wgrad_tf32x3(rows[0][:, :2 * H], diff, want_bias=False, dw_out=dw_hh[:2 * H], accumulate=True)
                gemm_wgrad_tf32x3(rows[2], diff, want_bias=False, dw_out=dw_hh[2 * H:], accumulate=True)
        return dx, dw_ih, dw_hh, db_ih, db_hh, dh0, dc0, None, None


def rnn_sequence(x_tm, w_ih, w_hh, b_ih, b_hh, h0, c0, cell, reset=None):
    """One recurrent layer (``RnnSequence``); ``reset`` = ``(slot [S, B] int32, h [K, B, H], c [K, B, H] | None)`` restarts
    the state inside sequences (see ``RnnSequence``), None is the plain recurrence."""
    return RnnSequence.apply(x_tm, w_ih, w_hh, b_ih, b_hh, h0, c0, cell, reset)


# --------------------------------------------------------------------------------------------- PPO loss
def hparam_block(device, lr=0.0, e_clip=0.0, entropy_coef=0.0, vf_coef=0.0, max_grad_norm=0.0, value_clip=None,
                 value_norm=None, kl_coef=0.0, kl_stop=None):
    """A device hyper-parameter block (``_lib.HPARAM_SLOTS`` fp64) holding the given values, for the ``hparams=``
    argument of ``ppo_loss_fwd_bwd`` / ``ppo_loss_packed`` / ``grad_finish``.  ``value_norm=(mu, sigma)`` makes the loss
    normalise the raw value targets as ``(r - mu) / sigma`` (sigma > 0); None leaves slots 6 and 7 at 0 (off).
    ``kl_coef`` is the KL penalty's beta and ``kl_stop`` the KL limit of the finish (None: no limit); only the KL entry
    points read them."""
    vals = [0.0] * _lib.HPARAM_SLOTS
    vals[_lib.HP_LR], vals[_lib.HP_E_CLIP], vals[_lib.HP_ENTROPY_COEF] = float(lr), float(e_clip), float(entropy_coef)
    vals[_lib.HP_VF_COEF], vals[_lib.HP_MAX_GRAD_NORM] = float(vf_coef), float(max_grad_norm)
    vals[_lib.HP_VALUE_CLIP] = float(value_clip or 0.0)
    if value_norm is not None:
        vals[_lib.HP_VALUE_NORM_MEAN], vals[_lib.HP_VALUE_NORM_STD] = float(value_norm[0]), float(value_norm[1])
    vals[_lib.HP_KL_COEF], vals[_lib.HP_KL_STOP] = float(kl_coef), float(kl_stop or 0.0)
    return torch.tensor(vals, dtype=torch.float64, device=device)


# --------------------------------------------------------------------------------------------- value normalisation
def value_norm_stats(x, valid=None):
    """``[count, sum x, sum x^2]`` (fp64 device tensor, no sync) over the elements of ``x`` (fp32) where ``valid`` (bool,
    same number of elements, or None: all) is True -- ``dc_value_norm_stats``, bitwise reproducible."""
    _need_cuda(x, valid)
    x = _f32c(x).reshape(-1)
    if valid is not None:
        valid = _u8(valid).reshape(-1)
        assert valid.numel() == x.numel(), "valid has %d elements for %d values" % (valid.numel(), x.numel())
    out = torch.empty(3, dtype=torch.float64, device=x.device)
    with PROFILE.span("value_norm_stats", 1, 4 * x.numel() + (0 if valid is None else x.numel())):
        _lib.check(_lib.load().dc_value_norm_stats(x.data_ptr(), _lib.ptr(valid), x.numel(), out.data_ptr(),
                                                   _lib.stream_ptr()), "dc_value_norm_stats")
    return out


def value_denorm(v, mu, sigma):
    """``fp32(mu + sigma * v)`` computed in float64 (``dc_value_denorm``): a contiguous fp32 tensor of ``v``'s shape.
    ``v`` may be a strided view whose elements lie at one stride, such as the value column of the packed head GEMM."""
    _need_cuda(v)
    flat = v.detach().reshape(-1)
    if flat.dtype != torch.float32:
        flat = flat.float()
    n = flat.numel()
    ld = flat.stride(0) if n > 1 else 1
    out = torch.empty(v.shape, dtype=torch.float32, device=v.device)
    with PROFILE.span("value_denorm", 1, 8 * n):
        _lib.check(_lib.load().dc_value_denorm(flat.data_ptr(), ld, n, float(mu), float(sigma), out.data_ptr(),
                                               _lib.stream_ptr()), "dc_value_denorm")
    return out


def value_head_rescale(weight, bias, old, new):
    """The POP step in place on a value head's fp32 ``weight`` (contiguous, any shape) and ``bias`` (one element):
    ``sigma v + mu`` is preserved when the statistics move from ``old = (mu, sigma)`` to ``new``
    (``dc_value_head_rescale``)."""
    _need_cuda(weight, bias)
    assert weight.dtype == torch.float32 and bias.dtype == torch.float32 and weight.is_contiguous() and bias.numel() == 1
    with PROFILE.span("value_head_rescale", 1, 8 * (weight.numel() + 1)):
        _lib.check(_lib.load().dc_value_head_rescale(weight.data_ptr(), weight.numel(), bias.data_ptr(), float(old[0]),
                                                     float(old[1]), float(new[0]), float(new[1]), _lib.stream_ptr()),
                   "dc_value_head_rescale")


def _ppo_dev_args(hparams, old_value, stats, N, dev, valid=None, joint=False):
    """Checks the extra operands of ``dc_ppo_loss_fwd_bwd_dev`` / ``_masked`` / ``_joint``; allocates ``stats`` when not
    given."""
    if joint and hparams is None:
        raise ValueError("the joint-ratio PPO loss needs the device hyper-parameter block (hparams=)")
    if hparams is None:
        raise ValueError("the valid mask of the PPO loss needs the device hyper-parameter block (hparams=)")
    _need_cuda(hparams, old_value, valid)
    assert hparams.dtype == torch.float64 and hparams.numel() == _lib.HPARAM_SLOTS and hparams.is_contiguous()
    if old_value is not None:
        old_value = _f32c(old_value)
        assert old_value.numel() == N
    if valid is not None:
        if valid.dtype not in (torch.bool, torch.uint8):
            raise ValueError("valid must be a bool (or 0/1 uint8) tensor, got %s" % valid.dtype)
        valid = _u8(valid)
        assert valid.numel() == N, "valid has %d elements for %d tokens" % (valid.numel(), N)
    if stats is None:
        stats = torch.empty(_lib.PPO_STATS_SLOTS, dtype=torch.float32, device=dev)
    assert stats.dtype == torch.float32 and stats.numel() == _lib.PPO_STATS_SLOTS and stats.is_contiguous()
    return old_value, stats, valid


def _kl_args(old_log_probs, kl_out, N):
    """Checks the extra operands of ``dc_ppo_loss_fwd_bwd_kl``: ``old_log_probs`` [..., 65] fp32 (contiguous) and
    ``kl_out`` (2 fp32, or None)."""
    _need_cuda(old_log_probs, kl_out)
    old_log_probs = _f32c(old_log_probs)
    assert old_log_probs.numel() == N * _lib.KL_ROW_FLOATS, "old_log_probs has %d elements for %d tokens" % (
        old_log_probs.numel(), N)
    if kl_out is not None:
        assert kl_out.dtype == torch.float32 and kl_out.numel() == 2 and kl_out.is_contiguous()
    return old_log_probs


def _teacher_args(teacher_log_probs, teacher_coef, teacher_stats, N, dev):
    """Checks the extra operands of ``dc_ppo_loss_fwd_bwd_teacher``: ``teacher_log_probs`` [..., 65] fp32 (contiguous),
    ``teacher_coef`` (1 fp64 on the device) and ``teacher_stats`` (``_lib.TEACHER_STATS_SLOTS`` fp32, allocated when
    None)."""
    if teacher_coef is None:
        raise ValueError("the teacher term needs its coefficient on the device (teacher_coef=)")
    _need_cuda(teacher_log_probs, teacher_coef, teacher_stats)
    teacher_log_probs = _f32c(teacher_log_probs)
    assert teacher_log_probs.numel() == N * _lib.KL_ROW_FLOATS, "teacher_log_probs has %d elements for %d tokens" % (
        teacher_log_probs.numel(), N)
    assert teacher_coef.dtype == torch.float64 and teacher_coef.numel() == 1
    if teacher_stats is None:
        teacher_stats = torch.empty(_lib.TEACHER_STATS_SLOTS, dtype=torch.float32, device=dev)
    assert teacher_stats.dtype == torch.float32 and teacher_stats.numel() == _lib.TEACHER_STATS_SLOTS \
        and teacher_stats.is_contiguous()
    return teacher_log_probs, teacher_stats


def _bc_args(bc_stats, dev, joint, old_log_probs, teacher_log_probs):
    """Checks the extra operand of ``dc_ppo_loss_fwd_bwd_bc``: ``bc_stats`` (``_lib.BC_STATS_SLOTS`` fp32, allocated when
    None), and that nothing that belongs to the policy-gradient objective was asked for with it."""
    if joint or old_log_probs is not None or teacher_log_probs is not None:
        raise ValueError("behaviour cloning has no PPO ratio, KL penalty or teacher term (joint / old_log_probs / "
                         "teacher_log_probs)")
    _need_cuda(bc_stats)
    if bc_stats is None:
        bc_stats = torch.empty(_lib.BC_STATS_SLOTS, dtype=torch.float32, device=dev)
    assert bc_stats.dtype == torch.float32 and bc_stats.numel() == _lib.BC_STATS_SLOTS and bc_stats.is_contiguous()
    return bc_stats


def _dual_clip_args(dual_clip, dual_clip_stats, dev):
    """Checks the extra operands of ``dc_ppo_loss_fwd_bwd_dual_clip``: ``dual_clip`` (1 fp64 on the device, c > 1) and
    ``dual_clip_stats`` (``_lib.DUAL_CLIP_STATS_SLOTS`` fp32, allocated when None)."""
    _need_cuda(dual_clip, dual_clip_stats)
    assert dual_clip.dtype == torch.float64 and dual_clip.numel() == 1
    if dual_clip_stats is None:
        dual_clip_stats = torch.empty(_lib.DUAL_CLIP_STATS_SLOTS, dtype=torch.float32, device=dev)
    assert dual_clip_stats.dtype == torch.float32 and dual_clip_stats.numel() == _lib.DUAL_CLIP_STATS_SLOTS \
        and dual_clip_stats.is_contiguous()
    return dual_clip_stats


def _ppo_dev_call(lib, lptr, ld_l, masks, actions, old_logp, adv_raw, ret, value_ptr, ld_v, old_value, valid, N, hparams,
                  dptr, ld_d, dvalue_ptr, ld_dv, out, stats, n_actions, ws, joint=False, old_log_probs=None, kl_out=None,
                  teacher_log_probs=None, teacher_coef=None, teacher_stats=None, bc_stats=None, dual_clip=None,
                  dual_clip_stats=None):
    """``dc_ppo_loss_fwd_bwd_dev``, or ``dc_ppo_loss_fwd_bwd_masked`` when a valid mask is given, or
    ``dc_ppo_loss_fwd_bwd_joint`` (valid or not) when ``joint``; ``dc_ppo_loss_fwd_bwd_kl`` (either ratio mode) when
    ``old_log_probs`` is given; ``dc_ppo_loss_fwd_bwd_teacher`` (either ratio mode, old rows or not) when
    ``teacher_log_probs`` is given; ``dc_ppo_loss_fwd_bwd_bc`` (valid or not; ``old_logp`` unused) when ``bc_stats`` is
    given; ``dc_ppo_loss_fwd_bwd_dual_clip`` (either ratio mode, with or without the old and the teacher's rows) when
    ``dual_clip`` is given."""
    if bc_stats is not None:
        with PROFILE.span("ppo_loss", 2):
            _lib.check(lib.dc_ppo_loss_fwd_bwd_bc(
                lptr, ld_l, _lib.ptr5(masks), _lib.ptr5(actions), adv_raw.data_ptr(), ret.data_ptr(), value_ptr, ld_v,
                _lib.ptr(old_value), _lib.ptr(valid), N, hparams.data_ptr(), dptr, ld_d, dvalue_ptr, ld_dv, out.data_ptr(),
                stats.data_ptr(), bc_stats.data_ptr(), n_actions.data_ptr(), ws.data_ptr(), _lib.stream_ptr()),
                "dc_ppo_loss_fwd_bwd_bc")
        return
    head = (lptr, ld_l, _lib.ptr5(masks), _lib.ptr5(actions), old_logp.data_ptr(), adv_raw.data_ptr(), ret.data_ptr(),
            value_ptr, ld_v, _lib.ptr(old_value))
    tail = (N, hparams.data_ptr(), dptr, ld_d, dvalue_ptr, ld_dv, out.data_ptr(), stats.data_ptr(), n_actions.data_ptr(),
            ws.data_ptr(), _lib.stream_ptr())
    rows = (old_log_probs is not None) + (teacher_log_probs is not None)
    with PROFILE.span("ppo_loss", 2, _lib.KL_ROW_FLOATS * 4 * N * rows):
        if dual_clip is not None:
            _lib.check(lib.dc_ppo_loss_fwd_bwd_dual_clip(
                lptr, ld_l, _lib.ptr5(masks), _lib.ptr5(actions), old_logp.data_ptr(), _lib.ptr(old_log_probs),
                _lib.ptr(teacher_log_probs), adv_raw.data_ptr(), ret.data_ptr(), value_ptr, ld_v, _lib.ptr(old_value),
                _lib.ptr(valid), N, hparams.data_ptr(), _lib.ptr(teacher_coef), dual_clip.data_ptr(), 1 if joint else 0,
                dptr, ld_d, dvalue_ptr, ld_dv, out.data_ptr(), stats.data_ptr(), _lib.ptr(kl_out),
                _lib.ptr(teacher_stats), dual_clip_stats.data_ptr(), n_actions.data_ptr(), ws.data_ptr(),
                _lib.stream_ptr()), "dc_ppo_loss_fwd_bwd_dual_clip")
        elif teacher_log_probs is not None:
            _lib.check(lib.dc_ppo_loss_fwd_bwd_teacher(
                lptr, ld_l, _lib.ptr5(masks), _lib.ptr5(actions), old_logp.data_ptr(), _lib.ptr(old_log_probs),
                teacher_log_probs.data_ptr(), adv_raw.data_ptr(), ret.data_ptr(), value_ptr, ld_v, _lib.ptr(old_value),
                _lib.ptr(valid), N, hparams.data_ptr(), teacher_coef.data_ptr(), 1 if joint else 0, dptr, ld_d, dvalue_ptr,
                ld_dv, out.data_ptr(), stats.data_ptr(), _lib.ptr(kl_out), teacher_stats.data_ptr(), n_actions.data_ptr(),
                ws.data_ptr(), _lib.stream_ptr()), "dc_ppo_loss_fwd_bwd_teacher")
        elif old_log_probs is not None:
            _lib.check(lib.dc_ppo_loss_fwd_bwd_kl(
                lptr, ld_l, _lib.ptr5(masks), _lib.ptr5(actions), old_logp.data_ptr(), old_log_probs.data_ptr(),
                adv_raw.data_ptr(), ret.data_ptr(), value_ptr, ld_v, _lib.ptr(old_value), _lib.ptr(valid), N,
                hparams.data_ptr(), 1 if joint else 0, dptr, ld_d, dvalue_ptr, ld_dv, out.data_ptr(), stats.data_ptr(),
                _lib.ptr(kl_out), n_actions.data_ptr(), ws.data_ptr(), _lib.stream_ptr()), "dc_ppo_loss_fwd_bwd_kl")
        elif joint:
            _lib.check(lib.dc_ppo_loss_fwd_bwd_joint(*head, _lib.ptr(valid), *tail), "dc_ppo_loss_fwd_bwd_joint")
        elif valid is None:
            _lib.check(lib.dc_ppo_loss_fwd_bwd_dev(*head, *tail), "dc_ppo_loss_fwd_bwd_dev")
        else:
            _lib.check(lib.dc_ppo_loss_fwd_bwd_masked(*head, valid.data_ptr(), *tail), "dc_ppo_loss_fwd_bwd_masked")


def ppo_loss_fwd_bwd(logits, masks, actions, old_logp, adv_raw, ret, value, e_clip, entropy_coef, vf_coef, hparams=None,
                     old_value=None, stats=None, valid=None, joint=False, old_log_probs=None, kl_out=None,
                     teacher_log_probs=None, teacher_coef=None, teacher_stats=None, bc=False, bc_stats=None,
                     dual_clip=None, dual_clip_stats=None):
    """Fused PPO loss + gradients (``optimizer.py:587-589,621-665`` and their backward).

    logits/masks/actions: sequences of 5 tensors [..., n_h] in HEAD_KEYS order (any leading dims,
    same token order everywhere); old_logp [..., 5]; adv_raw/ret/value [...].
    Returns (out[16] fp32, n_actions[5] int32, dlogits list, dvalue) -- all on device, no sync.

    ``hparams`` (a device block from ``hparam_block``): the hyper-parameters are read from it on the device
    (``dc_ppo_loss_fwd_bwd_dev``; ``e_clip`` / ``entropy_coef`` / ``vf_coef`` are then ignored), the value loss is clipped
    against ``old_value`` [...] when the block's value clip is > 0, and the PPO diagnostics go to ``stats``
    [``_lib.PPO_STATS_SLOTS``]; the return value gains that tensor as a fifth element.
    ``valid`` [...] bool (needs ``hparams``): tokens where it is False count for nothing and get zero gradients
    (``dc_ppo_loss_fwd_bwd_masked``); None is the unmasked loss.
    ``joint`` (needs ``hparams``): one clipped PPO ratio per token, of the whole hierarchical action, instead of one per
    head (``dc_ppo_loss_fwd_bwd_joint``, with or without ``valid``); ``stats`` then also holds the joint ratio's KL and
    clip fraction (``_lib.STAT_JOINT_APPROX_KL`` / ``STAT_JOINT_CLIP_FRACTION``).
    ``old_log_probs`` [..., 65] (needs ``hparams``): the prep-time masked log-prob rows (``selected_logp_rows``); the loss
    then adds the KL penalty ``hparams[HP_KL_COEF] * KL`` (``dc_ppo_loss_fwd_bwd_kl``, either ratio mode), ``stats``
    also holds the exact KL (``_lib.STAT_KL``...), and ``kl_out`` (2 fp32, or None) receives (sum_t KL_t, T_a).
    ``teacher_log_probs`` [..., 65] (needs ``hparams`` and ``teacher_coef``, 1 fp64 on the device): a teacher policy's
    masked log-prob rows; the loss then adds ``teacher_coef * KL(teacher || policy)`` (``dc_ppo_loss_fwd_bwd_teacher``,
    either ratio mode, with or without ``old_log_probs``), and ``teacher_stats`` (``_lib.TEACHER_STATS_SLOTS`` fp32,
    allocated when None) receives the KL, the KL per head and the term; the result then gains it as a sixth element.
    ``bc`` (needs ``hparams``): behaviour cloning, the negative log-likelihood of the actions in place of the PPO surrogate
    (``dc_ppo_loss_fwd_bwd_bc``, with or without ``valid``; ``old_logp`` may be None and is not read); ``bc_stats``
    (``_lib.BC_STATS_SLOTS`` fp32, allocated when None) receives the NLL, per head, the token accuracy and per head, and the
    result gains it as a sixth element.
    ``dual_clip`` (needs ``hparams``; 1 fp64 on the device, c > 1): dual-clip PPO, the surrogate of every row with a
    negative normalised advantage A is floored at c A (``dc_ppo_loss_fwd_bwd_dual_clip``, either ratio mode, with or
    without ``valid``, ``old_log_probs`` and ``teacher_log_probs``); ``dual_clip_stats``
    (``_lib.DUAL_CLIP_STATS_SLOTS`` fp32, allocated when None) receives the shares of the rows where the floor binds, and the
    result gains it as its last element (after ``teacher_stats`` with a teacher).
    """
    if bc and dual_clip is not None:
        raise ValueError("behaviour cloning has no PPO surrogate for dual clip to bound")
    logits = [_f32c(l.detach()) for l in logits]
    _need_cuda(*logits)
    N = logits[0].numel() // HEAD_SIZES[0]
    masks = [_u8(m) for m in masks]
    actions = [_u8(a) for a in actions]
    for h in range(5):
        assert logits[h].numel() == N * HEAD_SIZES[h] and masks[h].numel() == N * HEAD_SIZES[h] \
            and actions[h].numel() == N * HEAD_SIZES[h], "head %d shape mismatch" % h
    old_logp = None if bc else _f32c(old_logp)
    adv_raw, ret, value = _f32c(adv_raw), _f32c(ret), _f32c(value.detach())
    assert (bc or old_logp.numel() == N * 5) and adv_raw.numel() == N and ret.numel() == N and value.numel() == N
    dev = logits[0].device
    dlogits = [torch.empty_like(l) for l in logits]
    dvalue = torch.empty_like(value)
    out = torch.empty(_lib.LOSS_SLOTS, dtype=torch.float32, device=dev)
    n_actions = torch.empty(5, dtype=torch.int32, device=dev)
    ws = torch.empty(_lib.PPO_WORKSPACE_BYTES, dtype=torch.uint8, device=dev)
    lib = _lib.load()
    teacher = teacher_log_probs is not None
    dual = dual_clip is not None
    if hparams is not None or valid is not None or joint or old_log_probs is not None or teacher or bc or dual:
        if (old_log_probs is not None or teacher or bc or dual) and hparams is None:
            raise ValueError("the KL penalty, the teacher term, behaviour cloning and dual clip need the device "
                             "hyper-parameter block (hparams=)")
        old_value, stats, valid = _ppo_dev_args(hparams, old_value, stats, N, dev, valid, joint)
        if bc:
            bc_stats = _bc_args(bc_stats, dev, joint, old_log_probs, teacher_log_probs)
        if dual:
            dual_clip_stats = _dual_clip_args(dual_clip, dual_clip_stats, dev)
        if old_log_probs is not None:
            old_log_probs = _kl_args(old_log_probs, kl_out, N)
        if teacher:
            teacher_log_probs, teacher_stats = _teacher_args(teacher_log_probs, teacher_coef, teacher_stats, N, dev)
        ld = (ctypes.c_int64 * 5)(*HEAD_SIZES)
        _ppo_dev_call(lib, _lib.ptr5(logits), ld, masks, actions, old_logp, adv_raw, ret, value.data_ptr(), 1, old_value,
                      valid, N, hparams, _lib.ptr5(dlogits), ld, dvalue.data_ptr(), 1, out, stats, n_actions, ws, joint,
                      old_log_probs, kl_out, teacher_log_probs, teacher_coef, teacher_stats, bc_stats if bc else None,
                      dual_clip, dual_clip_stats)
        res = (out, n_actions, dlogits, dvalue, stats)
        res = res + (teacher_stats,) if teacher else res + (bc_stats,) if bc else res
        return res + (dual_clip_stats,) if dual else res
    with PROFILE.span("ppo_loss", 2):
        _lib.check(lib.dc_ppo_loss_fwd_bwd(_lib.ptr5(logits), _lib.ptr5(masks), _lib.ptr5(actions),
                                           old_logp.data_ptr(), adv_raw.data_ptr(), ret.data_ptr(), value.data_ptr(),
                                           N, float(e_clip), float(entropy_coef), float(vf_coef), _lib.ptr5(dlogits),
                                           dvalue.data_ptr(), out.data_ptr(), n_actions.data_ptr(), ws.data_ptr(),
                                           _lib.stream_ptr()), "dc_ppo_loss_fwd_bwd")
    return out, n_actions, dlogits, dvalue


def selected_logp(logits, masks, actions):
    """Dense [N,5] log-prob of the taken action per head (0 where none) -- ``optimizer.py:387-390``."""
    logits = [_f32c(l.detach()) for l in logits]
    _need_cuda(*logits)
    N = logits[0].numel() // HEAD_SIZES[0]
    masks = [_u8(m) for m in masks]
    actions = [_u8(a) for a in actions]
    out = torch.empty((N, 5), dtype=torch.float32, device=logits[0].device)
    lib = _lib.load()
    with PROFILE.span("selected_logp", 1):
        _lib.check(lib.dc_selected_logp(_lib.ptr5(logits), _lib.ptr5(masks), _lib.ptr5(actions), N, out.data_ptr(),
                                        _lib.stream_ptr()), "dc_selected_logp")
    return out


def selected_logp_rows(logits, masks, actions):
    """``selected_logp``'s dense [N,5] log-probs (the same bits) and every head's full masked log-prob row, [N,65] in head
    order with 0 at illegal entries -- the prep-time distribution the KL penalty compares against
    (``dc_selected_logp_rows``)."""
    logits = [_f32c(l.detach()) for l in logits]
    _need_cuda(*logits)
    N = logits[0].numel() // HEAD_SIZES[0]
    masks = [_u8(m) for m in masks]
    actions = [_u8(a) for a in actions]
    dev = logits[0].device
    out = torch.empty((N, 5), dtype=torch.float32, device=dev)
    rows = torch.empty((N, _lib.KL_ROW_FLOATS), dtype=torch.float32, device=dev)
    with PROFILE.span("selected_logp_rows", 1, 4 * N * _lib.KL_ROW_FLOATS):
        _lib.check(_lib.load().dc_selected_logp_rows(_lib.ptr5(logits), _lib.ptr5(masks), _lib.ptr5(actions), N,
                                                     out.data_ptr(), rows.data_ptr(), _lib.stream_ptr()),
                   "dc_selected_logp_rows")
    return out, rows


# --------------------------------------------------------------------------------------------- grad finish
def grad_flags(flat_grad, total, seg_head, n_actions):
    lib = _lib.load()
    with PROFILE.span("grad_flags", 1):
        _lib.check(lib.dc_grad_flags(flat_grad.data_ptr(), total, seg_head.data_ptr(), seg_head.numel(),
                                     n_actions.data_ptr(), _lib.stream_ptr()), "dc_grad_flags")


def grad_finish(flat_param, flat_grad, exp_avg, exp_avg_sq, steps, seg_lo, seg_hi, seg_head, total, lr, betas, eps,
                max_norm, loss_out, metrics, workspace, hparams=None, kl=False):
    """Count-divide, grad norms, clip and Adam on the flat buffers.  With ``hparams`` (a device block, ``hparam_block``)
    ``lr`` and ``max_norm`` are read from it on the device (``dc_grad_finish_dev``) and the arguments are ignored.
    ``kl`` (needs ``hparams``): ``flat_grad`` carries the all-reduced (sum_t KL_t, T_a) behind the flags, the step is
    skipped when that KL exceeds the block's KL limit, and ``metrics`` (``_lib.FINISH_KL_METRICS``) also gets the KL and
    the skip flag (``dc_grad_finish_kl``)."""
    lib = _lib.load()
    if kl and hparams is None:
        raise ValueError("the KL early stop needs the device hyper-parameter block (hparams=)")
    if hparams is not None:
        _need_cuda(hparams)
        assert hparams.dtype == torch.float64 and hparams.numel() == _lib.HPARAM_SLOTS and hparams.is_contiguous()
        if kl:
            n_seg = seg_head.numel()
            assert flat_grad.numel() >= total + n_seg + 2 and metrics.numel() >= _lib.FINISH_KL_METRICS
        with PROFILE.span("grad_finish", 3):
            _lib.check((lib.dc_grad_finish_kl if kl else lib.dc_grad_finish_dev)(flat_param.data_ptr(), flat_grad.data_ptr(), exp_avg.data_ptr(),
                                              exp_avg_sq.data_ptr(), steps.data_ptr(), seg_lo.data_ptr(), seg_hi.data_ptr(),
                                              seg_head.data_ptr(), seg_head.numel(), total, hparams.data_ptr(),
                                              float(betas[0]), float(betas[1]), float(eps), _lib.ptr(loss_out),
                                              metrics.data_ptr(), workspace.data_ptr(), _lib.stream_ptr()),
                       "dc_grad_finish_kl" if kl else "dc_grad_finish_dev")
        return
    with PROFILE.span("grad_finish", 3):
        _lib.check(lib.dc_grad_finish(flat_param.data_ptr(), flat_grad.data_ptr(), exp_avg.data_ptr(),
                                      exp_avg_sq.data_ptr(), steps.data_ptr(), seg_lo.data_ptr(), seg_hi.data_ptr(),
                                      seg_head.data_ptr(),
                                      seg_head.numel(), total, float(lr), float(betas[0]), float(betas[1]), float(eps),
                                      float(max_norm), _lib.ptr(loss_out), metrics.data_ptr(), workspace.data_ptr(),
                                      _lib.stream_ptr()), "dc_grad_finish")


# --------------------------------------------------------------------------------------------- tensor-core GEMM
def gemm_tf32x3_supported(M, N, K):
    return bool(_lib.load().dc_gemm_tf32x3_supported(int(M), int(N), int(K)))


def gemm_tf32x3(a, b, bias=None, relu=False, out=None):
    """``out[M,N] = a[M,K] @ b[N,K]^T (+ bias) (ReLU)`` on Hopper tensor cores (wgmma) with the 3xTF32 split
    (fp32-level accuracy).  ``a``/``b``/``out`` are 2-D fp32 CUDA tensors whose rows are contiguous (row stride
    may exceed the width: column-slice views are fine)."""
    _need_cuda(a, b, bias)
    assert a.dim() == 2 and b.dim() == 2 and a.shape[1] == b.shape[1]
    if a.stride(1) != 1:
        a = a.contiguous()
    if b.stride(1) != 1:
        b = b.contiguous()
    M, K = a.shape
    N = b.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    assert out.shape == (M, N) and out.stride(1) == 1
    lib = _lib.load()
    with PROFILE.span("gemm_tf32x3", 1, 4 * (M * K + N * K + M * N)):
        _lib.check(lib.dc_gemm_tf32x3(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), _lib.ptr(bias), out.data_ptr(),
                                      out.stride(0), M, N, K, 1 if relu else 0, _lib.stream_ptr()), "dc_gemm_tf32x3")
    return out


class LinearTC(torch.autograd.Function):
    """``y = x W^T + b`` (optionally ReLU): forward, data gradient and weight gradient (+ bias gradient from the same pass
    over ``dy``) all on the wgmma 3xTF32 GEMMs.  No library GEMM: unsupported shapes raise ``DC_EUNSUPPORTED``."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu):
        shp = x.shape
        x2 = _f32c(x.detach()).reshape(-1, shp[-1])
        w = _f32c(weight.detach())
        y = gemm_tf32x3(x2, w, None if bias is None else _f32c(bias.detach()), relu=relu)
        ctx.relu = relu
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x2, w, y if relu else None)
        return y.view(*shp[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w, y = ctx.saved_tensors
        N, K = w.shape
        dy2 = _f32c(dy).reshape(-1, N)
        if ctx.relu:
            dy2 = torch.ops.aten.threshold_backward(dy2, y, 0.0)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = gemm_tf32x3(dy2, w.t().contiguous()).view(*dy.shape[:-1], K)
        dw = db = None
        if ctx.needs_input_grad[1]:
            dw, db = gemm_wgrad_tf32x3(dy2, x2, want_bias=ctx.has_bias)     # dW = dy^T x, db = colsum(dy), one pass over dy
        return dx, dw, db, None


def linear(x, weight, bias=None, relu=False):
    """Dense layer on the wgmma 3xTF32 GEMM (out features % 32 == 0, in features % 32 == 0; CUDA tensors only)."""
    _need_cuda(x, weight, bias)
    return LinearTC.apply(x, weight, bias, relu)


_wgrad_ws = {}


def gemm_wgrad_supported(T, No, Ni):
    return T > 0 and No % 32 == 0 and Ni % 32 == 0


def gemm_wgrad_tf32x3(dy, x, want_bias=True, dw_out=None, db_out=None, accumulate=False, t_dev=None, t_host=None, x_rows=None):
    """``dW[No,Ni] = dy[T,No]^T @ x[T,Ni]`` and ``db[No] = dy.sum(0)`` on wgmma (3xTF32, split-K, deterministic).

    ``dy`` / ``x`` are 2-D fp32 CUDA tensors with contiguous rows (column-slice views allowed).  ``t_dev`` / ``t_host``:
    only the rows ``t < min(T, t_dev)`` (an int32 CUDA tensor of one element) are summed; ``t_host``: that count when the
    caller knows it, for the profile's byte count only.  ``x_rows`` (int32, with ``t_dev``): row t of the product is row
    ``x_rows[t]`` of ``x``."""
    _need_cuda(dy, x)
    assert dy.dim() == 2 and x.dim() == 2 and (x_rows is not None or dy.shape[0] == x.shape[0])
    if dy.stride(1) != 1:
        dy = dy.contiguous()
    if x.stride(1) != 1:
        x = x.contiguous()
    T, No = dy.shape
    Ni = x.shape[1]
    dev = dy.device
    if dw_out is None:
        dw_out = torch.empty((No, Ni), dtype=torch.float32, device=dev)
    if want_bias and db_out is None:
        db_out = torch.empty(No, dtype=torch.float32, device=dev)
    lib = _lib.load()
    key = (No, Ni, dev)
    ws = _wgrad_ws.get(key)
    if ws is None:
        ws = torch.empty(int(lib.dc_gemm_wgrad_workspace_bytes(No, Ni)), dtype=torch.uint8, device=dev)
        _wgrad_ws[key] = ws
    Tb = T if t_host is None else t_host
    with PROFILE.span("gemm_wgrad", 2, 4 * (Tb * No + Tb * Ni + No * Ni)):
        if t_dev is None:
            _lib.check(lib.dc_gemm_wgrad_tf32x3(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), T, No, Ni,
                                                dw_out.data_ptr(), dw_out.stride(0), _lib.ptr(db_out) if want_bias else None,
                                                1 if accumulate else 0, ws.data_ptr(), _lib.stream_ptr()),
                       "dc_gemm_wgrad_tf32x3")
        else:
            _lib.check(lib.dc_gemm_wgrad_tf32x3_rows(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), _lib.ptr(x_rows), T,
                                                     t_dev.data_ptr(),
                                                     No, Ni, dw_out.data_ptr(), dw_out.stride(0),
                                                     _lib.ptr(db_out) if want_bias else None, 1 if accumulate else 0,
                                                     ws.data_ptr(), _lib.stream_ptr()), "dc_gemm_wgrad_tf32x3_rows")
    return dw_out, (db_out if want_bias else None)


def select_actions(logits, masks, u):
    """Hierarchical action selection for ``A`` agents in one launch (``policy.py:190-216``).

    ``logits`` / ``masks``: five ``[A, n_h]`` tensors in ``HEAD_KEYS`` order (rows may be strided column slices);
    ``u``: ``[A, 5]`` uniforms in [0, 1).  Returns ``(chosen [A,5] int32, logp [A,5] fp32)``; ``chosen`` is -1 for the
    sub-heads the sampled enum does not use.  The index function is ``oracle.ref_policy.sample_index``'s inverse CDF; the
    two differ in fp32 rounding (CUDA ``expf`` and a sequential normaliser against torch's), so they can take adjacent legal
    indices when u lies within that rounding of a cumulative boundary."""
    _need_cuda(u, *logits, *masks)
    A = u.shape[0]
    ls, lds, ms = [], [], []
    for h, (l, m) in enumerate(zip(logits, masks)):
        l2 = l.reshape(A, HEAD_SIZES[h]).float()
        if l2.stride(1) != 1:
            l2 = l2.contiguous()
        ls.append(l2)
        lds.append(l2.stride(0))
        ms.append(m.reshape(A, HEAD_SIZES[h]).contiguous().view(torch.uint8))
    u2 = _f32c(u).reshape(A, 5)
    chosen = torch.empty((A, 5), dtype=torch.int32, device=u.device)
    logp = torch.empty((A, 5), dtype=torch.float32, device=u.device)
    with PROFILE.span("select_actions", 1):
        _lib.check(_lib.load().dc_select_actions(_lib.ptr5(ls), (ctypes.c_int64 * 5)(*lds), _lib.ptr5(ms), u2.data_ptr(), A,
                                                 chosen.data_ptr(), logp.data_ptr(), _lib.stream_ptr()), "dc_select_actions")
    return chosen, logp


# --------------------------------------------------------------------------------------------- packed small heads
PACK_COLS = {"enum": (0, 4), "x": (4, 13), "y": (13, 22), "ability": (22, 25), "value": (25, 26)}   # columns of the packed GEMM
PACK_WIDTH = 128


def pack_cols(K=1):
    """The columns of the packed GEMM for a policy with ``K`` value heads: ``PACK_COLS`` with ``value`` = (25, 25 + K)."""
    return dict(PACK_COLS, value=(25, 25 + int(K)))


_value_heads_ws = {}


def value_heads_loss(packed, d_packed, ret, hparams, out, head_stats, old_value=None, valid=None, stats=None):
    """The value term of ``K`` value heads (``dc_value_heads_loss``), run after ``ppo_loss_packed`` with a hparams block
    whose value term is off: reads the K value columns of ``packed`` [..., PACK_WIDTH] and ``ret`` [N, K] (``old_value``
    [N, K] for the clipped loss, ``valid`` [N]), writes the K value columns of ``d_packed``, ``out[3]`` (and adds it to
    ``out[0]``), ``head_stats`` [``_lib.VALUE_HEADS_STATS_SLOTS``] and the total's explained variance into ``stats``."""
    _need_cuda(packed, d_packed, ret, hparams, out, head_stats, old_value, valid, stats)
    p2 = packed.detach().reshape(-1, PACK_WIDTH)
    d2 = d_packed.reshape(-1, PACK_WIDTH)
    N = p2.shape[0]
    ret = _f32c(ret)
    K = ret.numel() // max(N, 1)
    if ret.numel() != N * K or not 1 <= K <= _lib.VALUE_HEADS_MAX:
        raise ValueError("ret has %d elements for %d tokens" % (ret.numel(), N))
    assert p2.is_contiguous() and d2.is_contiguous() and p2.dtype == torch.float32 and d2.dtype == torch.float32
    assert hparams.dtype == torch.float64 and hparams.numel() == _lib.HPARAM_SLOTS
    assert head_stats.dtype == torch.float32 and head_stats.numel() == _lib.VALUE_HEADS_STATS_SLOTS
    if old_value is not None:
        old_value = _f32c(old_value)
        assert old_value.numel() == N * K
    if valid is not None:
        valid = _u8(valid)
        assert valid.numel() == N
    ws = _value_heads_ws.get(p2.device)
    if ws is None:
        ws = _value_heads_ws[p2.device] = torch.empty(_lib.VALUE_HEADS_WORKSPACE_BYTES, dtype=torch.uint8, device=p2.device)
    col = 4 * PACK_COLS["value"][0]
    with PROFILE.span("value_heads_loss", 3, N * (12 * K + (0 if valid is None else 1) + (0 if old_value is None else 4 * K))):
        _lib.check(_lib.load().dc_value_heads_loss(p2.data_ptr() + col, PACK_WIDTH, ret.data_ptr(), _lib.ptr(old_value),
                                                   _lib.ptr(valid), N, K, hparams.data_ptr(), d2.data_ptr() + col,
                                                   PACK_WIDTH, out.data_ptr(), _lib.ptr(stats), head_stats.data_ptr(),
                                                   ws.data_ptr(), _lib.stream_ptr()), "dc_value_heads_loss")


def ppo_loss_packed(packed, logits_tu, masks, actions, old_logp, adv_raw, ret, e_clip, entropy_coef, vf_coef, hparams=None,
                    old_value=None, stats=None, valid=None, joint=False, old_log_probs=None, kl_out=None,
                    teacher_log_probs=None, teacher_coef=None, teacher_stats=None, bc=False, bc_stats=None,
                    dual_clip=None, dual_clip_stats=None):
    """Fused PPO loss where the four small heads and the value head are column ranges of ONE packed ``[N,128]``
    tensor-core GEMM output (``PACK_COLS``) and the target-unit logits are a separate ``[N,40]`` tensor.

    Returns (out[16], n_actions[5], d_packed [N,128], d_logits_tu [N,40]): the gradients go straight back into the two
    producers, so no slice/cat kernels run and the five tiny K=131072 weight-gradient GEMMs become one wgmma wgrad.
    ``hparams`` / ``old_value`` / ``stats`` / ``valid`` / ``joint`` / ``old_log_probs`` / ``kl_out`` /
    ``teacher_log_probs`` / ``teacher_coef`` / ``teacher_stats`` / ``bc`` / ``bc_stats`` / ``dual_clip`` /
    ``dual_clip_stats``: as ``ppo_loss_fwd_bwd`` (the fifth element of the result is then ``stats``, and with a teacher the
    sixth ``teacher_stats``, with ``bc`` ``bc_stats``; with ``dual_clip`` ``dual_clip_stats`` comes last).
    """
    if bc and dual_clip is not None:
        raise ValueError("behaviour cloning has no PPO surrogate for dual clip to bound")
    _need_cuda(packed, logits_tu)
    p2 = _f32c(packed.detach()).reshape(-1, PACK_WIDTH)
    N = p2.shape[0]
    tu = _f32c(logits_tu.detach()).reshape(N, 40)
    masks = [_u8(m) for m in masks]
    actions = [_u8(a) for a in actions]
    old_logp = None if bc else _f32c(old_logp)
    adv_raw, ret = _f32c(adv_raw), _f32c(ret)
    dev = p2.device
    d_packed = torch.zeros_like(p2)            # the 102 padding columns must carry a zero gradient
    d_tu = torch.empty_like(tu)
    out = torch.empty(_lib.LOSS_SLOTS, dtype=torch.float32, device=dev)
    n_actions = torch.empty(5, dtype=torch.int32, device=dev)
    ws = torch.empty(_lib.PPO_WORKSPACE_BYTES, dtype=torch.uint8, device=dev)

    def col(t, key):
        return t.data_ptr() + 4 * PACK_COLS[key][0]
    c = _lib._c
    lptr = _lib._ptr5(col(p2, "enum"), col(p2, "x"), col(p2, "y"), tu.data_ptr(), col(p2, "ability"))
    dptr = _lib._ptr5(col(d_packed, "enum"), col(d_packed, "x"), col(d_packed, "y"), d_tu.data_ptr(), col(d_packed, "ability"))
    ld = (c.c_int64 * 5)(PACK_WIDTH, PACK_WIDTH, PACK_WIDTH, 40, PACK_WIDTH)
    lib = _lib.load()
    teacher = teacher_log_probs is not None
    dual = dual_clip is not None
    if hparams is not None or valid is not None or joint or old_log_probs is not None or teacher or bc or dual:
        if (old_log_probs is not None or teacher or bc or dual) and hparams is None:
            raise ValueError("the KL penalty, the teacher term, behaviour cloning and dual clip need the device "
                             "hyper-parameter block (hparams=)")
        old_value, stats, valid = _ppo_dev_args(hparams, old_value, stats, N, dev, valid, joint)
        if bc:
            bc_stats = _bc_args(bc_stats, dev, joint, old_log_probs, teacher_log_probs)
        if dual:
            dual_clip_stats = _dual_clip_args(dual_clip, dual_clip_stats, dev)
        if old_log_probs is not None:
            old_log_probs = _kl_args(old_log_probs, kl_out, N)
        if teacher:
            teacher_log_probs, teacher_stats = _teacher_args(teacher_log_probs, teacher_coef, teacher_stats, N, dev)
        _ppo_dev_call(lib, lptr, ld, masks, actions, old_logp, adv_raw, ret, col(p2, "value"), PACK_WIDTH, old_value, valid,
                      N, hparams, dptr, ld, col(d_packed, "value"), PACK_WIDTH, out, stats, n_actions, ws, joint,
                      old_log_probs, kl_out, teacher_log_probs, teacher_coef, teacher_stats, bc_stats if bc else None,
                      dual_clip, dual_clip_stats)
        res = (out, n_actions, d_packed.view_as(packed), d_tu.view_as(logits_tu), stats)
        res = res + (teacher_stats,) if teacher else res + (bc_stats,) if bc else res
        return res + (dual_clip_stats,) if dual else res
    with PROFILE.span("ppo_loss", 2):
        _lib.check(lib.dc_ppo_loss_fwd_bwd_strided(lptr, ld, _lib.ptr5(masks), _lib.ptr5(actions), old_logp.data_ptr(),
                                                   adv_raw.data_ptr(), ret.data_ptr(), col(p2, "value"), PACK_WIDTH, N,
                                                   float(e_clip), float(entropy_coef), float(vf_coef), dptr, ld,
                                                   col(d_packed, "value"), PACK_WIDTH, out.data_ptr(), n_actions.data_ptr(),
                                                   ws.data_ptr(), _lib.stream_ptr()), "dc_ppo_loss_fwd_bwd_strided")
    return out, n_actions, d_packed.view_as(packed), d_tu.view_as(logits_tu)
