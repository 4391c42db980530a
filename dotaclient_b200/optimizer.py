"""``DotaOptimizer`` -- drop-in for the hot path of the reference's ``optimizer.py``.

Keeps the reference's module surface (``DotaOptimizer``, ``Sequence``, ``MessageQueue``,
``advantage_returns``, ``discount``, ``init_distribution``, ``main``, the CLI flags) while one
optimizer step runs as:  unit-encoder kernel chain + wgmma 3xTF32 GEMMs -> hand-written recurrence kernels ->
fused PPO loss+grad kernel -> autograd backward through the same kernels -> ONE NCCL all-reduce of
a flat gradient buffer -> fused count-divide / grad-norm / clip / Adam kernel -- replayed from a CUDA graph
when the batch is device-resident.  CUDA only.

Line references are to TimZaman/dotaclient ``optimizer.py`` @ 8615b90.
"""
import argparse
import collections.abc
import gc
import io
import logging
import math
import numbers
import os
import pickle
import queue
import re
import socket
import threading
import time
import typing
from datetime import datetime

import numpy as np
import torch
import torch.distributed as dist

from . import _lib, ops
from .distributed import DistributedDataParallelSparseParamCPU
from .flat import FlatParameterSpace, VALUE_SLOT
from .policy import Policy, REWARD_KEYS, fold_value_heads, split_value_head

logging.basicConfig(format='%(asctime)s %(levelname)-8s %(message)s')
logger = logging.getLogger(__name__)
logger.setLevel(logging.INFO)

eps = np.finfo(np.float32).eps.item()                                  # :38
GAMMA, LAMBDA = 0.98, 0.97                                              # :421


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError("dotaclient_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    return torch.device('cuda', torch.cuda.current_device())


def is_distributed():                                                   # :42-43
    return dist.is_available() and dist.is_initialized()


def is_master():                                                        # :46-50
    return dist.get_rank() == 0 if is_distributed() else True


# ------------------------------------------------------------------------------------------ GAE
def advantage_returns(rewards, values, gamma, lam):
    """GAE advantages and rewards-to-go (:57-64) on the GPU scan kernel.

    ``rewards`` / ``values`` carry one trailing bootstrap element like the reference's
    (:417-420, both 0 for terminated rollouts).  numpy in -> numpy out; torch in -> torch (cuda) out.
    """
    as_numpy = isinstance(rewards, np.ndarray)
    dev = _device()
    r = torch.as_tensor(rewards, dtype=torch.float32).to(dev)
    v = torch.as_tensor(values, dtype=torch.float32).to(dev)
    n = r.numel() - 1
    seg = torch.tensor([0, n], dtype=torch.int64, device=dev)
    adv, ret = ops.gae_scan(r[:n], v[:n], seg, gamma=gamma, lam=lam, boot_value=v[n:n + 1].contiguous(),
                            boot_reward=r[n:n + 1].contiguous())
    if as_numpy:
        return adv.cpu().numpy(), ret.cpu().numpy()
    return adv, ret


def discount(x, gamma):
    """Reverse discounted cumulative sum (:53-54), float64 accumulate, fp32 result."""
    as_numpy = isinstance(x, np.ndarray)
    dev = _device()
    xt = torch.as_tensor(x, dtype=torch.float32).to(dev).contiguous()
    seg = torch.tensor([0, xt.numel()], dtype=torch.int64, device=dev)
    _, ret = ops.gae_scan(xt, torch.zeros_like(xt), seg, gamma=gamma, lam=1.0)
    return ret.cpu().numpy() if as_numpy else ret


# ------------------------------------------------------------------------------------------ broker
class _Delivery:
    def __init__(self, tag):
        self.delivery_tag = tag


class _Broker:
    """In-process stand-in for the RabbitMQ broker: one 'experience' queue, one 'model' slot."""
    _registry = {}
    _lock = threading.Lock()

    def __init__(self):
        self.experience = queue.Queue()
        self.model = None            # (body, headers): x-recent-history exchange of length 1 (:118-122)
        self.model_lock = threading.Lock()
        self.tag = 0

    @classmethod
    def get(cls, host, port):
        with cls._lock:
            return cls._registry.setdefault((host, port), _Broker())


class MessageQueue:
    """Same interface as the reference's pika client (:67-174), backed by an in-process broker.

    The real AMQP transport is out of scope (no broker, no pika here); actors running in the same
    process publish with ``publish_experience`` and read weights with ``latest_model``.
    """
    EXPERIENCE_QUEUE_NAME = 'experience'
    MODEL_EXCHANGE_NAME = 'model'
    MAX_RETRIES = 10

    def __init__(self, host, port, prefetch_count, use_model_exchange):
        self.host, self.port = host, port
        self.prefetch_count = prefetch_count
        self.use_model_exchange = use_model_exchange
        self._broker = None

    def connect(self):
        if self._broker is None:
            self._broker = _Broker.get(self.host, self.port)

    @property
    def xp_queue_size(self):
        return self._broker.experience.qsize() if self._broker else None

    def process_events(self):
        pass

    def process_data_events(self):          # heartbeat in the reference (:132-137)
        pass

    def publish_model(self, msg, hdr):
        with self._broker.model_lock:
            self._broker.model = (msg, dict(hdr))

    def consume_xp(self, timeout=None):
        body = self._broker.experience.get(timeout=timeout)
        self._broker.tag += 1
        return _Delivery(self._broker.tag), None, body

    def close(self):
        self._broker = None

    # -- actor side of the in-process broker ------------------------------------------------
    def publish_experience(self, body):
        self._broker.experience.put(body)

    def latest_model(self):
        with self._broker.model_lock:
            return self._broker.model


# ------------------------------------------------------------------------------------------ records
class Sequence:
    """One ``seq_len`` chunk of a rollout (:176-190).

    ``log_probs_sel`` (compact per-head vectors, reference form) is derived lazily from the dense
    ``old_logp [S, 5]`` the kernels produce, so building a Sequence never syncs the device.
    """

    def __init__(self, game_id, weight_version, team_id, observations, actions, masks, values, rewards, hidden,
                 log_probs_sel=None, old_logp=None, valid=None, old_log_probs=None, teacher_log_probs=None):
        self.game_id = game_id
        self.weight_version = weight_version
        self.team_id = team_id
        self.observations = observations
        self.actions = actions
        self.masks = masks
        self.rewards = rewards
        self.values = values
        self.hidden = hidden
        self._log_probs_sel = log_probs_sel
        self.old_logp = old_logp
        self.valid = valid          # [S] bool, real steps vs zero padding (set by prep under DotaOptimizer(mask_padding=True))
        self.old_log_probs = old_log_probs  # [S, 65] prep-time masked log-prob rows (set by prep under KL control)
        self.teacher_log_probs = teacher_log_probs  # [S, 65] the teacher's masked log-prob rows (set by prep with a teacher)
        self.advantages = None
        self.returns = None

    @property
    def log_probs_sel(self):
        if self._log_probs_sel is None and self.old_logp is not None:
            self._log_probs_sel = {}
            for h, key in enumerate(ops.HEAD_KEYS):
                step = self.actions[key].bool().any(dim=-1)
                self._log_probs_sel[key] = self.old_logp[:, h][step]
        return self._log_probs_sel

    def dense_old_logp(self):
        if self.old_logp is None:
            ref = self.actions['enum']
            dense = torch.zeros((ref.shape[0], 5), dtype=torch.float32, device=ref.device)
            for h, key in enumerate(ops.HEAD_KEYS):
                step = self.actions[key].bool().any(dim=-1)
                dense[step, h] = self._log_probs_sel[key].to(ref.device)
            self.old_logp = dense
        return self.old_logp


# Token count of a training batch from which the target-unit head runs on its active tokens only (Policy._head_outputs with
# `active`).  Smaller batches (C1: 64 tokens) are bound by kernel launches, and the row list adds five of them.
TARGET_ROWS_MIN_TOKENS = 4096

class ExperienceBatch:
    """A training batch stacked time-major ``[S, B, ...]`` -- the layout the kernels consume.

    ``DotaOptimizer.train`` accepts either a list of ``Sequence`` (reference API) or one of these.
    Tensors may live in pinned host memory; ``to(device)`` issues the asynchronous H2D copies.
    ``old_values [S, B]`` (optional) are the critic's values at experience prep, which the clipped value loss
    (``DotaOptimizer(value_clip=...)``) needs; a batch without them has no such entry in ``tensors()``.
    ``valid [S, B]`` (optional, bool) marks the real steps against the zero padding of each rollout's last chunk, which
    ``DotaOptimizer(mask_padding=True)`` leaves out of the loss; like ``old_values`` it is absent from ``tensors()`` when None.
    A packed batch (``DotaOptimizer(pack_sequences=True)``, ``pack_layout``) holds several rollout tails in one column and
    carries the recurrent-state resets between them: ``reset_slot [S, B]`` int32 (-1: carry the state; k >= 0: the state
    entering that step is row (k, column) of the tables), ``reset_h [K, B, L*H]`` and, for the LSTM, ``reset_c`` (every
    layer's state side by side).  They are gathered column by column like every other field, and absent when None.
    ``old_log_probs [S, B, 65]`` (optional) are every head's full masked log-prob rows at experience prep, in head order
    with 0 at illegal entries, which the KL penalty and the KL early stop (``DotaOptimizer(kl_coef=..., kl_stop=...)``)
    compare against; absent from ``tensors()`` when None.
    ``teacher_log_probs [S, B, 65]`` (optional) are the same rows of a frozen teacher policy, which the kickstarting term
    (``DotaOptimizer(teacher_model=...)``) compares against; absent from ``tensors()`` when None.
    With ``K > 1`` value heads (``DotaOptimizer(value_heads=...)``) ``returns`` and ``old_values`` are ``[S, B, K]``, one
    column per head; ``advantages`` stay ``[S, B]``, the heads' sum.
    """
    FIELDS = ("advantages", "returns", "old_logp", "h0", "c0", "old_values", "valid", "reset_slot", "reset_h", "reset_c",
              "old_log_probs", "teacher_log_probs")

    def __init__(self, observations, masks, actions, old_logp, advantages, returns, h0, c0=None, old_values=None,
                 valid=None, reset_slot=None, reset_h=None, reset_c=None, old_log_probs=None, teacher_log_probs=None):
        self.observations, self.masks, self.actions = observations, masks, actions
        self.old_logp, self.advantages, self.returns, self.h0, self.c0 = old_logp, advantages, returns, h0, c0
        self.old_values = old_values
        self.old_log_probs = old_log_probs
        self.teacher_log_probs = teacher_log_probs
        self.valid = valid
        self.reset_slot, self.reset_h, self.reset_c = reset_slot, reset_h, reset_c
        self._ready = {}        # data_ptr -> event of an upload still to be waited for (``to`` from pinned memory)
        self._slot = None       # the DotaOptimizer input slot whose static buffers these tensors are (``prefetch``)
        self.refresh = None     # AdvantageRefresh of batch_from_rollouts under recompute_advantages; not copied by map
        self.state_refresh = None   # StateRefresh of batch_from_rollouts under recompute_states; not copied by map

    def map(self, fn):
        """A batch of the same structure with ``fn(tensor)`` in every slot; absent optional fields stay None."""
        def opt(v):
            return None if v is None else fn(v)
        return ExperienceBatch({k: fn(v) for k, v in self.observations.items()}, {k: fn(v) for k, v in self.masks.items()},
                               {k: fn(v) for k, v in self.actions.items()}, **{f: opt(getattr(self, f)) for f in self.FIELDS})

    def graph_key(self):
        """The shape a captured step graph is specialised to (old_values, valid, the reset tables of a packed batch, the
        old and the teacher's log-prob rows: more static inputs)."""
        key = (self.seq_len, self.batch_size, self.old_values is not None)
        key = key if self.valid is None else key + ('valid',)
        key = key if self.reset_slot is None else key + (('reset', self.reset_h.shape[0]),)
        key = key if self.old_log_probs is None else key + ('old_log_probs',)
        return key if self.teacher_log_probs is None else key + ('teacher_log_probs',)

    def reset(self):
        """The ``reset`` operand of ``Policy._recur`` (None for a batch that is not packed)."""
        return None if self.reset_slot is None else (self.reset_slot, self.reset_h, self.reset_c)

    def wait(self, *tensors):
        """Makes the current stream wait for the uploads of ``tensors`` (None allowed) that are still outstanding; each
        upload is waited for once."""
        for t in tensors:
            ev = None if t is None else self._ready.pop(t.data_ptr(), None)
            if ev is not None:
                torch.cuda.current_stream().wait_event(ev)

    @property
    def seq_len(self):
        return self.advantages.shape[0]

    @property
    def batch_size(self):
        return self.advantages.shape[1]

    def tensors(self):
        for d in (self.observations, self.masks, self.actions):
            for k, v in d.items():
                yield d, k, v
        for f in self.FIELDS:
            v = getattr(self, f)
            if v is not None:
                yield self, f, v

    def nbytes(self):
        return sum(v.numel() * v.element_size() for _, _, v in self.tensors())

    def to(self, device, non_blocking=True, prefetch=False):
        """Host -> device.  From pinned memory the copies are issued on a side stream in the order the step consumes
        them (env, states, unit groups, then the loss inputs) and every tensor gets an event, kept by the returned batch:
        ``train`` makes the compute stream wait per tensor (``wait``) right before first use, so the PCIe transfer of unit
        group g+1 overlaps the encoder kernels of group g and the loss inputs arrive during forward/backward."""
        overlap = non_blocking and self.advantages.is_pinned()
        compute = torch.cuda.current_stream(device)
        side = _copy_stream(device) if overlap else None
        if overlap and not prefetch:
            side.wait_stream(compute)            # prefetch=True: the copies start now, next to whatever the compute stream is doing
        def priority(item):                      # copy order == order of first use in the step
            holder, k, _ = item
            if holder is self.observations:
                return 0 if k == 'env' else 3 + Policy.INPUT_KEYS.index(k)
            if not isinstance(holder, dict) and k in ('h0', 'c0', 'reset_slot', 'reset_h', 'reset_c'):
                return 1
            return 100
        moved, ready = {}, {}
        for _, _, v in sorted(self.tensors(), key=priority):
            if overlap:
                with torch.cuda.stream(side):
                    d = v.to(device, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(side)
                d.record_stream(compute)
                ready[d.data_ptr()] = ev
            else:
                d = v.to(device, non_blocking=non_blocking)
            moved[id(v)] = d
        out = self.map(lambda v: moved[id(v)])
        out._ready = ready
        return out

    def pin_memory(self):
        return self.map(lambda v: v.cpu().pin_memory())

    def gather(self, index):
        """A new device batch of the sequence columns ``index`` (host integers, in that order; repeats allowed) of every
        tensor, ``h0`` / ``c0`` included: ``index_select(1, index)`` of each, done by ONE ``dc_gather_columns`` launch.
        Each sequence carries its own initial recurrent state, so the result is an exact batch of those sequences."""
        n = len(index)
        out = self.map(lambda v: torch.empty((v.shape[0], n) + tuple(v.shape[2:]), dtype=v.dtype, device=v.device))
        srcs = [v for _, _, v in self.tensors()]
        if self._slot is not None:               # uploaded by prefetch() into graph input buffers: wait for that upload
            torch.cuda.current_stream().wait_event(self._slot["ready"])
        self.wait(*srcs)
        ops.gather_columns(list(zip(srcs, [v for _, _, v in out.tensors()])), index)
        return out

    @staticmethod
    def from_sequences(experiences, device):
        """Stacks ``Sequence`` records along dim 1 (the reference stacks along dim 0, :587-615)."""
        def stack(ts):
            return torch.stack([t.to(device) for t in ts], dim=1)
        obs = {k: stack([e.observations[k] for e in experiences]) for k in Policy.INPUT_KEYS}
        masks = {k: stack([e.masks[k] for e in experiences]) for k in Policy.OUTPUT_KEYS}
        actions = {k: stack([e.actions[k] for e in experiences]) for k in Policy.OUTPUT_KEYS}
        old = stack([e.dense_old_logp() for e in experiences])
        adv = stack([torch.as_tensor(e.advantages) for e in experiences])
        ret = stack([torch.as_tensor(e.returns) for e in experiences])
        if isinstance(experiences[0].hidden, tuple):
            h0 = torch.cat([e.hidden[0].to(device) for e in experiences], dim=1)
            c0 = torch.cat([e.hidden[1].to(device) for e in experiences], dim=1)
        else:
            h0, c0 = torch.cat([e.hidden.to(device) for e in experiences], dim=1), None      # :591
        old_values = None
        if all(e.values is not None for e in experiences):
            def rows(v):                        # [1, S, 1] -> [S]; [1, S, K] (value heads) -> [S, K]
                v = torch.as_tensor(v).detach().float()
                return v.reshape(-1) if v.dim() == 1 or v.shape[-1] == 1 else v.reshape(-1, v.shape[-1])
            old_values = stack([rows(e.values) for e in experiences])
        valid = None
        if all(getattr(e, 'valid', None) is not None for e in experiences):
            valid = stack([torch.as_tensor(e.valid).reshape(-1).bool() for e in experiences])
        old_log_probs = None
        if all(getattr(e, 'old_log_probs', None) is not None for e in experiences):
            old_log_probs = stack([torch.as_tensor(e.old_log_probs).float() for e in experiences])
        teacher_log_probs = None
        if all(getattr(e, 'teacher_log_probs', None) is not None for e in experiences):
            teacher_log_probs = stack([torch.as_tensor(e.teacher_log_probs).float() for e in experiences])
        return ExperienceBatch(obs, masks, actions, old, adv, ret, h0.detach(), None if c0 is None else c0.detach(),
                               old_values=old_values, valid=valid, old_log_probs=old_log_probs,
                               teacher_log_probs=teacher_log_probs)


class AdvantageRefresh(typing.NamedTuple):
    """What the advantage refresh between PPO epochs (``DotaOptimizer(recompute_advantages=True)``) needs beyond the batch,
    as experience prep had it (device tensors, rows rollout-major): ``rewards [n_rows, 10]``, the scan segments
    ``seg_off [n_seg + 1]`` (``rollout_segments``), the per-segment bootstraps ``boot [n_seg]`` (None: all 0), ``tok
    [n_rows]`` (``refresh_token_map``) and, for V-trace, the behaviour log-probs ``behaviour_logp [n_rows, 5]`` and
    ``valid_len [n_seg]``.  ``batch_from_rollouts`` sets it as ``ExperienceBatch.refresh``, a plain attribute outside
    ``FIELDS``: ``map``, ``gather``, ``to`` and the graph input slots do not carry it."""
    rewards: torch.Tensor
    seg_off: torch.Tensor
    boot: typing.Optional[torch.Tensor]
    tok: typing.Optional[torch.Tensor]
    behaviour_logp: typing.Optional[torch.Tensor]
    valid_len: typing.Optional[torch.Tensor]


class StateRefreshLayout(typing.NamedTuple):
    """Where the state refresh (``DotaOptimizer(recompute_states=True)``) finds its inputs and puts its states, for rollouts
    whose forward runs time-major over ``[L_max, R]`` (row ``t * R + i``: step t of rollout i) and a ``[S, B]`` training
    batch (token ``t * B + c``), from ``state_refresh_layout`` (host int64 arrays):
    ``obs_token [L_max * R]`` the batch token holding row r's observation, or -1 where the batch holds none (the row is fed
    zeros, as experience prep pads); ``token_row [S * B]`` the row each token holds, or -1 (padding of a packed column);
    ``step``, ``rollout``, ``slot`` ``[n]``, sorted by step: the state entering ``step`` (a multiple of ``seq_len``, >= 1) of
    ``rollout`` is written to ``h0[:, slot]`` for ``slot < B`` or to row ``slot - B = k * B + c`` of the reset tables."""
    R: int
    L_max: int
    obs_token: np.ndarray
    token_row: np.ndarray
    step: np.ndarray
    rollout: np.ndarray
    slot: np.ndarray


class StateRefresh(typing.NamedTuple):
    """What the state refresh between PPO epochs (``DotaOptimizer(recompute_states=True)``) needs beyond the batch: the
    ``layout`` (host ``StateRefreshLayout``) and its index arrays on the device (``obs_token``, ``token_row``, ``step``,
    ``rollout``, ``slot``); prep's start states ``h0`` / ``c0 [L, R, H]`` (None: all zero); and, with
    ``recompute_advantages``, the cut rollouts' extra observation rows ``obs_next`` (``[1, R', ...]`` per input key), their
    lengths ``cut_len`` and columns ``cut_rollout`` (host int64 ``[R']``) and prep's bootstrap slot map ``boot_slot [n_seg]``
    (None when no rollout is cut).  ``batch_from_rollouts`` sets it as ``ExperienceBatch.state_refresh``, a plain attribute
    outside ``FIELDS``: ``map``, ``gather``, ``to`` and the graph input slots do not carry it."""
    layout: StateRefreshLayout
    obs_token: torch.Tensor
    token_row: torch.Tensor
    step: torch.Tensor
    rollout: torch.Tensor
    slot: torch.Tensor
    h0: typing.Optional[torch.Tensor]
    c0: typing.Optional[torch.Tensor]
    obs_next: typing.Optional[dict]
    cut_len: typing.Optional[np.ndarray]
    cut_rollout: typing.Optional[np.ndarray]
    boot_slot: typing.Optional[torch.Tensor]


class _CapturedStep(typing.NamedTuple):
    """A CUDA graph of the whole step, its static input batch and its device result vector (loss slots)."""
    static: ExperienceBatch
    graph: torch.cuda.CUDAGraph
    out: torch.Tensor


_copy_streams = {}


def _copy_stream(device):
    key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    if key not in _copy_streams:
        _copy_streams[key] = torch.cuda.Stream(device=device)
    return _copy_streams[key]


def all_gather(t):                                                        # :193-196 (unused by the reference too)
    out = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t)
    return torch.cat(out)


# ------------------------------------------------------------------------------------------ optimizer
ADVANTAGE_ESTIMATORS = ('gae', 'vtrace')
# 'per_head': the reference's objective, one clipped ratio per action head; 'joint': one clipped ratio per step, of the
# whole hierarchical action (the product of the sampled heads' probabilities)
POLICY_RATIOS = ('per_head', 'joint')
# 'ppo': the reference's objective, the clipped surrogate on the batch's advantages; 'bc': behaviour cloning, every rollout
# is a demonstration and the policy term is the negative log-likelihood of its actions (supervised pretraining)
OBJECTIVES = ('ppo', 'bc')
# the heads Policy.select_actions samples after each enum value (0 none, 1 move, 2 attack, 3 ability)
ENUM_FOLLOWS = {0: (), 1: ('x', 'y'), 2: ('target_unit',), 3: ('ability',)}


def check_ppo_settings(gamma, gae_lambda, clip_range, max_grad_norm, value_clip=None, *, advantage_estimator='gae',
                       vtrace_rho_clip=1.0, vtrace_c_clip=1.0, num_minibatches=1, mask_padding=False, pack_sequences=False,
                       policy_ratio='per_head', value_norm=False, value_norm_decay=0.99, kl_coef=0.0, kl_target=None,
                       kl_stop=None, recompute_advantages=False, recompute_states=False, value_heads=None,
                       value_gammas=None, teacher_model=None, teacher_coef=1.0, teacher_anneal_iterations=None,
                       upgo_coef=0.0, objective='ppo', dual_clip=None):
    """Raises ``ValueError`` for PPO settings outside their domain: 0 < gamma <= 1, 0 <= gae_lambda <= 1, clip_range > 0,
    max_grad_norm > 0, value_clip None (off) or >= 0 (0 is off too), advantage_estimator one of ``ADVANTAGE_ESTIMATORS``,
    vtrace_rho_clip > 0, vtrace_c_clip > 0, num_minibatches an int >= 1 (not a bool), mask_padding a bool,
    pack_sequences a bool that is True only with mask_padding, policy_ratio one of ``POLICY_RATIOS``, value_norm a bool
    and 0 <= value_norm_decay < 1, finite kl_coef >= 0, kl_target None or finite > 0 (and then kl_coef > 0), kl_stop None
    or finite > 0, recompute_advantages and recompute_states bools, value_heads / value_gammas as ``value_head_groups``
    checks them (value heads refuse V-trace and value_norm), finite teacher_coef >= 0 and teacher_anneal_iterations None
    or an int >= 1, both left at their defaults without a teacher_model, upgo_coef as ``check_upgo_coef`` checks it,
    objective one of ``OBJECTIVES`` and dual_clip as ``check_dual_clip`` checks it; 'bc' refuses what acts only on the
    policy-gradient term or needs a behaviour policy (V-trace, the joint ratio, KL control, a teacher, UPGO, dual clip).
    NaN fails every check."""
    if not isinstance(recompute_states, bool):
        raise ValueError("recompute_states=%r: must be True or False" % (recompute_states,))
    if not isinstance(recompute_advantages, bool):
        raise ValueError("recompute_advantages=%r: must be True or False" % (recompute_advantages,))
    if not isinstance(value_norm, bool):
        raise ValueError("value_norm=%r: must be True or False" % (value_norm,))
    if isinstance(value_norm_decay, bool) or not isinstance(value_norm_decay, numbers.Real) \
            or not 0.0 <= float(value_norm_decay) < 1.0:
        raise ValueError("value_norm_decay=%r: the decay of the value statistics must be in [0, 1)" % (value_norm_decay,))
    if not isinstance(policy_ratio, str) or policy_ratio not in POLICY_RATIOS:
        raise ValueError("policy_ratio=%r: must be one of %s" % (policy_ratio, ", ".join(POLICY_RATIOS)))
    if not isinstance(mask_padding, bool):
        raise ValueError("mask_padding=%r: must be True or False" % (mask_padding,))
    if not isinstance(pack_sequences, bool):
        raise ValueError("pack_sequences=%r: must be True or False" % (pack_sequences,))
    if pack_sequences and not mask_padding:
        raise ValueError("pack_sequences=True needs mask_padding=True: without the mask, experience prep gives padded steps "
                         "advantages and value targets that packing would drop")
    if isinstance(num_minibatches, bool) or not isinstance(num_minibatches, numbers.Integral) or num_minibatches < 1:
        raise ValueError("num_minibatches=%r: the number of minibatches per epoch must be an int >= 1" % (num_minibatches,))
    def number(name, v):
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise ValueError("%s=%r is not a number" % (name, v))
        return float(v)
    if not 0.0 < number('gamma', gamma) <= 1.0:
        raise ValueError("gamma=%r: the discount factor must be in (0, 1]" % (gamma,))
    if not 0.0 <= number('gae_lambda', gae_lambda) <= 1.0:
        raise ValueError("gae_lambda=%r: the GAE lambda must be in [0, 1]" % (gae_lambda,))
    if not number('clip_range', clip_range) > 0.0:
        raise ValueError("clip_range=%r: the PPO clip range must be > 0" % (clip_range,))
    if not number('max_grad_norm', max_grad_norm) > 0.0:
        raise ValueError("max_grad_norm=%r: the gradient-norm limit must be > 0" % (max_grad_norm,))
    if value_clip is not None and not number('value_clip', value_clip) >= 0.0:
        raise ValueError("value_clip=%r: the value clip range must be >= 0 (or None: no value clipping)" % (value_clip,))
    if advantage_estimator not in ADVANTAGE_ESTIMATORS:
        raise ValueError("advantage_estimator=%r: must be one of %s" % (advantage_estimator, ", ".join(ADVANTAGE_ESTIMATORS)))
    if not number('vtrace_rho_clip', vtrace_rho_clip) > 0.0:
        raise ValueError("vtrace_rho_clip=%r: the V-trace rho truncation must be > 0" % (vtrace_rho_clip,))
    if not number('vtrace_c_clip', vtrace_c_clip) > 0.0:
        raise ValueError("vtrace_c_clip=%r: the V-trace c truncation must be > 0" % (vtrace_c_clip,))
    if not 0.0 <= number('kl_coef', kl_coef) < math.inf:
        raise ValueError("kl_coef=%r: the KL penalty coefficient must be finite and >= 0" % (kl_coef,))
    if kl_target is not None:
        if not 0.0 < number('kl_target', kl_target) < math.inf:
            raise ValueError("kl_target=%r: the KL target must be finite and > 0 (or None: a fixed kl_coef)" % (kl_target,))
        if not float(kl_coef) > 0.0:
            raise ValueError("kl_target=%r needs kl_coef > 0: the adaptive coefficient starts from kl_coef and only "
                             "doubles or halves it" % (kl_target,))
    if kl_stop is not None and not 0.0 < number('kl_stop', kl_stop) < math.inf:
        raise ValueError("kl_stop=%r: the KL limit must be finite and > 0 (or None: no early stop)" % (kl_stop,))
    if not 0.0 <= number('teacher_coef', teacher_coef) < math.inf:
        raise ValueError("teacher_coef=%r: the teacher coefficient must be finite and >= 0" % (teacher_coef,))
    if teacher_anneal_iterations is not None and (isinstance(teacher_anneal_iterations, bool)
                                                  or not isinstance(teacher_anneal_iterations, numbers.Integral)
                                                  or teacher_anneal_iterations < 1):
        raise ValueError("teacher_anneal_iterations=%r: the anneal length must be an int >= 1 (or None: a fixed "
                         "teacher_coef)" % (teacher_anneal_iterations,))
    if teacher_model is None and float(teacher_coef) != 1.0:
        raise ValueError("teacher_coef=%r needs teacher_model" % (teacher_coef,))
    if teacher_model is None and teacher_anneal_iterations is not None:
        raise ValueError("teacher_anneal_iterations=%r needs teacher_model" % (teacher_anneal_iterations,))
    value_head_groups(value_heads, value_gammas, gamma)
    if value_heads is not None and advantage_estimator == 'vtrace':
        raise ValueError("value_heads with advantage_estimator='vtrace': per-head V-trace targets are not defined yet "
                         "(the importance weights would need a per-head definition); use 'gae'")
    if value_heads is not None and value_norm:
        raise ValueError("value_heads with value_norm=True: PopArt would need one set of statistics per head and a "
                         "per-row rescale of the value head, which is not implemented")
    check_upgo_coef(upgo_coef, value_heads)
    check_dual_clip(dual_clip)
    if not isinstance(objective, str) or objective not in OBJECTIVES:
        raise ValueError("objective=%r: must be one of %s" % (objective, ", ".join(OBJECTIVES)))
    if objective == 'bc':
        refused = [("advantage_estimator='vtrace'", advantage_estimator == 'vtrace',
                    "V-trace corrects for a behaviour policy, and a demonstration has none"),
                   ("policy_ratio='joint'", policy_ratio == 'joint', "there is no PPO ratio to clip"),
                   ("kl_coef=%r" % (kl_coef,), float(kl_coef) > 0.0, "there is no prep-time policy to stay close to"),
                   ("kl_target=%r" % (kl_target,), kl_target is not None, "there is no KL penalty to adapt"),
                   ("kl_stop=%r" % (kl_stop,), kl_stop is not None, "there is no prep-time policy to stop at"),
                   ("teacher_model=%r" % (teacher_model,), teacher_model is not None,
                    "the demonstrations are the teacher; run the teacher term with objective='ppo'"),
                   ("upgo_coef=%r" % (upgo_coef,), float(upgo_coef) > 0.0, "UPGO changes the advantages, which the "
                    "behaviour-cloning loss does not read"),
                   ("dual_clip=%r" % (dual_clip,), dual_clip is not None, "there is no PPO surrogate to bound")]
        for what, bad, why in refused:
            if bad:
                raise ValueError("%s with objective='bc': %s" % (what, why))


def check_dual_clip(dual_clip):
    """Raises ``ValueError`` unless ``dual_clip`` is None (off) or a finite number c > 1 (not a bool): the floor c A under
    the surrogate of a negative-advantage row must lie below the clipped surrogate's own (1 + clip_range) A at r = 1."""
    if dual_clip is None:
        return
    if isinstance(dual_clip, bool) or not isinstance(dual_clip, numbers.Real) or not 1.0 < float(dual_clip) < math.inf:
        raise ValueError("dual_clip=%r: the dual-clip constant must be a finite number > 1 (or None: off)" % (dual_clip,))


def check_upgo_coef(upgo_coef, value_heads=None):
    """Raises ``ValueError`` unless ``upgo_coef`` is a finite number >= 0 (not a bool), and 0 with ``value_heads``: the
    UPGO switch compares one return with one critic value, and heads with different discounts have no single return."""
    if isinstance(upgo_coef, bool) or not isinstance(upgo_coef, numbers.Real) or not 0.0 <= float(upgo_coef) < math.inf:
        raise ValueError("upgo_coef=%r: the UPGO coefficient must be a finite number >= 0" % (upgo_coef,))
    if float(upgo_coef) > 0.0 and value_heads is not None:
        raise ValueError("upgo_coef=%r with value_heads: UPGO compares one return with one critic value, and value heads "
                         "with different discounts have no single return" % (upgo_coef,))


class ValueHeads(typing.NamedTuple):
    """The value heads of ``DotaOptimizer(value_heads=...)``: ``names`` in head order, ``keys`` the ``REWARD_KEYS`` of each,
    ``group`` (int32 [10]) the head of every reward column, ``gammas`` (float64 [K]) their discounts."""
    names: tuple
    keys: tuple
    group: np.ndarray
    gammas: np.ndarray


def value_head_groups(value_heads, value_gammas, gamma):
    """Checks ``value_heads`` (None, or an ordered mapping ``{name: [reward keys]}`` of K >= 1 groups that together hold
    every key of ``REWARD_KEYS`` exactly once, names matching ``[A-Za-z0-9_]+``) and ``value_gammas`` (None, or a mapping
    of some of the names to a discount in (0, 1]; the others take ``gamma``).  Returns None for None, else ``ValueHeads``.
    Raises ``ValueError``."""
    if value_heads is None:
        if value_gammas is not None:
            raise ValueError("value_gammas=%r needs value_heads" % (value_gammas,))
        return None
    if not isinstance(value_heads, collections.abc.Mapping) or not value_heads:
        raise ValueError("value_heads=%r: must be a non-empty mapping {name: [reward keys]}" % (value_heads,))
    names, keys, group = [], [], np.full(len(REWARD_KEYS), -1, dtype=np.int32)
    for name, ks in value_heads.items():
        if not isinstance(name, str) or not re.fullmatch(r'[A-Za-z0-9_]+', name):
            raise ValueError("value head name %r: names must be non-empty and match [A-Za-z0-9_]+" % (name,))
        if isinstance(ks, str) or not isinstance(ks, collections.abc.Iterable):
            raise ValueError("value head %r: its reward keys must be a list, got %r" % (name, ks))
        ks = list(ks)
        if not ks:
            raise ValueError("value head %r has no reward keys" % name)
        for k in ks:
            if k not in REWARD_KEYS:
                raise ValueError("value head %r: %r is not a reward key (%s)" % (name, k, ", ".join(REWARD_KEYS)))
            i = REWARD_KEYS.index(k)
            if group[i] >= 0:
                raise ValueError("reward key %r is in more than one value head group" % k)
            group[i] = len(names)
        names.append(name)
        keys.append(tuple(ks))
    missing = [REWARD_KEYS[i] for i in np.flatnonzero(group < 0)]
    if missing:
        raise ValueError("value_heads leaves the reward keys %s out: every key must be in exactly one group, so that the "
                         "summed reward does not change" % ", ".join(missing))
    gammas = np.full(len(names), float(gamma), dtype=np.float64)
    if value_gammas is not None:
        if not isinstance(value_gammas, collections.abc.Mapping):
            raise ValueError("value_gammas=%r: must be a mapping {head name: discount}" % (value_gammas,))
        for name, g in value_gammas.items():
            if name not in names:
                raise ValueError("value_gammas names %r, which is not a value head (%s)" % (name, ", ".join(names)))
            if isinstance(g, bool) or not isinstance(g, numbers.Real) or not 0.0 < float(g) <= 1.0:
                raise ValueError("value_gammas[%r]=%r: the discount must be in (0, 1]" % (name, g))
            gammas[names.index(name)] = float(g)
    return ValueHeads(tuple(names), tuple(keys), group, gammas)


def parse_value_heads(text):
    """``--value-heads``: ``'name=key,key;name=key,...'`` -> ``{name: [keys]}`` in the order given (checked later by
    ``value_head_groups``)."""
    out = {}
    for part in text.split(';'):
        name, sep, keys = part.partition('=')
        name = name.strip()
        if not sep or name in out:
            raise ValueError("--value-heads %r: expected 'name=key,key;name=key', each name once" % text)
        out[name] = [k.strip() for k in keys.split(',') if k.strip()]
    return out


def parse_value_gammas(text):
    """``--value-gammas``: ``'name=0.999;name=0.9'`` -> ``{name: float}``."""
    out = {}
    for part in text.split(';'):
        name, sep, g = part.partition('=')
        if not sep or name.strip() in out:
            raise ValueError("--value-gammas %r: expected 'name=discount;name=discount', each name once" % text)
        out[name.strip()] = float(g)
    return out


def _drift(sq_change, sq_old):
    """sqrt(sum (new - old)^2 / sum old^2) from the two sums of ``dc_refresh_states``; 0 when nothing moved."""
    if sq_old > 0:
        return math.sqrt(sq_change / sq_old)
    return 0.0 if sq_change == 0 else math.inf


def kl_coef_update(kl_coef, kl, kl_target):
    """The adaptive KL coefficient after an iteration whose steps measured a mean KL of ``kl`` (Schulman et al. 2017,
    section 4): doubled when kl > 1.5 kl_target, halved when kl < kl_target / 1.5, unchanged otherwise (the boundaries
    included)."""
    if kl > 1.5 * kl_target:
        return kl_coef * 2.0
    if kl < kl_target / 1.5:
        return kl_coef / 2.0
    return kl_coef


def value_norm_moments(state, min_std):
    """(mu, sigma) of the value statistics ``state = (m, q, w)`` (float64 EMAs of the target mean and mean square, and
    their debias weight): (0, 1) while w = 0, else mu = m / w and sigma = max(sqrt(max(q / w - mu^2, 0)), min_std)."""
    m, q, w = state
    if w == 0.0:
        return 0.0, 1.0
    mu = m / w
    return mu, max(math.sqrt(max(q / w - mu * mu, 0.0)), min_std)


def value_norm_update(state, n, s1, s2, decay):
    """The value statistics after one batch of ``n`` targets with sum ``s1`` and sum of squares ``s2`` (float64):
    m <- d m + (1 - d) s1 / n, q <- d q + (1 - d) s2 / n, w <- d w + (1 - d).  ``n`` = 0 leaves ``state`` as it is."""
    if n <= 0:
        return state
    m, q, w = state
    d = float(decay)
    return d * m + (1.0 - d) * (s1 / n), d * q + (1.0 - d) * (s2 / n), d * w + (1.0 - d)


def load_teacher(path):
    """The frozen teacher ``Policy`` of ``DotaOptimizer(teacher_model=path)``, on the CPU without gradients: the ``state_dict``
    file at ``path`` loaded strictly into the architecture it describes (``Policy.from_state_dict``), whose width must be
    one the kernels run, a multiple of 32.  Raises ``ValueError`` for a missing file or a file that is not a ``Policy``
    state_dict."""
    if not os.path.isfile(path):
        raise ValueError("teacher_model=%r: no such file" % (path,))
    state = torch.load(path, map_location='cpu')
    if not isinstance(state, dict):
        raise ValueError("teacher_model=%r does not hold a state_dict" % (path,))
    try:
        teacher = Policy.from_state_dict(state)
    except ValueError as e:
        raise ValueError("teacher_model=%r: %s" % (path, e)) from None
    if teacher.hidden_size % 32:
        raise ValueError("teacher_model=%r has hidden_size %d; the kernels run multiples of 32"
                         % (path, teacher.hidden_size))
    teacher.requires_grad_(False)
    logger.info('Teacher %s: %s-%d, %d layer(s)', path, teacher.cell, teacher.hidden_size, teacher.num_layers)
    return teacher


def check_minibatch_count(num_minibatches, min_seq_per_epoch):
    """Raises ``ValueError`` when an iteration could hold fewer sequences than minibatches.  An iteration holds at least
    ``min_seq_per_epoch`` sequences on every rank, so with ``num_minibatches <= min_seq_per_epoch`` every rank forms all its
    minibatches and the ranks' all-reduces stay in lockstep, whatever their batch sizes."""
    if num_minibatches > min_seq_per_epoch:
        raise ValueError("num_minibatches=%r exceeds min_seq_per_epoch=%r: every minibatch needs at least one sequence"
                         % (num_minibatches, min_seq_per_epoch))


def minibatch_indices(B, num_minibatches, rng):
    """The sequence columns of each minibatch of one epoch over a batch of ``B`` sequences: with one minibatch the whole
    batch in order (``rng`` is not drawn from), otherwise ``np.array_split`` of a permutation drawn from ``rng`` (a numpy
    ``Generator``), so the sizes differ by at most one and every sequence is used exactly once per epoch."""
    if num_minibatches == 1:
        return [np.arange(B)]
    return np.array_split(rng.permutation(B), num_minibatches)


def rollout_segments(lengths, terminal, seq_len, mask_padding):
    """The scan segments of experience prep.  Rollout i occupies its padded length ``Lp_i`` (``lengths[i]`` rounded up to a
    multiple of ``seq_len``) of the rollout-major rows.  A terminal rollout without ``mask_padding`` is one segment of
    ``Lp_i`` rows ending on the terminal bootstrap of 0 (the reference's layout).  Otherwise it is two: its ``lengths[i]``
    real rows, then its ``Lp_i - lengths[i]`` padding rows (possibly none), which end on 0.  The real segment of a rollout
    that is not ``terminal[i]`` ends on the bootstrap value of the state its game continues from; that of a terminal one on 0.

    Returns int64 arrays ``(seg_off [n_seg + 1], boot [n_seg], valid_len [n_seg])``: ``boot[s]`` is the index, among the
    non-terminal rollouts in order, of the one whose bootstrap value ends segment ``s``, or -1 for 0; ``valid_len[s]`` is
    the number of real steps in segment ``s``."""
    off, boot, valid = [0], [], []
    base = n_cut = 0
    for L, term in zip(lengths, terminal):
        L = int(L)
        Lp = (L + seq_len - 1) // seq_len * seq_len
        if term and not mask_padding:
            off.append(base + Lp)
            boot.append(-1)
            valid.append(L)
        else:
            off += [base + L, base + Lp]
            boot += [-1 if term else n_cut, -1]
            valid += [L, 0]
        n_cut += not term
        base += Lp
    return np.array(off, dtype=np.int64), np.array(boot, dtype=np.int64), np.array(valid, dtype=np.int64)


def padded_segment_offsets(lengths, seq_len):
    """Row offsets of the scan segments of experience prep under ``mask_padding`` for terminal rollouts
    (``rollout_segments``): a real segment of ``lengths[i]`` rows and a padding segment, so that the real segment ends on
    the terminal bootstrap of 0.  Returns int64 ``[2R + 1]``: ``0, L_0, Lp_0, Lp_0 + L_1, Lp_0 + Lp_1, ...``."""
    return rollout_segments(lengths, [True] * len(lengths), seq_len, True)[0]


def chunk_valid_lengths(lengths, seq_len):
    """The real steps of every ``seq_len`` chunk, rollout by rollout and chunk by chunk (the batch's sequence order): chunk
    j of a rollout of length L has ``min(seq_len, L - j * seq_len)``."""
    return [min(seq_len, int(L) - j * seq_len) for L in lengths for j in range((int(L) + seq_len - 1) // seq_len)]


class PackLayout(typing.NamedTuple):
    """The packed training batch of ``pack_layout``: ``B`` columns of ``seq_len`` steps.  For every token (t, c):
    ``rollout[t, c]`` / ``step[t, c]`` the rollout and its step that the token holds (-1 / -1 for padding), ``reset_slot[t, c]``
    (int32) -1, or k >= 0 where a tail starts after others in its column (its k-th such tail: row k of the column's reset
    tables, the state at ``step[t, c]``).  ``h0_rollout[c]`` / ``h0_step[c]``: the state entering column c, state-buffer slot
    ``h0_step[c]`` of that rollout.  ``K``: the largest number of such mid-column tails in a column.  ``n_full``: the
    columns 0 .. n_full - 1 hold the full chunks, rollout by rollout, chunk by chunk."""
    B: int
    K: int
    n_full: int
    rollout: np.ndarray
    step: np.ndarray
    reset_slot: np.ndarray
    h0_rollout: np.ndarray
    h0_step: np.ndarray


def _first_fit_decreasing(tails, seq_len):
    """Column (0, 1, ...) and offset of every tail ``(length, rollout)`` of ``tails``, placed in the order
    first-fit-decreasing by length, ties by rollout order, each whole into the first column with room for it."""
    order = sorted(range(len(tails)), key=lambda j: (-tails[j][0], tails[j][1]))
    free = np.empty(len(tails), dtype=np.int64)
    n_col = 0
    col, off = [0] * len(tails), [0] * len(tails)
    for j in order:
        r = tails[j][0]
        fits = np.flatnonzero(free[:n_col] >= r)
        c = int(fits[0]) if fits.size else n_col
        if c == n_col:
            free[c] = seq_len
            n_col += 1
        col[j], off[j] = c, seq_len - int(free[c])
        free[c] -= r
    return col, off, n_col


def pack_layout(lengths, seq_len):
    """The packed layout of rollouts of ``lengths`` real steps (``DotaOptimizer(pack_sequences=True)``).  A rollout of L
    steps has ``L // seq_len`` full chunks, which keep one column each and start from the state at their first step, as in
    the unpacked batch, and a tail of ``L % seq_len`` steps (none when 0).  The tails are packed whole into shared columns
    of ``seq_len`` steps, first-fit-decreasing by length with ties broken by rollout order, so the layout depends on the
    lengths alone.  The first tail of a column starts from the column's initial state; every later one from a reset to the
    state at its own first step.  So each tail starts from the same state and ends at the same truncation point as in the
    unpacked batch.  The unused end of a tail column is padding.  Returns a ``PackLayout``."""
    S = int(seq_len)
    Ls = [int(L) for L in lengths]
    segs = [[(i, j * S, S)] for i, L in enumerate(Ls) for j in range(L // S)]            # (rollout, first step, steps)
    n_full = len(segs)
    tails = [(L % S, i) for i, L in enumerate(Ls) if L % S]
    col, off, n_col = _first_fit_decreasing(tails, S)
    tail_cols = [[] for _ in range(n_col)]
    for (r, i), c, o in sorted(zip(tails, col, off), key=lambda x: (x[1], x[2])):
        tail_cols[c].append((i, Ls[i] - r, r))
    segs += tail_cols
    B = len(segs)
    rollout = np.full((S, B), -1, dtype=np.int64)
    step = np.full((S, B), -1, dtype=np.int64)
    reset_slot = np.full((S, B), -1, dtype=np.int32)
    h0_rollout = np.empty(B, dtype=np.int64)
    h0_step = np.empty(B, dtype=np.int64)
    K = 0
    for c, col_segs in enumerate(segs):
        h0_rollout[c], h0_step[c] = col_segs[0][0], col_segs[0][1]
        t = 0
        for k, (i, first, n) in enumerate(col_segs):
            rollout[t:t + n, c] = i
            step[t:t + n, c] = np.arange(first, first + n)
            if k:
                reset_slot[t, c] = k - 1
            t += n
        K = max(K, len(col_segs) - 1)
    return PackLayout(B, K, n_full, rollout, step, reset_slot, h0_rollout, h0_step)


def chunk_columns(t, Lps, seq_len, whole=False):
    """The unpacked batch layout: a time-major ``[L_max, R, ...]`` tensor -> ``[seq_len, sum(Lp_i / seq_len), ...]``, rollout
    i's ``Lps[i]`` padded rows cut into ``seq_len`` chunks of one column each, rollout by rollout, chunk by chunk.
    ``whole``: every rollout is exactly one chunk, and ``t`` is returned as it is."""
    if whole:
        return t
    S = int(seq_len)
    parts = [t[:Lps[i], i].reshape((Lps[i] // S, S) + tuple(t.shape[2:])).transpose(0, 1) for i in range(len(Lps))]
    return torch.cat(parts, dim=1)


def packed_rows(lay, Lps):
    """The rollout-major row of experience prep (rollout i's padded rows follow rollouts 0 .. i-1's) that every token of
    the packed layout ``lay`` holds: int64 ``[S, B]``, -1 at padding tokens."""
    base = np.concatenate([[0], np.cumsum(Lps)[:-1]]).astype(np.int64)
    return np.where(lay.rollout >= 0, base[np.maximum(lay.rollout, 0)] + lay.step, -1)


def _batch_rows(Ls, S, pack, layout=None):
    """The rollout-major row of experience prep (rollout i's ``Lp_i`` padded rows follow rollouts 0 .. i-1's) that every
    token of the ``[S, B]`` batch of ``batch_from_rollouts`` holds, -1 at padding tokens of a packed batch: ``packed_rows``
    of the pack layout, or ``chunk_columns`` applied to the row numbers."""
    Lps = [(L + S - 1) // S * S for L in Ls]
    if pack:
        return packed_rows(pack_layout(Ls, S) if layout is None else layout, Lps)
    base = np.concatenate([[0], np.cumsum(Lps)[:-1]]).astype(np.int64)
    Lmax = max(Lps, default=0)
    t = np.arange(Lmax, dtype=np.int64)[:, None]
    grid = torch.from_numpy(np.where(t < np.asarray(Lps)[None, :], base[None, :] + t, -1))
    return chunk_columns(grid, Lps, S).numpy().reshape(S, -1) if Lps else np.zeros((S, 0), dtype=np.int64)


def state_refresh_layout(lengths, seq_len, pack, layout=None):
    """The ``StateRefreshLayout`` of the batch that ``batch_from_rollouts`` builds from rollouts of ``lengths`` real steps
    (``pack``: the packed batch; ``layout`` its ``pack_layout`` when the caller has it), derived from the batch's own layout
    (``chunk_columns`` / ``packed_rows``).  A batch column starts at the row its first token holds, and a packed reset at
    the row of its token; a start at step 0 keeps prep's state (it is data, not a product of the network) and is not a
    destination.  Checked with ``check_state_refresh_layout``."""
    S = int(seq_len)
    Ls = [int(L) for L in lengths]
    Lps = [(L + S - 1) // S * S for L in Ls]
    R, Lmax = len(Ls), max(Lps, default=0)
    if pack and layout is None:
        layout = pack_layout(Ls, S)
    rows = _batch_rows(Ls, S, pack, layout)                              # [S, B] rollout-major rows
    B = rows.shape[1]
    base = np.concatenate([[0], np.cumsum(Lps)[:-1]]).astype(np.int64)
    row_rollout = np.repeat(np.arange(R, dtype=np.int64), Lps)
    row_step = np.arange(int(sum(Lps)), dtype=np.int64) - np.repeat(base, Lps)
    held = rows >= 0
    r = np.where(held, rows, 0)
    tm = np.where(held, row_step[r] * R + row_rollout[r], -1)            # [S, B] rows of the [L_max, R] forward
    token_row = tm.reshape(-1).astype(np.int64)
    obs_token = np.full(Lmax * R, -1, dtype=np.int64)
    obs_token[token_row[token_row >= 0]] = np.flatnonzero(token_row >= 0)
    dst_rows, dst_slot = [rows[0]], [np.arange(B, dtype=np.int64)]      # every column's initial state
    if pack:                                                             # every reset inside a column
        t_rs, c_rs = np.nonzero(layout.reset_slot >= 0)
        dst_rows.append(rows[t_rs, c_rs])
        dst_slot.append(B + layout.reset_slot[t_rs, c_rs].astype(np.int64) * B + c_rs)
    dst_rows, dst_slot = np.concatenate(dst_rows), np.concatenate(dst_slot)
    step, rollout = row_step[dst_rows], row_rollout[dst_rows]
    keep = step > 0
    order = np.argsort(step[keep], kind="stable")
    return StateRefreshLayout(R, Lmax, obs_token, token_row, step[keep][order], rollout[keep][order],
                              dst_slot[keep][order])


def check_state_refresh_layout(lay, B, K):
    """Raises ``ValueError`` unless the host ``StateRefreshLayout`` ``lay`` indexes a ``[S, B]`` batch with ``K`` reset rows
    per column: tokens and rows in range or -1, destinations at steps in [1, L_max) of rollouts in [0, R), sorted by step,
    and slots in [0, B + K*B), none twice.  ``dc_gather_columns_fill`` and ``dc_refresh_states`` index with them on the
    device, where they cannot be checked."""
    n_tok = lay.token_row.size
    if n_tok % max(B, 1) or lay.obs_token.size != lay.L_max * lay.R:
        raise ValueError("state refresh layout: %d tokens for %d columns, %d rows for L_max=%d, R=%d"
                         % (n_tok, B, lay.obs_token.size, lay.L_max, lay.R))
    for name, a, hi in (("obs_token", lay.obs_token, n_tok), ("token_row", lay.token_row, lay.obs_token.size)):
        if a.size and (a.min() < -1 or a.max() >= hi):
            raise ValueError("state refresh layout: %s values %d..%d outside [-1, %d)" % (name, a.min(), a.max(), hi))
    n = lay.step.size
    if lay.rollout.size != n or lay.slot.size != n:
        raise ValueError("state refresh layout: step, rollout and slot differ in length")
    if n and (lay.step.min() < 1 or lay.step.max() >= lay.L_max or np.any(np.diff(lay.step) < 0)):
        raise ValueError("state refresh layout: destination steps must be sorted and in [1, %d)" % lay.L_max)
    if n and (lay.rollout.min() < 0 or lay.rollout.max() >= lay.R):
        raise ValueError("state refresh layout: destination rollouts outside [0, %d)" % lay.R)
    if n and (lay.slot.min() < 0 or lay.slot.max() >= B + K * B):
        raise ValueError("state refresh layout: destination slots %d..%d outside [0, %d)"
                         % (lay.slot.min(), lay.slot.max(), B + K * B))
    if np.unique(lay.slot).size != n:
        raise ValueError("state refresh layout: a destination slot is written twice")


def refresh_token_map(lengths, seq_len, pack, mask_padding, layout=None):
    """For the rollout-major rows of experience prep (rollout i's ``Lp_i`` padded rows in turn), the token ``t * B + c``
    of the ``[S, B]`` training batch that ``batch_from_rollouts`` builds from rollouts of ``lengths`` real steps, or -1
    where the batch holds no such row or prep zeroes it (under ``mask_padding``: the rows after a rollout's real steps).
    Derived from the batch's own layout: ``chunk_columns`` applied to the row numbers, or with ``pack`` the inverse of
    ``packed_rows``.  Returns int64 ``[sum(Lp_i)]``.  The advantage refresh (``recompute_advantages``) scans the rows and
    reads values from, and writes advantages to, these tokens (``ops.gae_scan_indexed``).  ``layout``: with ``pack``, the
    ``pack_layout`` of ``lengths`` when the caller has it already."""
    S = int(seq_len)
    Ls = [int(L) for L in lengths]
    Lps = [(L + S - 1) // S * S for L in Ls]
    n_rows = int(sum(Lps))
    base = np.concatenate([[0], np.cumsum(Lps)[:-1]]).astype(np.int64)
    rows = _batch_rows(Ls, S, pack, layout)
    tok = np.full(n_rows, -1, dtype=np.int64)
    held = rows >= 0
    tok[rows[held]] = np.flatnonzero(held.reshape(-1))
    if mask_padding:                           # prep zeroes the advantages and returns of padded rows
        step = np.arange(n_rows, dtype=np.int64) - np.repeat(base, Lps)
        tok[step >= np.repeat(np.asarray(Ls, dtype=np.int64), Lps)] = -1
    return tok


def sequence_count(lengths, seq_len, pack=False):
    """The number of training sequences that rollouts of ``lengths`` steps make: ``ceil(L / seq_len)`` each, or with
    ``pack`` the columns of their ``pack_layout``."""
    unpacked = sum((int(L) + seq_len - 1) // seq_len for L in lengths)
    if not pack or not unpacked:
        return unpacked
    tails = [(int(L) % seq_len, i) for i, L in enumerate(lengths) if int(L) % seq_len]
    return sum(int(L) // seq_len for L in lengths) + _first_fit_decreasing(tails, seq_len)[2]


def check_reset_slots(reset_slot, K):
    """Raises ``ValueError`` unless every value of the host array ``reset_slot`` lies in [-1, K) and no reset row (k, column)
    is used twice: the recurrence kernels index the reset tables with them on the device, where they cannot be checked."""
    rs = np.asarray(reset_slot)
    if rs.size and (rs.min() < -1 or rs.max() >= K):
        raise ValueError("reset slots %d..%d outside [-1, %d)" % (rs.min(), rs.max(), K))
    t, c = np.nonzero(rs >= 0)
    rows = rs[t, c].astype(np.int64) * rs.shape[1] + c
    if np.unique(rows).size != rows.size:
        raise ValueError("a reset row is used by two tokens")


def check_behaviour_logp(datas):
    """Raises ``ValueError``, naming the rollout's ``game_id`` / ``player_id``, when a rollout lacks ``'behaviour_logp'``,
    when it is not ``[L, 5]``, or when it is not finite on a head that took an action (the host ``actions`` say which).
    Runs on the host before anything is uploaded; values on heads that did not act are ignored."""
    for d in datas:
        who = "rollout game_id=%r player_id=%r" % (d.get('game_id'), d.get('player_id'))
        if 'behaviour_logp' not in d:
            raise ValueError("%s has no 'behaviour_logp': advantage_estimator='vtrace' needs the actor's log-probabilities "
                             "of its actions ([L, 5], the logp of Policy.act_batched)" % who)
        L = int(d['rewards'].shape[0])
        blp = torch.as_tensor(d['behaviour_logp'])
        if tuple(blp.shape) != (L, len(ops.HEAD_KEYS)) or not blp.is_floating_point():
            raise ValueError("%s: 'behaviour_logp' must be a float [%d, %d] array, got %s %s"
                             % (who, L, len(ops.HEAD_KEYS), blp.dtype, tuple(blp.shape)))
        acted = torch.stack([torch.as_tensor(d['actions'][k]).reshape(L, -1).any(dim=1) for k in ops.HEAD_KEYS], dim=1)
        bad = acted & ~torch.isfinite(blp)
        if bool(bad.any()):
            t, h = (int(i) for i in bad.nonzero()[0])
            raise ValueError("%s: 'behaviour_logp' is %r at step %d on head %r, which took an action there"
                             % (who, float(blp[t, h]), t, ops.HEAD_KEYS[h]))


def check_demonstrations(datas):
    """Raises ``ValueError``, naming the rollout's ``game_id`` / ``player_id``, the step and the head, when a demonstration's
    action rows cannot be the log-likelihood's targets: a row with more than one entry set, a set entry that the step's
    mask makes illegal (its log-probability is -inf), or rows that do not follow the hierarchy ``Policy.select_actions``
    samples (one enum row; enum 1 -> x and y, 2 -> target_unit, 3 -> ability, 0 -> none; no other head has a row).  The
    first such step is reported.  Runs on the host before anything is uploaded."""
    keys = ops.HEAD_KEYS
    for d in datas:
        who = "rollout game_id=%r player_id=%r" % (d.get('game_id'), d.get('player_id'))
        L = int(d['rewards'].shape[0])
        acts = {k: torch.as_tensor(d['actions'][k]).reshape(L, -1).bool() for k in keys}
        masks = {k: torch.as_tensor(d['masks'][k]).reshape(L, -1).bool() for k in keys}
        enum = acts['enum']
        kind = torch.where(enum.any(dim=1), enum.int().argmax(dim=1), torch.full((L,), -1))
        found = []                                      # (step, head index, message) of the first failure of each check
        for h, k in enumerate(keys):
            checks = [(acts[k].sum(dim=1) > 1, "its action row has more than one entry set"),
                      ((acts[k] & ~masks[k]).any(dim=1), "its action is illegal under the step's mask")]
            if k == 'enum':
                checks.append((kind < 0, "there is no enum row; every step of a demonstration takes an enum action"))
            else:
                want = torch.zeros(L, dtype=torch.bool)
                for e, follow in ENUM_FOLLOWS.items():
                    if k in follow:
                        want |= kind == e
                has = acts[k].any(dim=1)
                checks.append((has & ~want, "it has an action row, which the step's enum action does not sample"))
                checks.append((want & ~has, "it has no action row, which the step's enum action samples"))
            for bad, why in checks:
                if bool(bad.any()):
                    t = int(bad.nonzero()[0])
                    found.append((t, h, "%s: step %d, head %r (enum %d): %s" % (who, t, k, int(kind[t]), why)))
        if found:
            raise ValueError("demonstration " + min(found)[2])


def check_continuation(datas, cell, num_layers, hidden_size):
    """Raises ``ValueError``, naming the rollout's ``game_id`` / ``player_id``, when one of the optional keys of a rollout
    cut from a longer game is malformed: an ``'initial_hidden'`` that is not the structure ``Policy.init_hidden()`` returns
    (a ``[num_layers, 1, hidden_size]`` float tensor or array; an ``(h, c)`` pair of them for the LSTM) or that is not
    finite; a ``'terminal'`` that is not a bool; a non-terminal rollout of no steps.  Also raises when an observation key
    does not have L rows (terminal) or L + 1 rows (non-terminal: row L is the state the game continues from).  Runs on the
    host before anything is uploaded."""
    want = (int(num_layers), 1, int(hidden_size))
    for d in datas:
        who = "rollout game_id=%r player_id=%r" % (d.get('game_id'), d.get('player_id'))
        terminal = d.get('terminal', True)
        if not isinstance(terminal, (bool, np.bool_)):
            raise ValueError("%s: 'terminal' must be True or False, got %r" % (who, terminal))
        L = int(d['rewards'].shape[0])
        if not terminal and L < 1:
            raise ValueError("%s: a non-terminal rollout needs at least one step" % who)
        rows = L if terminal else L + 1
        for k in Policy.INPUT_KEYS:
            n = int(d['observations'][k].shape[0])
            if n != rows:
                raise ValueError("%s: observations[%r] has %d rows; a %s rollout of %d steps carries %d"
                                 % (who, k, n, "terminal" if terminal else "non-terminal", L, rows))
        if 'initial_hidden' not in d:
            continue
        h = d['initial_hidden']
        pair = isinstance(h, (tuple, list))
        parts = list(h) if pair else [h]
        if pair != (cell == "lstm") or len(parts) != (2 if cell == "lstm" else 1):
            raise ValueError("%s: 'initial_hidden' must be %s, as Policy.init_hidden() returns for the %s"
                             % (who, "an (h, c) pair of [%d, %d, %d] arrays" % want if cell == "lstm"
                                else "one [%d, %d, %d] array" % want, cell.upper()))
        for p in parts:
            if not isinstance(p, (torch.Tensor, np.ndarray)):
                raise ValueError("%s: 'initial_hidden' holds a %s, not a tensor or an array" % (who, type(p).__name__))
            t = torch.as_tensor(p)
            if tuple(t.shape) != want or not t.is_floating_point():
                raise ValueError("%s: 'initial_hidden' must be float [%d, %d, %d], got %s %s"
                                 % ((who,) + want + (t.dtype, tuple(t.shape))))
            if not bool(torch.isfinite(t).all()):
                raise ValueError("%s: 'initial_hidden' is not finite" % who)


class DotaOptimizer:
    MODEL_FILENAME_FMT = "model_%09d.pt"
    ADAM_FILENAME_FMT = "adam_%09d.state"         # extension: Adam moments of the same iteration (torch.optim.Adam layout)
    ADAM_FILES_KEPT = 3
    # extension: the value statistics and the normalised value head of the same iteration (value_norm=True)
    VALUE_NORM_FILENAME_FMT = "value_norm_%09d.state"
    KL_COEF_FILENAME_FMT = "kl_coef_%09d.state"     # the adaptive KL coefficient of the same iteration (kl_target)
    # the K-row value head and its groups of the same iteration (value_heads); the published model holds it folded
    VALUE_HEADS_FILENAME_FMT = "value_heads_%09d.state"
    # the iterations trained with the teacher, its coefficient and its path, of the same iteration (teacher_model)
    TEACHER_FILENAME_FMT = "teacher_%09d.state"
    VALUE_NORM_MIN_STD = 1e-2       # floor of the value statistics' sigma: bounds the value head's rescale factor
    BUCKET_NAME = 'dotaservice'
    MODEL_HISTOGRAM_FREQ = 128
    MAX_GRAD_NORM = 0.5
    # the advantage and state refreshes (recompute_advantages, recompute_states) run their forwards over blocks of time
    # steps of about this many tokens
    REFRESH_CHUNK_TOKENS = 32768
    value_heads, n_value_heads, _vh_shape = None, 1, ()     # set by __init__ (value_heads)
    objective = 'ppo'                                       # set by __init__
    SPEED_KEY = 'steps per s'
    ADAM_BETAS = (0.9, 0.999)       # torch.optim.Adam defaults (:275)
    ADAM_EPS = 1e-8
    # Policy has 30 parameter tensors outside the recurrent core and 4 per recurrent layer; the fused gradient-finish
    # kernel (csrc/grad_finish.cu) keeps per-tensor slots for at most _lib.MAX_PARAM_TENSORS = 96 of them -> 16 layers.
    MAX_LAYERS = (_lib.MAX_PARAM_TENSORS - 30) // 4

    def __init__(self, rmq_host, rmq_port, epochs, min_seq_per_epoch, seq_len,
                 learning_rate, checkpoint, pretrained_model, mq_prefetch_count, log_dir,
                 entropy_coef, vf_coef, run_local, *, hidden_size=256, cell="gru", num_layers=1, mq=None,
                 iterations=100000, rollout_prefetch=0, gamma=GAMMA, gae_lambda=LAMBDA, clip_range=0.1,
                 max_grad_norm=0.5, value_clip=None, advantage_estimator='gae', vtrace_rho_clip=1.0, vtrace_c_clip=1.0,
                 num_minibatches=1, mask_padding=False, pack_sequences=False, policy_ratio='per_head', value_norm=False,
                 value_norm_decay=0.99, kl_coef=0.0, kl_target=None, kl_stop=None, recompute_advantages=False,
                 recompute_states=False, value_heads=None, value_gammas=None, teacher_model=None, teacher_coef=1.0,
                 teacher_anneal_iterations=None, upgo_coef=0.0, objective='ppo', dual_clip=None):
        if not 1 <= num_layers <= self.MAX_LAYERS:
            raise ValueError("num_layers=%r: DotaOptimizer trains 1 to %d recurrent layers (the fused gradient-finish kernel "
                             "handles at most %d parameter tensors, 30 + 4 per layer)"
                             % (num_layers, self.MAX_LAYERS, _lib.MAX_PARAM_TENSORS))
        check_ppo_settings(gamma, gae_lambda, clip_range, max_grad_norm, value_clip, advantage_estimator=advantage_estimator,
                           vtrace_rho_clip=vtrace_rho_clip, vtrace_c_clip=vtrace_c_clip, num_minibatches=num_minibatches,
                           mask_padding=mask_padding, pack_sequences=pack_sequences, policy_ratio=policy_ratio,
                           value_norm=value_norm, value_norm_decay=value_norm_decay, kl_coef=kl_coef, kl_target=kl_target,
                           kl_stop=kl_stop, recompute_advantages=recompute_advantages, recompute_states=recompute_states,
                           value_heads=value_heads, value_gammas=value_gammas, teacher_model=teacher_model,
                           teacher_coef=teacher_coef, teacher_anneal_iterations=teacher_anneal_iterations,
                           upgo_coef=upgo_coef, objective=objective, dual_clip=dual_clip)
        check_minibatch_count(num_minibatches, min_seq_per_epoch)
        # dual-clip PPO: the surrogate of every row with a negative normalised advantage A is floored at dual_clip * A
        # (dc_ppo_loss_fwd_bwd_dual_clip).  On or off is fixed here (the step's graph holds the loss kernel); the value can
        # be changed between steps, the upload before every step carries it to the device
        self.dual_clip = None if dual_clip is None else float(dual_clip)
        self._dual_clip_on = dual_clip is not None
        self.last_dual_clip_stats = None    # the shares of the rows where the floor binds, of the last step
        # 'bc': every rollout is a demonstration (check_demonstrations at prep) and the loss is dc_ppo_loss_fwd_bwd_bc's, the
        # NLL of the demonstrated actions with the entropy and value terms of 'ppo'.  Fixed per optimizer, like policy_ratio
        self.objective = objective
        self.last_bc_stats = None           # NLL, accuracy (and per head) of the last 'bc' step
        # value heads: one critic column per reward group, each with its own discount.  Prep scans every group
        # (gae_scan_heads), the policy trains on the summed advantage, the value loss is dc_value_heads_loss's and the
        # published model holds the heads folded into one row.  None: the reference's single critic, and none of this runs
        self.value_heads = value_head_groups(value_heads, value_gammas, gamma)
        self.n_value_heads = 1 if self.value_heads is None else len(self.value_heads.names)
        self._vh_shape = () if self.n_value_heads == 1 else (self.n_value_heads,)   # trailing dim of values / returns
        # True: before every epoch after the first, train_epochs reruns every rollout of the batch whole with the current
        # weights and writes the recurrent states entering its chunks (after the first) over the batch's h0 / c0 and reset
        # tables (_refresh_states); batch_from_rollouts then attaches what that needs (ExperienceBatch.state_refresh)
        self.recompute_states = recompute_states
        self._state_refresh_sums = []       # (device float64 [2] drift sums, states replaced) of this iteration's refreshes
        # True: before every epoch after the first, train_epochs recomputes the batch's advantages and returns with the
        # current critic (and, for V-trace, the current policy as the target), from prep's rewards, segments and bootstraps
        # (_refresh_advantages); batch_from_rollouts then attaches what that needs (ExperienceBatch.refresh)
        self.recompute_advantages = recompute_advantages
        # KL control: the loss adds kl_coef * KL(pi_prep || pi), the exact KL over the legal actions of every sampled head,
        # and a step whose all-ranks KL exceeds kl_stop is skipped and ends the iteration's updates.  kl_target adapts
        # kl_coef once per iteration.  kl_control fixes at construction whether prep stores the old distribution and the
        # step runs the KL kernels; kl_coef and kl_stop can then be scheduled like the other hyper-parameters.
        self.kl_coef = float(kl_coef)
        self.kl_target = None if kl_target is None else float(kl_target)
        self.kl_stop = None if kl_stop is None else float(kl_stop)
        self.kl_control = self.kl_coef > 0.0 or self.kl_stop is not None
        self.last_kl_updates = None         # (updates run, updates skipped) of the last train_epochs under kl_stop
        # True: PopArt.  The critic learns (R - mu) / sigma, with (mu, sigma) from running statistics of the value targets
        # (_value_norm = (m, q, w), updated once per prepared batch); the value head is rescaled at every update so that
        # sigma v + mu does not move.  policy_base's `value` output is then sigma^-1 (V - mu); prep, the batch, the
        # published model and agents see V.
        self.value_norm = value_norm
        self.value_norm_decay = float(value_norm_decay)
        self._value_norm = (0.0, 0.0, 0.0)
        # 'joint': the loss clips one PPO ratio per step, of the whole hierarchical action (log r = sum over the sampled
        # heads of logp_new - logp_old), averaged over the steps with an action; 'per_head': the reference's five ratios
        self.policy_ratio = policy_ratio
        # True: batch_from_rollouts packs the rollouts' tails into shared columns with state resets between them
        # (pack_layout), so the padding of every rollout's last chunk is not trained on
        self.pack_sequences = pack_sequences
        # True: the zero padding of each rollout's last chunk counts for nothing -- prep bootstraps at the real end and
        # marks the real steps (ExperienceBatch.valid), the loss leaves padded tokens out of every mean
        self.mask_padding = mask_padding
        # every epoch is split into num_minibatches shuffled minibatches of sequences, one optimizer step each (train_epochs)
        self.num_minibatches = int(num_minibatches)
        self.minibatch_rng = np.random.default_rng(7 + (dist.get_rank() if is_distributed() else 0))   # seed 7 as :34-36
        self.gamma, self.gae_lambda = float(gamma), float(gae_lambda)     # GAE of experience prep (:421)
        # 'vtrace': experience prep corrects advantages and value targets for the actors' stale weights, from the
        # behaviour log-probabilities each rollout carries ('behaviour_logp')
        self.advantage_estimator = advantage_estimator
        self.vtrace_rho_clip, self.vtrace_c_clip = float(vtrace_rho_clip), float(vtrace_c_clip)
        self._vtrace_seg_stats = None       # per-rollout sums of the last V-trace prep (device), see last_vtrace_stats
        # UPGO (AlphaStar): experience prep adds upgo_coef times the upgoing advantage to the GAE / V-trace advantage
        # (dc_upgo_scan), and the advantage refresh does the same.  Read at every prep, so it can be scheduled between
        # iterations; 0 runs nothing.  _upgo_prep: (coefficient, per-segment sums on the device) of the last prep with c > 0
        self.upgo_coef = float(upgo_coef)
        self._upgo_prep = None
        self.MAX_GRAD_NORM = float(max_grad_norm)     # shadows the class constant; read before every step, like lr below
        self.value_clip = None if value_clip is None else float(value_clip)
        self.rmq_host, self.rmq_port = rmq_host, rmq_port
        self.epochs = epochs
        self.min_seq_per_epoch = min_seq_per_epoch
        self.seq_len = seq_len
        self.learning_rate = learning_rate
        self.checkpoint = checkpoint
        self.mq_prefetch_count = mq_prefetch_count
        self.iteration_start = 1
        self.log_dir = log_dir
        self.entropy_coef = entropy_coef
        self.vf_coef = vf_coef
        self.run_local = run_local
        self.iterations = iterations        # :226
        self.model_upload_freq = 10         # :227
        self.e_clip = float(clip_range)     # :229
        self.device = _device()
        _lib.load()                         # fail loudly, up front, if the CUDA library is missing

        with torch.random.fork_rng(devices=[]):     # :34 seeds torch with 7 at import and Policy() init depends on it;
            torch.manual_seed(7)                    # forked so that constructing an optimizer leaves the caller's RNG alone
            self.policy_base = Policy(hidden_size=hidden_size, cell=cell, num_layers=num_layers,
                                      value_heads=self.n_value_heads)
        # Kickstarting: the loss adds teacher_coef * KL(pi_teacher || pi) over the legal actions of every sampled head, with
        # the teacher's rows computed once at prep.  teacher_coef can be scheduled between steps like kl_coef; with
        # teacher_anneal_iterations, run_iteration sets it to teacher_coef * max(0, 1 - n / N) (n: teacher_iterations) and
        # retires the teacher at 0.  The teacher is frozen: outside the flat parameters, Adam, the all-reduce and checkpoints
        self.teacher_model = teacher_model
        self.teacher_coef = float(teacher_coef)
        self._teacher_coef0 = self.teacher_coef
        self.teacher_anneal_iterations = teacher_anneal_iterations
        self.teacher_iterations = 0
        self.teacher = None
        if teacher_model is not None:
            with torch.random.fork_rng(devices=[]):   # building it draws from the RNG: leave the caller's alone, as above
                self.teacher = load_teacher(teacher_model).to(self.device)

        if self.checkpoint:
            logger.info('Checkpointing to: {}'.format(self.log_dir))
            os.makedirs(self.log_dir, exist_ok=True)
            if not self.run_local:
                logger.warning('GCS is out of scope for dotaclient_b200; checkpoints stay in %s', self.log_dir)
            latest_model = self.get_latest_model(prefix=self.log_dir)
            if latest_model is not None:
                logger.info('Found a latest model in pretrained dir: {}'.format(latest_model))
                if pretrained_model is not None:
                    logger.warning('Overriding pretrained model by latest model.')
                pretrained_model = os.path.join(self.log_dir, latest_model)
            if pretrained_model is not None:
                self.iteration_start = self.iteration_from_model_filename(filename=pretrained_model) + 1   # :253
        if pretrained_model is not None:
            # strict=False as the reference (:263-266): a checkpoint with fewer recurrent layers (e.g. a 1-layer model
            # loaded into num_layers=2) sets the layers it has and leaves rnn.*_l1 ... at their seeded initial values; its
            # Adam moments (keyed by parameter index) do not fit the new layout and are not restored (below)
            state = torch.load(pretrained_model, map_location='cpu')
            if self.value_heads is not None:        # the published head is one row: the K rows come from the side file
                state = self._value_heads_state(state, pretrained_model)
            self.policy_base.load_state_dict(state, strict=False)
            if self.checkpoint:
                # before the data-parallel wrapper broadcasts the weights: the normalised head must be in place
                self._restore_value_norm(os.path.join(os.path.dirname(pretrained_model),
                                                      self.VALUE_NORM_FILENAME_FMT % (self.iteration_start - 1)))
                self._restore_kl_coef(os.path.join(os.path.dirname(pretrained_model),
                                                   self.KL_COEF_FILENAME_FMT % (self.iteration_start - 1)))
                self._restore_teacher(os.path.join(os.path.dirname(pretrained_model),
                                                   self.TEACHER_FILENAME_FMT % (self.iteration_start - 1)))

        self.policy_base.to(self.device)
        self.flat = FlatParameterSpace(self.policy_base, self.device, kl_tail=self.kl_control)
        if is_distributed():
            self.policy = DistributedDataParallelSparseParamCPU(self.policy_base, flat_space=self.flat)   # :268-269
        else:
            self.policy = self.policy_base

        # Adam state lives next to the flat parameter buffer; `optimizer` keeps a torch-like handle (:275).
        self.exp_avg = torch.zeros_like(self.flat.param)
        self.exp_avg_sq = torch.zeros_like(self.flat.param)
        self.adam_steps = torch.zeros(self.flat.n_seg, dtype=torch.int32, device=self.device)
        self.optimizer = _FusedAdamHandle(self)
        if self.checkpoint and pretrained_model is not None:
            adam_file = os.path.join(os.path.dirname(pretrained_model), self.ADAM_FILENAME_FMT % (self.iteration_start - 1))
            if os.path.isfile(adam_file):
                logger.info('Restoring Adam state from {}'.format(adam_file))
                try:
                    self.optimizer.load_state_dict(torch.load(adam_file, map_location='cpu'))
                except ValueError as e:     # e.g. a 1-layer run's moments next to the weights loaded into num_layers=2
                    logger.warning('Not restoring Adam state from %s (%s): the moments start from zero', adam_file, e)
        self._sync_resume_state()
        self._n_actions = torch.zeros(8, dtype=torch.int32, device=self.device)   # + value-head flag (_upload_hparams)
        # grad-norm metrics and PPO diagnostics side by side: the step reads both back with one copy.  KL control: two more
        # metrics, the all-ranks KL and the skip flag of dc_grad_finish_kl
        self._n_metrics = _lib.FINISH_KL_METRICS if self.kl_control else 4
        # value heads: their statistics (dc_value_heads_loss) follow the PPO diagnostics, read back by the same copy
        n_vh = 0 if self.value_heads is None else _lib.VALUE_HEADS_STATS_SLOTS
        # the teacher's statistics (KL, per head, the loss term) come last, read back by the same copy
        n_t = 0 if self.teacher_model is None else _lib.TEACHER_STATS_SLOTS
        # behaviour cloning: its statistics (NLL, accuracy, per head) in the same place (a teacher is refused with it)
        n_bc = _lib.BC_STATS_SLOTS if objective == 'bc' else 0
        # dual clip: the shares of the rows where its floor binds, after all of the above
        n_dc = _lib.DUAL_CLIP_STATS_SLOTS if self._dual_clip_on else 0
        self._result_dev = torch.zeros(self._n_metrics + _lib.PPO_STATS_SLOTS + n_vh + n_t + n_bc + n_dc,
                                       dtype=torch.float32, device=self.device)
        self._metrics = self._result_dev[:self._n_metrics]
        self._ppo_stats = self._result_dev[self._n_metrics:self._n_metrics + _lib.PPO_STATS_SLOTS]
        o = self._n_metrics + _lib.PPO_STATS_SLOTS
        self._value_head_stats = self._result_dev[o:o + n_vh] if n_vh else None
        self._teacher_stats = self._result_dev[o + n_vh:o + n_vh + n_t] if n_t else None
        self._bc_stats = self._result_dev[o + n_vh:o + n_vh + n_bc] if n_bc else None
        self._dual_clip_off = o + n_vh + n_t + n_bc       # offset of the dual-clip statistics in _result_dev
        self._dual_clip_stats = self._result_dev[self._dual_clip_off:] if n_dc else None
        self._finish_ws = torch.zeros(_lib.FINISH_WORKSPACE_BYTES, dtype=torch.uint8, device=self.device)
        # learning_rate, e_clip, entropy_coef, vf_coef, MAX_GRAD_NORM and value_clip are read by the step's kernels from this
        # device block, rewritten from the pinned host copy before every step: a captured graph of the step holds the
        # block's address, not the values, so assignments between steps reach replayed steps too
        # Value heads: a second block, the first with vf_coef = 0 and no value clip, for the PPO loss, whose value term
        # dc_value_heads_loss replaces; both blocks go up in the one copy
        # Teacher: its coefficient is one more double after the blocks (not a block slot), uploaded by the same copy
        # Dual clip: its constant c is one more double after those, uploaded by the same copy
        n_blocks = 1 if self.value_heads is None else 2
        n_tc = 0 if self.teacher_model is None else 1
        n_hp = n_blocks * _lib.HPARAM_SLOTS + n_tc + (1 if self._dual_clip_on else 0)
        self._hparams_host_flat = torch.zeros(n_hp, dtype=torch.float64).pin_memory()
        self._hparams_dev_flat = torch.zeros(n_hp, dtype=torch.float64, device=self.device)
        self._hparams_host_all = self._hparams_host_flat[:n_blocks * _lib.HPARAM_SLOTS].view(n_blocks, _lib.HPARAM_SLOTS)
        self._hparams_dev_all = self._hparams_dev_flat[:n_blocks * _lib.HPARAM_SLOTS].view(n_blocks, _lib.HPARAM_SLOTS)
        o_tc = n_blocks * _lib.HPARAM_SLOTS
        self._teacher_coef_host = self._hparams_host_flat[o_tc:o_tc + n_tc]
        self._teacher_coef_dev = self._hparams_dev_flat[o_tc:o_tc + n_tc]
        self._dual_clip_host = self._hparams_host_flat[o_tc + n_tc:]
        self._dual_clip_dev = self._hparams_dev_flat[o_tc + n_tc:]
        self._hparams_host, self._hparams_dev = self._hparams_host_all[0], self._hparams_dev_all[0]
        self._hparams_dev_ppo = self._hparams_dev_all[n_blocks - 1]
        self._hparams_uploaded = None       # the values the device block holds
        self.last_ppo_stats = None          # approx_kl, clip_fraction (and per head), explained_variance of the last step
        self._host_result = torch.zeros(_lib.LOSS_SLOTS + self._result_dev.numel(), dtype=torch.float32).pin_memory()
        self.last_step_launch_estimate = 0
        self._staging, self._staging_event = {}, None    # pinned host staging of the batched experience prep
        # rollout_prefetch > 0: a background thread pulls and unpickles up to that many rollouts ahead (same order, same
        # rollouts as the reference's one-at-a-time loop, :448-466) while the GPU trains on the current iteration
        self.rollout_prefetch = int(rollout_prefetch)
        self._rollout_q, self._prefetch_thread = None, None
        self.use_cuda_graph = True          # replay device-resident batches of a known shape from a captured graph of the step
        self._graphs = {}                   # graph key -> "seen" (ran once), "eager" (capture failed) or a _CapturedStep
        self._input_slots = {}              # batch shape -> up to two sets of static device input buffers (prefetch + graph)
        self._last_iteration_shape = None
        self.time_last_it = time.time()

        self.mq = mq if mq is not None else MessageQueue(host=self.rmq_host, port=self.rmq_port,
                                                        prefetch_count=mq_prefetch_count,
                                                        use_model_exchange=self.checkpoint)
        self.mq.connect()
        self.upload_model(version=self.iteration_start)                  # :284

    def close(self):
        """Releases the captured step graphs (they hold NCCL work when data-parallel: destroy them BEFORE
        ``dist.destroy_process_group()``, which otherwise waits forever) and the pinned staging buffers."""
        self._graphs.clear()
        self._input_slots.clear()
        self._staging.clear()
        gc.collect()
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    def _sync_resume_state(self):
        """Data-parallel resume: only the master scans ``log_dir`` and restores (``checkpoint = is_master()``, :751), so the
        restored Adam moments, step counters and ``iteration_start`` are broadcast from rank 0 -- otherwise the replicas
        would apply different Adam updates to the same all-reduced gradient and silently diverge.  (The weights themselves
        are broadcast by the wrapper's ``sync_parameters``, distributed.py:71-74.)"""
        if not is_distributed():
            return
        dist.broadcast(self.exp_avg, 0)
        dist.broadcast(self.exp_avg_sq, 0)
        dist.broadcast(self.adam_steps, 0)
        it = torch.tensor([self.iteration_start], dtype=torch.int64, device=self.device)
        dist.broadcast(it, 0)
        self.iteration_start = int(it.item())
        if self.value_norm:                 # the value statistics (the normalised head travels with the weights)
            vn = torch.tensor(self._value_norm, dtype=torch.float64, device=self.device)
            dist.broadcast(vn, 0)
            self._value_norm = tuple(vn.tolist())
        if self.kl_target is not None:      # the adaptive KL coefficient
            kc = torch.tensor([self.kl_coef], dtype=torch.float64, device=self.device)
            dist.broadcast(kc, 0)
            self.kl_coef = float(kc.item())
        if self.teacher_model is not None:  # the iterations trained with the teacher and its coefficient
            tc = torch.tensor([float(self.teacher_iterations), self.teacher_coef], dtype=torch.float64, device=self.device)
            dist.broadcast(tc, 0)
            self.teacher_iterations, self.teacher_coef = int(tc[0].item()), float(tc[1].item())

    def _restore_teacher(self, path):
        """Resume with a teacher: the iterations already trained with it and its coefficient from ``path`` (written by
        ``upload_model``).  Without the file both start afresh; without a teacher the file is ignored."""
        if not os.path.isfile(path):
            return
        if self.teacher_model is None:
            logger.warning('Ignoring %s: this run has no teacher_model', path)
            return
        st = torch.load(path, map_location='cpu')
        logger.info('Restoring the teacher schedule from %s (%d iterations, coefficient %r)', path, st['iterations'],
                    st['teacher_coef'])
        self.teacher_iterations, self.teacher_coef = int(st['iterations']), float(st['teacher_coef'])
        if self.teacher_coef == 0.0 and self.teacher_anneal_iterations is not None:
            self._retire_teacher()

    def _retire_teacher(self):
        """The anneal reached 0: prep stops running the teacher, batches carry no teacher rows, the step runs without the
        term, and the teacher's device memory is released."""
        if self.teacher is not None:
            logger.info('The teacher coefficient has annealed to 0: retiring the teacher')
            self.teacher = None
            gc.collect()
            if torch.cuda.is_available():
                torch.cuda.empty_cache()

    def _restore_kl_coef(self, path):
        """Resume with ``kl_target``: the adaptive KL coefficient from ``path`` (written by ``upload_model``).  Without the
        file the coefficient starts from ``kl_coef``; without ``kl_target`` the file is ignored."""
        if not os.path.isfile(path):
            return
        if self.kl_target is None:
            logger.warning('Ignoring %s: kl_target is off, so kl_coef stays at %r', path, self.kl_coef)
            return
        logger.info('Restoring the adaptive KL coefficient from {}'.format(path))
        self.kl_coef = float(torch.load(path, map_location='cpu')['kl_coef'])

    def _value_heads_state(self, state, model_path):
        """Resume with ``value_heads``: ``state`` (the published model at ``model_path``, whose value head is one row) with
        the K-row head from the ``VALUE_HEADS_FILENAME_FMT`` file of the same iteration next to it (``upload_model``).  Raises ``ValueError`` when the file's groups are not this run's: its rows
        cannot be reinterpreted.  Without the file -- a model of the reference or of a run without heads -- every head
        starts from ``split_value_head``: W / K and b / K, so the summed value starts where the one-row head's was."""
        vh = self.value_heads
        it = re.search(r'(\d+)(?=\.pt$)', os.path.basename(model_path))
        path = os.path.join(os.path.dirname(model_path), self.VALUE_HEADS_FILENAME_FMT % int(it.group(0))) if it else ''
        if os.path.isfile(path):
            st = torch.load(path, map_location='cpu')
            saved = (tuple(st['names']), tuple(tuple(k) for k in st['keys']))
            if saved != (vh.names, vh.keys):
                raise ValueError("%s holds value heads %s; this run's are %s: the heads cannot be reinterpreted"
                                 % (path, dict(zip(*saved)), dict(zip(vh.names, vh.keys))))
            logger.info('Restoring the %d value heads from %s', len(vh.names), path)
            return dict(state, **{'affine_value.weight': st['weight'], 'affine_value.bias': st['bias']})
        if 'affine_value.weight' in state and state['affine_value.weight'].shape[0] == 1:
            logger.info('No value heads next to %s: every one of the %d heads starts from 1/%d of its one-row value head',
                        model_path, self.n_value_heads, self.n_value_heads)
            return split_value_head(state, self.n_value_heads)
        return state

    def _restore_value_norm(self, path):
        """Resume with ``value_norm``: the statistics and the exact normalised value head from ``path`` (written by
        ``upload_model`` next to the weights).  Without the file -- e.g. a model trained without the feature -- the
        statistics start at identity and the head stays as loaded, which is then already in raw units.  Without the feature
        the file is ignored."""
        if not os.path.isfile(path):
            return
        if not self.value_norm:
            logger.warning('Ignoring %s: value_norm is off, so the value head stays in the raw units it was published in',
                           path)
            return
        logger.info('Restoring the value statistics and the normalised value head from {}'.format(path))
        st = torch.load(path, map_location='cpu')
        self._value_norm = (float(st['m']), float(st['q']), float(st['w']))
        with torch.no_grad():
            self.policy_base.affine_value.weight.copy_(st['weight'])
            self.policy_base.affine_value.bias.copy_(st['bias'])

    # -- checkpoints (:287-308, :697-723) --------------------------------------------------------
    @staticmethod
    def iteration_from_model_filename(filename):
        return int(re.search(r'(\d+)(?=.pt)', filename).group(0))

    def get_latest_model(self, prefix):
        """Lexicographically latest ``*.pt`` in ``prefix`` (local listing; the reference's local branch
        is broken -- ``os.path.isfile`` relative to cwd and ``.name`` on a str, :296,302 -- this is the intent)."""
        if not os.path.isdir(prefix):
            return None
        names = sorted(f for f in os.listdir(prefix) if f.endswith('.pt') and os.path.isfile(os.path.join(prefix, f)))
        return names[-1] if names else None

    def upload_model(self, version):
        if not is_master():
            return
        buffer = io.BytesIO()
        state_dict = {k: v.detach().cpu().clone() for k, v in self.policy_base.state_dict().items()}
        if self.value_norm:
            # the published head is the denormalised one, sigma W and sigma b + mu (float64, rounded once): plain Policy
            # users and agents read raw-scale values, and the state_dict keeps its keys and shapes
            mu, sigma = self._value_norm_moments()
            w_n, b_n = state_dict['affine_value.weight'], state_dict['affine_value.bias']
            state_dict['affine_value.weight'] = (sigma * w_n.double()).float()
            state_dict['affine_value.bias'] = (sigma * b_n.double() + mu).float()
        if self.value_heads is not None:
            # the published model is the reference's network: the K rows folded into one, V = sum_k V_k (strict-loadable
            # by unmodified agents); the rows themselves go to the side file below
            w_h, b_h = state_dict['affine_value.weight'], state_dict['affine_value.bias']
            state_dict = fold_value_heads(state_dict)
        torch.save(obj=state_dict, f=buffer)                              # same bytes-format as :705-709
        state_dict_b = buffer.getvalue()
        if self.checkpoint:
            with open(os.path.join(self.log_dir, self.MODEL_FILENAME_FMT % version), 'wb') as f:
                f.write(state_dict_b)
            # extension (SURVEY.md 8(f)3): the Adam moments next to the weights, in torch.optim.Adam's own format.  The name
            # does not end in .pt, so the reference's "latest *.pt" scan and its agents never see it.
            torch.save(self.optimizer.state_dict(), os.path.join(self.log_dir, self.ADAM_FILENAME_FMT % version))
            side = [r'adam_\d{9}\.state']
            if self.value_norm:             # the statistics and the exact normalised head, for resume
                m, q, w = self._value_norm
                torch.save({'m': m, 'q': q, 'w': w, 'weight': w_n, 'bias': b_n},
                           os.path.join(self.log_dir, self.VALUE_NORM_FILENAME_FMT % version))
                side.append(r'value_norm_\d{9}\.state')
            if self.value_heads is not None:    # the K rows and what they mean, for resume
                vh = self.value_heads
                torch.save({'names': list(vh.names), 'keys': [list(k) for k in vh.keys], 'gammas': vh.gammas.tolist(),
                            'weight': w_h, 'bias': b_h}, os.path.join(self.log_dir, self.VALUE_HEADS_FILENAME_FMT % version))
                side.append(r'value_heads_\d{9}\.state')
            if self.kl_target is not None:  # the adaptive KL coefficient the next iteration trains with, for resume
                torch.save({'kl_coef': self.kl_coef}, os.path.join(self.log_dir, self.KL_COEF_FILENAME_FMT % version))
                side.append(r'kl_coef_\d{9}\.state')
            if self.teacher_model is not None:  # the teacher schedule the next iteration continues, for resume
                torch.save({'iterations': self.teacher_iterations, 'teacher_coef': self.teacher_coef,
                            'teacher_model': str(self.teacher_model)},
                           os.path.join(self.log_dir, self.TEACHER_FILENAME_FMT % version))
                side.append(r'teacher_\d{9}\.state')
            for pattern in side:            # resume only ever needs the newest: bound the disk growth
                stale = sorted(f for f in os.listdir(self.log_dir) if re.fullmatch(pattern, f))[:-self.ADAM_FILES_KEPT]
                for f in stale:
                    os.remove(os.path.join(self.log_dir, f))
        self.mq.publish_model(msg=state_dict_b, hdr={'version': version})   # :716

    # -- experience intake (:314-430) -------------------------------------------------------------
    def get_rollout(self):
        method, properties, body = self.mq.consume_xp()
        return self._describe_rollout(pickle.loads(body))

    @staticmethod
    def _describe_rollout(data):
        rollout_len = data['rewards'].shape[0]
        subrewards = data['rewards'].sum(axis=0)
        return data, subrewards, rollout_len, data['weight_version'], data.get('canvas')

    def _next_rollout(self):
        """``get_rollout()``, optionally served by the decode-ahead thread -- same rollouts, same order as the reference's
        one-at-a-time loop (:448-466).  (A pool of decoder PROCESSES was measured and dropped: ``pickle.loads`` of a 2.7 MB
        rollout is 4 ms here, shipping the bytes out and the tensors back through shared memory costs 9x that.)"""
        if self.rollout_prefetch <= 0:
            return self.get_rollout()
        if self._prefetch_thread is None:
            self._rollout_q = queue.Queue(maxsize=self.rollout_prefetch)

            def pump():
                while True:
                    self._rollout_q.put(self.get_rollout())
            self._prefetch_thread = threading.Thread(target=pump, daemon=True, name="dc-rollout-decode")
            self._prefetch_thread.start()
        return self._rollout_q.get()

    def experiences_from_rollout(self, data):
        """Rollout -> list of ``Sequence`` (:328-430): ``experiences_from_rollouts`` on a batch of one.

        Running the recurrence over the whole zero-padded rollout from the zero state is exactly the
        reference's chunk-by-chunk forward with carried hidden (:340,384-385); the hidden state entering
        chunk i is read back from the recurrence's state buffer.  Old log-probs come from the fused
        selected-log-prob kernel, advantages/returns from the GAE scan kernel (padding inside the scan).
        """
        return self.experiences_from_rollouts([data])[0]

    def _prepare_rollouts(self, datas):
        """The batched no-grad half of an iteration (SURVEY.md 8(f)2): all rollouts become the batch dimension of ONE
        time-major ``[L_max, R, ...]`` pass -- encoder chain, recurrence from the zero state, heads, selected log-probs
        (:384-390) -- followed by ONE segmented GAE scan over every rollout's own padded length (:417-421), or with
        ``advantage_estimator='vtrace'`` ONE segmented V-trace scan of the same segments.  With ``mask_padding`` each
        rollout is two segments, its real steps and its padding (``rollout_segments``), so the terminal bootstrap
        follows the last real step; advantages and returns of padded rows are then zeroed and ``valid [S, B]`` marks the
        real steps of every chunk.

        A rollout cut from a longer game (``check_continuation``) starts the pass from its ``'initial_hidden'`` instead of
        the zero state.  One that is not ``'terminal'`` is always two segments, and its real segment bootstraps from
        V(s_L), the critic's value of its extra observation row: ONE more single-step forward of batch R' (the number of
        such rollouts) from each one's state after its last step, state buffer slot L_i.  The extra row enters neither the
        main pass nor the batch.  Without either key in any rollout none of this runs.

        With a teacher (``teacher_model``) and ``teacher_coef > 0``, one more no-grad forward of the teacher over the same
        observations, from the teacher's zero state (also for a rollout with ``'initial_hidden'``: the actor's state is the
        student's), gives the teacher's masked log-prob rows ``teacher_log_probs [Lmax, R, 65]``.

        With ``value_norm`` the values and bootstraps read from the normalised head are denormalised first, so the scans,
        ``Sequence.values`` and the batch stay in raw units; at the end the value statistics take this batch's targets and
        the value head is rescaled (``_update_value_norm``).  Data-parallel, that update all-reduces across the ranks, so
        prep is then a collective: every rank must prepare a batch for each iteration.  Returns the raw device tensors;
        ``experiences_from_rollouts`` / ``batch_from_rollouts`` slice them."""
        S, dev, pol = self.seq_len, self.device, self.policy_base
        R = len(datas)
        n_layers, H, lstm = pol.num_layers, pol.hidden_size, pol.cell == "lstm"
        vtrace = self.advantage_estimator == 'vtrace'
        if vtrace:
            check_behaviour_logp(datas)                # refused before anything is uploaded
        if self.objective == 'bc':
            check_demonstrations(datas)                # so is a demonstration whose actions have no log-likelihood
        check_continuation(datas, pol.cell, n_layers, H)
        upgo = self._upgo_coef_now()                   # so is a coefficient assigned outside its domain
        Ls = [int(d['rewards'].shape[0]) for d in datas]
        Lps = [(L + S - 1) // S * S for L in Ls]
        Lmax = max(Lps)
        same = all(L == Lmax for L in Ls)
        terminal = [bool(d.get('terminal', True)) for d in datas]
        cut = [i for i in range(R) if not terminal[i]]           # the rollouts whose game goes on: bootstrapped from V(s_L)
        carried = any('initial_hidden' in d for d in datas)

        if self._staging_event is not None:
            self._staging_event.synchronize()          # the previous iteration's uploads have left the staging buffers

        def pinned(key, shape, dtype):
            buf = self._staging.get(key)
            if buf is None or buf.shape != shape or buf.dtype != dtype:
                buf = torch.empty(shape, dtype=dtype).pin_memory()
                self._staging[key] = buf
            return buf

        def batched(group, key, dtype):
            """Rollouts -> one time-major ``[Lmax, R, ...]`` device tensor.  The host side only does contiguous per-rollout
            copies into a cached PINNED ``[R, Lmax, ...]`` staging buffer (memcpy speed; stacking time-major on the host is a
            768-byte-granular scatter, 3x slower) and uploads asynchronously; the transposition to time-major runs on the GPU.
            ``group`` None: a top-level key of the rollout."""
            srcs = [torch.as_tensor(d[group][key] if group else d[key]) for d in datas]
            buf = pinned((group, key), (R, Lmax) + tuple(srcs[0].shape[1:]), dtype)
            for i, t in enumerate(srcs):
                buf[i, :Ls[i]].copy_(t[:Ls[i]])                                        # not the extra row of a cut rollout
                if Ls[i] < Lmax:
                    buf[i, Ls[i]:].zero_()                                             # zero padding (:367-382)
            return buf.to(dev, non_blocking=True).transpose(0, 1).contiguous()

        obs = {k: batched('observations', k, torch.float32) for k in Policy.INPUT_KEYS}
        masks = {k: batched('masks', k, torch.bool) for k in Policy.OUTPUT_KEYS}
        actions = {k: batched('actions', k, torch.bool) for k in Policy.OUTPUT_KEYS}
        behaviour_logp = batched(None, 'behaviour_logp', torch.float32) if vtrace else None      # [Lmax, R, 5]
        if carried:                                    # the actors' states entering each rollout, zero where absent
            buf = pinned(('initial_hidden',), (2 if lstm else 1, n_layers, R, H), torch.float32)
            buf.zero_()
            for i, d in enumerate(datas):
                if 'initial_hidden' in d:
                    for j, part in enumerate(d['initial_hidden'] if lstm else [d['initial_hidden']]):
                        buf[j, :, i].copy_(torch.as_tensor(part).reshape(n_layers, H))
            state0 = buf.to(dev, non_blocking=True)
        seg_np, boot_src, seg_valid = rollout_segments(Ls, terminal, S, self.mask_padding)
        if cut:                                        # the observation each cut game continues from: row L_i, [1, R', ...]
            obs_next = {}
            for k in Policy.INPUT_KEYS:
                srcs = [torch.as_tensor(datas[i]['observations'][k])[Ls[i]] for i in cut]
                buf = pinned(('bootstrap', k), (len(cut),) + tuple(srcs[0].shape), torch.float32)
                for j, t in enumerate(srcs):
                    buf[j].copy_(t)
                obs_next[k] = buf.to(dev, non_blocking=True).unsqueeze(0)
            # state buffer slot (L_i) and column (i) of every cut rollout's state after its last step, and for every segment
            # the slot of its bootstrap in [0, b_0, b_1, ...]
            idx = torch.from_numpy(np.concatenate([[Ls[i] for i in cut], cut, boot_src + 1]).astype(np.int64))
            idx = idx.pin_memory().to(dev, non_blocking=True)
            slot_last, col_last, boot_slot = idx[:len(cut)], idx[len(cut):2 * len(cut)], idx[2 * len(cut):]
        self._staging_event = torch.cuda.Event()
        self._staging_event.record()
        rewards_np = np.zeros((R, Lmax, len(REWARD_KEYS)), dtype=np.float32)
        for i, d in enumerate(datas):
            rewards_np[i, :Ls[i]] = np.asarray(d['rewards'], dtype=np.float32)
        with torch.no_grad():
            if carried:
                h0, c0 = state0[0], (state0[1] if lstm else None)
            else:
                h0 = torch.zeros((n_layers, R, H), dtype=torch.float32, device=dev)
                c0 = torch.zeros_like(h0) if lstm else None
            # every layer's state buffers are kept: the state entering chunk j of rollout i is ybufs[k][j*S, i] per layer k
            ybufs, cbufs, logits, values = self._rollout_forward(obs, h0, c0)
            # value_norm: the head is normalised; everything prep makes from it is in raw units, V = mu + sigma v with the
            # statistics this forward ran under (denormalised from the packed column into a contiguous [Lmax, R] tensor)
            vn = self._value_norm_moments() if self.value_norm else None
            bootstrap = boot = None
            if cut:                                    # V(s_L) of every cut rollout: one step of batch R' from slot L_i
                hb = ops.stack_layers([yb[slot_last, col_last] for yb in ybufs])
                cb = ops.stack_layers([c[slot_last, col_last] for c in cbufs]) if lstm else None
                bootstrap = self._rollout_forward(obs_next, hb, cb)[3].reshape((len(cut),) + self._vh_shape)
                if vn is not None:
                    bootstrap = ops.value_denorm(bootstrap, *vn)
                boot = torch.cat([bootstrap.new_zeros((1,) + self._vh_shape), bootstrap])[boot_slot]   # per segment
            keys = ops.HEAD_KEYS
            old_log_probs = None
            if self.kl_control:                        # and every head's full masked log-prob row, for the KL terms
                old_logp, old_log_probs = ops.selected_logp_rows([logits[k] for k in keys], [masks[k] for k in keys],
                                                                 [actions[k] for k in keys])
                old_logp, old_log_probs = old_logp.view(Lmax, R, 5), old_log_probs.view(Lmax, R, _lib.KL_ROW_FLOATS)
            else:
                old_logp = ops.selected_logp([logits[k] for k in keys], [masks[k] for k in keys],
                                             [actions[k] for k in keys]).view(Lmax, R, 5)        # :387-390
            teacher_log_probs = None
            if self.teacher is not None and self.teacher_coef > 0.0:
                t = self.teacher
                ht = torch.zeros((t.num_layers, R, t.hidden_size), dtype=torch.float32, device=dev)
                t_logits = self._rollout_forward(obs, ht, torch.zeros_like(ht) if t.cell == "lstm" else None, pol=t)[2]
                teacher_log_probs = ops.selected_logp_rows([t_logits[k] for k in keys], [masks[k] for k in keys],
                                                           [actions[k] for k in keys])[1].view(Lmax, R, _lib.KL_ROW_FLOATS)
                del t_logits
            # GAE per rollout over ITS padded length: back-to-back segments, rollout-major
            values_lr = values.reshape((Lmax, R) + self._vh_shape) if vn is None else \
                ops.value_denorm(values, *vn).view(Lmax, R)

            def rollout_major(t):                    # [Lmax, R, ...] -> the rows of every rollout's padded length in turn
                if same:
                    return t.transpose(0, 1).reshape((R * Lmax,) + tuple(t.shape[2:]))
                return torch.cat([t[:Lps[i], i] for i in range(R)])
            vals_c = rollout_major(values_lr)
            if same:
                rew_c = torch.from_numpy(rewards_np.reshape(R * Lmax, -1)).to(dev, non_blocking=True)
            else:
                rew_c = torch.from_numpy(np.concatenate([rewards_np[i, :Lps[i]] for i in range(R)])).to(dev)
            # [real | padding] per rollout under mask_padding or when cut: the bootstrap follows step L_i
            seg = torch.tensor(seg_np, dtype=torch.int64, device=dev)
            blp_c = lt_c = valid_len = None
            if vtrace:
                # heads that took no action carry no behaviour log-prob (old_logp is 0 there too); padding rows are 0 already
                acted = torch.stack([actions[k].any(dim=-1) for k in keys], dim=-1)
                behaviour_logp = torch.where(acted, behaviour_logp, 0.0)
                valid_len = torch.from_numpy(seg_valid).pin_memory().to(dev, non_blocking=True)  # padding: no real steps
                blp_c, lt_c = rollout_major(behaviour_logp), rollout_major(old_logp)
                adv_c, ret_c, self._vtrace_seg_stats = ops.vtrace_scan(
                    rew_c, vals_c, lt_c, blp_c, seg, gamma=self.gamma,
                    lam=self.gae_lambda, rho_clip=self.vtrace_rho_clip, c_clip=self.vtrace_c_clip, boot_value=boot,
                    valid_len=valid_len, stats=True)
            elif self.value_heads is not None:
                # every group's GAE with its own discount and head, the advantages summed; ret_c [rows(, K)]
                vh = self.value_heads
                adv_c, ret_c = ops.gae_scan_heads(rew_c, vals_c.reshape(-1, self.n_value_heads), seg, vh.group,
                                                  vh.gammas, self.gae_lambda, boot_value=boot, boot_reward=boot)
                ret_c = ret_c.view((-1,) + self._vh_shape)
            else:
                # :417-421; a cut rollout's returns go on past the cut as gamma^(L-t) V(s_L), its advantages from V(s_L)
                adv_c, ret_c = ops.gae_scan(rew_c, vals_c, seg, gamma=self.gamma, lam=self.gae_lambda, boot_value=boot,
                                            boot_reward=boot)
            self._upgo_prep = None
            if upgo > 0.0:
                # + c A^U over the same segments, values and bootstraps, before the padded rows are zeroed below
                upgo_valid = valid_len if valid_len is not None else \
                    torch.from_numpy(seg_valid).pin_memory().to(dev, non_blocking=True)
                _, upgo_stats = ops.upgo_scan(rew_c, vals_c, seg, adv_c, self.gamma, upgo, boot_value=boot,
                                              logp_target=lt_c, logp_behaviour=blp_c, rho_clip=self.vtrace_rho_clip,
                                              valid_len=upgo_valid, stats=True)
                self._upgo_prep = (upgo, upgo_stats)
            valid = None
            if self.mask_padding:
                lens = torch.tensor(chunk_valid_lengths(Ls, S), dtype=torch.int64).pin_memory().to(dev, non_blocking=True)
                valid = torch.arange(S, device=dev).unsqueeze(1) < lens.unsqueeze(0)             # [S, B]
                real = valid.t().reshape(-1)                                                      # rollout-major rows
                adv_c.masked_fill_(~real, 0.0)
                ret_c.masked_fill_(~real.view((-1,) + (1,) * len(self._vh_shape)), 0.0)
            if self.value_norm:                        # the statistics of this batch's raw targets, then the POP rescale
                self._update_value_norm(ret_c, real if self.mask_padding else None)
        return dict(obs=obs, masks=masks, actions=actions, rewards_np=rewards_np, old_logp=old_logp, values_lr=values_lr,
                    adv_c=adv_c, ret_c=ret_c, ybufs=ybufs, cbufs=cbufs, Ls=Ls, Lps=Lps, Lmax=Lmax, same=same, valid=valid,
                    bootstrap=bootstrap, old_log_probs=old_log_probs, teacher_log_probs=teacher_log_probs,
                    refresh=dict(rewards=rew_c, seg_off=seg, boot=boot, behaviour_logp=blp_c, valid_len=valid_len),
                    state_refresh=dict(h0=h0, c0=c0,
                                       obs_next=obs_next if cut else None,
                                       cut_len=np.array([Ls[i] for i in cut], dtype=np.int64) if cut else None,
                                       cut_rollout=np.array(cut, dtype=np.int64) if cut else None,
                                       boot_slot=boot_slot if cut else None))

    def _rollout_forward(self, obs, h0, c0, pol=None):
        """The no-grad rollout-major forward of experience prep and of the state refresh (of ``pol``: the student
        ``policy_base`` by default, or the teacher): the encoder over time-major
        ``[T, R, ...]`` observations (``Policy.INPUT_KEYS``), every recurrent layer from ``h0`` / ``c0 [L, R, H]`` (c0 None
        for the GRU) keeping its state buffers, and the heads.  Returns ``(ybufs, cbufs, logits, values)``: per layer the
        ``[T + 1, R, H]`` state buffers of ``ops.rnn_stack_forward_states`` (slot t: the state entering step t), the head
        logits and the value columns ``[T, R, K]`` of the packed head output (K = the value heads, 1 without them;
        normalised under ``value_norm``)."""
        pol = self.policy_base if pol is None else pol
        x, unit_embedding = pol._encode(obs['env'], [obs[k] for k in Policy.INPUT_KEYS[1:]])
        layers = [pol.rnn.layer(k) for k in range(pol.num_layers)]
        ybufs, cbufs = ops.rnn_stack_forward_states(x.contiguous(), layers, h0, c0, pol.cell)
        logits, values = pol._heads(ybufs[-1][1:], unit_embedding)
        return ybufs, cbufs, logits, values

    def experiences_from_rollouts(self, datas):
        """``experiences_from_rollout`` (:328-430) for all rollouts of an iteration at once: per rollout the result equals a
        batch of one -- own padding to a multiple of ``seq_len``, own terminal bootstrap, chunks beyond its padded
        length are not emitted -- but the work is one batched pass instead of ``R`` batch-1 passes."""
        S, pol = self.seq_len, self.policy_base
        p = self._prepare_rollouts(datas)
        obs, masks, actions, ybufs, cbufs, Lps = p['obs'], p['masks'], p['actions'], p['ybufs'], p['cbufs'], p['Lps']
        t_rows = p.get('teacher_log_probs')
        out = []
        for i, d in enumerate(datas):
            base = int(sum(Lps[:i]))
            col = base // S                          # the batch column of the rollout's first chunk
            sequences = []
            for j in range(Lps[i] // S):
                sl = slice(j * S, (j + 1) * S)
                h = ops.stack_layers([yb[j * S, i] for yb in ybufs]).unsqueeze(1)             # [L, 1, H]
                if pol.cell == "lstm":
                    hid = (h, ops.stack_layers([cb[j * S, i] for cb in cbufs]).unsqueeze(1))
                else:
                    hid = h
                seq = Sequence(game_id=d.get('game_id'), weight_version=d.get('weight_version'), team_id=d.get('team_id'),
                               observations={k: v[sl, i] for k, v in obs.items()},
                               actions={k: v[sl, i] for k, v in actions.items()},
                               masks={k: v[sl, i] for k, v in masks.items()},
                               values=p['values_lr'][sl, i].reshape(1, S, self.n_value_heads), rewards=p['rewards_np'][i, sl],
                               hidden=hid,
                               old_logp=p['old_logp'][sl, i],
                               valid=None if p['valid'] is None else p['valid'][:, col + j],
                               old_log_probs=None if p['old_log_probs'] is None else p['old_log_probs'][sl, i],
                               teacher_log_probs=None if t_rows is None else t_rows[sl, i])
                seq.advantages = p['adv_c'][base + j * S: base + (j + 1) * S]
                seq.returns = p['ret_c'][base + j * S: base + (j + 1) * S]
                sequences.append(seq)
            out.append(sequences)
        return out

    def batch_from_rollouts(self, datas):
        """Rollouts -> one stacked, time-major ``ExperienceBatch`` (what ``train`` consumes; :587-615 stacks the same
        sequences batch-first), in the order ``experiences_from_rollouts`` emits them (rollout by rollout, chunk by chunk).
        Built from the prepared ``[L_max, R, ...]`` tensors with a handful of tensor ops per ROLLOUT -- no per-sequence
        Python objects, no per-sequence re-stacking (an iteration of the stream has ~1000 sequences of 16 steps)."""
        S, pol = self.seq_len, self.policy_base
        p = self._prepare_rollouts(datas)
        lay = pack_layout(p['Ls'], S) if self.pack_sequences else None
        batch = self._packed_batch(p, lay) if self.pack_sequences else self._unpacked_batch(p)
        if self.recompute_advantages:          # the scan inputs of prep and where each of its rows sits in the batch
            tok = refresh_token_map(p['Ls'], S, self.pack_sequences, self.mask_padding, layout=lay)
            tok = torch.from_numpy(tok).pin_memory().to(self.device, non_blocking=True)
            batch.refresh = AdvantageRefresh(tok=tok, **p['refresh'])
        if self.recompute_states:              # where the rollouts' rows and chunk starts sit in the batch, checked here
            sl = state_refresh_layout(p['Ls'], S, self.pack_sequences, layout=lay)
            check_state_refresh_layout(sl, batch.batch_size, 0 if batch.reset_h is None else batch.reset_h.shape[0])
            idx = np.concatenate([sl.obs_token, sl.token_row, sl.step, sl.rollout, sl.slot])
            idx = torch.from_numpy(idx).pin_memory().to(self.device, non_blocking=True)
            n_o, n_t, n = sl.obs_token.size, sl.token_row.size, sl.step.size
            o = n_o + n_t
            rec = dict(p['state_refresh'])
            if not any('initial_hidden' in d for d in datas):       # every rollout starts from zeros
                rec.update(h0=None, c0=None)
            if not self.recompute_advantages:     # the bootstrap inputs serve only the advantages
                rec.update(obs_next=None, cut_len=None, cut_rollout=None, boot_slot=None)
            batch.state_refresh = StateRefresh(sl, idx[:n_o], idx[n_o:o], idx[o:o + n], idx[o + n:o + 2 * n],
                                               idx[o + 2 * n:], **rec)
        return batch

    def _unpacked_batch(self, p):
        """The ``ExperienceBatch`` of ``batch_from_rollouts`` without packing: every rollout's chunks in turn
        (``chunk_columns``)."""
        S, pol = self.seq_len, self.policy_base
        R, Lps = len(p['Ls']), p['Lps']
        n_chunks = [lp // S for lp in Lps]

        def chunked(t):                       # [Lmax, R, ...] -> [S, sum(n_chunks), ...]
            return chunk_columns(t, Lps, S, whole=p['same'] and p['Lmax'] == S)
        obs = {k: chunked(v) for k, v in p['obs'].items()}
        masks = {k: chunked(v) for k, v in p['masks'].items()}
        actions = {k: chunked(v) for k, v in p['actions'].items()}
        old_logp = chunked(p['old_logp'])
        B = sum(n_chunks)
        adv = p['adv_c'].view(B, S).t().contiguous()                  # the GAE outputs are rollout-major back-to-back segments
        ret = p['ret_c'].view((B, S) + tuple(p['ret_c'].shape[1:])).transpose(0, 1).contiguous()   # [S, B(, K)]
        # hidden state entering chunk j of rollout i = state buffer slot j*S of every layer (:340,384-385: carried, not
        # re-zeroed), stacked [L, B, H]
        t_idx = torch.tensor([j * S for i in range(R) for j in range(n_chunks[i])], dtype=torch.int64, device=self.device)
        r_idx = torch.tensor([i for i in range(R) for _ in range(n_chunks[i])], dtype=torch.int64, device=self.device)
        h0 = ops.stack_layers([yb[t_idx, r_idx] for yb in p['ybufs']])
        c0 = ops.stack_layers([cb[t_idx, r_idx] for cb in p['cbufs']]) if pol.cell == "lstm" else None
        old_values = chunked(p['values_lr']).contiguous()               # the critic at prep time (value clipping)
        old_log_probs = None if p['old_log_probs'] is None else chunked(p['old_log_probs']).contiguous()
        t_rows = p.get('teacher_log_probs')
        teacher_log_probs = None if t_rows is None else chunked(t_rows).contiguous()
        return ExperienceBatch(obs, masks, actions, old_logp, adv, ret, h0, c0, old_values=old_values, valid=p['valid'],
                               old_log_probs=old_log_probs, teacher_log_probs=teacher_log_probs)

    def _packed_batch(self, p, lay):
        """The packed ``ExperienceBatch`` of ``pack_layout`` from the prepared ``[L_max, R, ...]`` tensors: every field is
        one token gather per index (``dc_gather_columns`` over ``[1, L_max * R, ...]`` views, and over the rollout-major
        advantages and returns), so the assembly is a handful of launches whatever the number of sequences.  A padding token
        reads a padded row of a rollout with a tail: zeros, zero advantage and return, like the padding of the unpacked
        batch."""
        S, pol, dev = self.seq_len, self.policy_base, self.device
        Ls, Lps, Lmax = p['Ls'], p['Lps'], p['Lmax']
        R = len(Ls)
        check_reset_slots(lay.reset_slot, lay.K)
        B = lay.B
        real = lay.rollout >= 0
        pad_r = next((i for i, L in enumerate(Ls) if L % S), 0)           # any rollout with a tail has padded rows
        src_r = np.where(real, lay.rollout, pad_r)
        src_t = np.where(real, lay.step, Ls[pad_r])
        base = np.concatenate([[0], np.cumsum(Lps)[:-1]]).astype(np.int64)
        idx_tm = (src_t * R + src_r).reshape(-1)                          # rows of the time-major [L_max, R] tensors
        # rows of the rollout-major scan outputs
        idx_rm = np.where(real, packed_rows(lay, Lps), base[pad_r] + Ls[pad_r]).reshape(-1)

        def gather(tensors, index, n_src):
            outs = [torch.empty((S, B) + tuple(t.shape[2:]) if t.dim() >= 2 else (S, B), dtype=t.dtype, device=dev)
                    for t in tensors]
            ops.gather_columns([(t.contiguous().view((1, n_src) + tuple(t.shape[2:] if t.dim() >= 2 else ())),
                                 o.view((1, S * B) + tuple(o.shape[2:]))) for t, o in zip(tensors, outs)], index)
            return outs
        keys_o, keys_h = list(p['obs']), list(p['masks'])
        kl_rows = [] if p['old_log_probs'] is None else [p['old_log_probs']]
        t_rows = [] if p.get('teacher_log_probs') is None else [p['teacher_log_probs']]
        tm = [p['obs'][k] for k in keys_o] + [p['masks'][k] for k in keys_h] + [p['actions'][k] for k in keys_h] + \
            [p['old_logp'], p['values_lr']] + kl_rows + t_rows
        g = gather(tm, idx_tm, Lmax * R)
        obs = dict(zip(keys_o, g[:len(keys_o)]))
        masks = dict(zip(keys_h, g[len(keys_o):len(keys_o) + len(keys_h)]))
        actions = dict(zip(keys_h, g[len(keys_o) + len(keys_h):len(keys_o) + 2 * len(keys_h)]))
        n_tm = len(keys_o) + 2 * len(keys_h)
        old_logp, old_values = g[n_tm], g[n_tm + 1]
        old_log_probs = g[n_tm + 2] if kl_rows else None
        teacher_log_probs = g[n_tm + 2 + len(kl_rows)] if t_rows else None
        # the K returns of a row gathered as one [rows, 1, K] row of K elements
        ret_c = p['ret_c'] if p['ret_c'].dim() == 1 else p['ret_c'].unsqueeze(1)
        adv, ret = gather([p['adv_c'], ret_c], idx_rm, int(sum(Lps)))
        # the host layout goes up in one pinned copy: valid, the reset slots and the state-buffer coordinates
        t_rs, c_rs = np.nonzero(lay.reset_slot >= 0)
        meta = np.concatenate([real.reshape(-1), lay.reset_slot.reshape(-1), lay.h0_step, lay.h0_rollout,
                               lay.reset_slot[t_rs, c_rs], c_rs, lay.step[t_rs, c_rs], lay.rollout[t_rs, c_rs]]).astype(np.int64)
        meta = torch.from_numpy(meta).pin_memory().to(dev, non_blocking=True)
        n, o = S * B, 2 * S * B
        valid = meta[:n].view(S, B).bool()
        reset_slot = meta[n:o].view(S, B).to(torch.int32)
        h0_t, h0_r = meta[o:o + B], meta[o + B:o + 2 * B]
        m = len(t_rs)
        rk, rc, rt, rr = (meta[o + 2 * B + j * m:o + 2 * B + (j + 1) * m] for j in range(4))
        lstm = pol.cell == "lstm"
        h0 = ops.stack_layers([yb[h0_t, h0_r] for yb in p['ybufs']])
        c0 = ops.stack_layers([cb[h0_t, h0_r] for cb in p['cbufs']]) if lstm else None

        def table(bufs):                      # [K, B, L*H]: row (k, c) = every layer's state at the k-th reset of column c
            tab = torch.zeros((lay.K, B, pol.num_layers * pol.hidden_size), dtype=torch.float32, device=dev)
            if m:
                tab[rk, rc] = torch.cat([bf[rt, rr] for bf in bufs], dim=1)
            return tab
        return ExperienceBatch(obs, masks, actions, old_logp, adv, ret, h0, c0, old_values=old_values, valid=valid,
                               reset_slot=reset_slot, reset_h=table(p['ybufs']), reset_c=table(p['cbufs']) if lstm else None,
                               old_log_probs=old_log_probs, teacher_log_probs=teacher_log_probs)

    @staticmethod
    def list_of_dicts_to_dict_of_lists(x):
        return {k: torch.stack([torch.as_tensor(d[k]) for d in x]) for k in x[0]}

    # -- one optimizer step (:581-689) -------------------------------------------------------------
    def train(self, experiences):
        """One PPO/Adam step on a list of ``Sequence`` (or an ``ExperienceBatch``).

        Returns the reference's three dicts: losses, per-head entropies, grad norms (CPU scalars).  The PPO diagnostics of
        the step (approximate KL, clip fraction, explained variance) are left in ``last_ppo_stats``.
        A device-resident batch of a shape seen before is replayed from a CUDA graph of the whole step (forward, loss,
        backward, all-reduce, finish: ~80 kernel launches -> one graph launch); batches still in flight from the host
        (``prefetch``) run the same kernels launch by launch so that the upload overlaps them.  Either way the step uses
        the current ``learning_rate``, ``e_clip``, ``entropy_coef``, ``vf_coef``, ``MAX_GRAD_NORM`` and ``value_clip``
        (and under KL control ``kl_coef`` and ``kl_stop``, with a teacher ``teacher_coef``, with dual clip ``dual_clip``).
        A step that ``kl_stop`` skips returns normally, with the parameters, Adam moments and step counters unchanged;
        ``last_ppo_stats['kl_skipped']`` is then 1.
        """
        if isinstance(experiences, ExperienceBatch):
            batch = experiences if experiences.advantages.is_cuda else experiences.to(self.device)
        else:
            batch = ExperienceBatch.from_sequences(experiences, self.device)
        if self.value_clip and batch.old_values is None:
            raise ValueError("value_clip=%r needs the critic values of experience prep, and this batch has no old_values"
                             % self.value_clip)
        if self.mask_padding and batch.valid is None:
            raise ValueError("mask_padding=True needs the valid mask of experience prep, and this batch has no valid")
        if not self.kl_control and (self.kl_coef or self.kl_stop is not None):
            raise ValueError("kl_coef=%r / kl_stop=%r: KL control is off for this optimizer (construct it with kl_coef > 0 "
                             "or kl_stop set, so that prep stores the old distribution)" % (self.kl_coef, self.kl_stop))
        if self.kl_control and batch.old_log_probs is None:
            raise ValueError("kl_coef=%r / kl_stop=%r need the log-prob rows of experience prep, and this batch has no "
                             "old_log_probs" % (self.kl_coef, self.kl_stop))
        if self.teacher_model is not None and self.teacher_coef > 0.0 and batch.teacher_log_probs is None:
            raise ValueError("teacher_coef=%r needs the teacher's log-prob rows of experience prep, and this batch has no "
                             "teacher_log_probs" % (self.teacher_coef,))
        if batch.reset_slot is not None and not self.mask_padding:
            raise ValueError("a packed batch (reset_slot) trains only with mask_padding=True: its padding carries no "
                             "advantages or value targets")
        if self._dual_clip_on != (self.dual_clip is not None):
            raise ValueError("dual_clip=%r: dual clip was %s when this optimizer was constructed, and that is fixed (the "
                             "step's loss kernel depends on it)" % (self.dual_clip, "on" if self._dual_clip_on else "off"))
        check_dual_clip(self.dual_clip)
        t_enter = time.perf_counter()
        self._upload_hparams()
        slot = batch._slot
        if slot is not None:                       # uploaded by prefetch() straight into a graph's static input buffers
            torch.cuda.current_stream().wait_event(slot["ready"])
        # a batch whose uploads are still in flight runs launch by launch, so that each kernel waits only for its own inputs
        replay = slot is not None or (self.use_cuda_graph and not batch._ready)
        if replay and not ops.PROFILE.enabled:
            out, metrics = self._replay_step(batch)
        else:
            out, metrics = self._enqueue_step(batch)
        if slot is not None:
            slot["done"].record()
            slot["busy"] = False
        host = self._host_result
        host[:_lib.LOSS_SLOTS].copy_(out, non_blocking=True)
        host[_lib.LOSS_SLOTS:].copy_(self._result_dev, non_blocking=True)        # metrics, then the PPO diagnostics
        self.host_enqueue_s = time.perf_counter() - t_enter   # host time to launch the step (the GPU runs behind it)
        torch.cuda.current_stream().synchronize()      # the step's single host sync (result read-back)
        res = host.clone()
        keys = ops.HEAD_KEYS
        self.last_ppo_stats = self._ppo_stats_dict(res[_lib.LOSS_SLOTS + self._n_metrics:].tolist(),
                                                   joint=self.policy_ratio == 'joint', kl=self.kl_control,
                                                   bc=self.objective == 'bc')
        if self.value_heads is not None:    # per head: its share of the value loss and its explained variance
            hs = res[_lib.LOSS_SLOTS + self._n_metrics + _lib.PPO_STATS_SLOTS:].tolist()
            for k, name in enumerate(self.value_heads.names):
                self.last_ppo_stats['loss/value/' + name] = hs[k]
                self.last_ppo_stats['explained_variance/' + name] = hs[_lib.VALUE_HEADS_MAX + k]
        if self.kl_control:             # the all-ranks KL of the finish, and whether it skipped the update
            self.last_ppo_stats['kl_all_ranks'] = float(res[_lib.LOSS_SLOTS + 4])
            self.last_ppo_stats['kl_skipped'] = float(res[_lib.LOSS_SLOTS + 5])
        if self._teacher_step(batch):   # the KL to the teacher (this rank), per head, and the loss term lambda KL_T
            ts = res[_lib.LOSS_SLOTS + self._dual_clip_off - _lib.TEACHER_STATS_SLOTS:].tolist()
            self.last_ppo_stats['teacher/kl'] = ts[0]
            for h, k in enumerate(keys):
                self.last_ppo_stats['teacher/kl/' + k] = ts[1 + h]
            self.last_ppo_stats['loss/teacher'] = ts[6]
        if self.objective == 'bc':      # the NLL of the demonstrations (this rank) and the accuracy of the arg-max, per head
            bs = res[_lib.LOSS_SLOTS + self._dual_clip_off - _lib.BC_STATS_SLOTS:].tolist()
            self.last_bc_stats = {'nll': bs[0], 'accuracy': bs[1 + len(keys)]}
            for h, k in enumerate(keys):
                self.last_bc_stats['nll/' + k] = bs[1 + h]
                self.last_bc_stats['accuracy/' + k] = bs[2 + len(keys) + h]
            self.last_ppo_stats.update({'bc/' + k: v for k, v in self.last_bc_stats.items() if k != 'nll'})
        if self._dual_clip_on:          # the shares of the rows where the floor binds (this rank): mean, per head, joint
            ds = res[_lib.LOSS_SLOTS + self._dual_clip_off:].tolist()
            self.last_dual_clip_stats = {'fraction': ds[0]}
            for h, k in enumerate(keys):
                self.last_dual_clip_stats['fraction/' + k] = ds[1 + h]
            if self.policy_ratio == 'joint':
                self.last_dual_clip_stats['fraction/joint'] = ds[1 + len(keys)]
            self.last_ppo_stats.update({'dual_clip_' + k: v for k, v in self.last_dual_clip_stats.items()})
        if res[_lib.LOSS_SLOTS + 3] != 0:               # :667-669, :678-679 (parameters were left untouched)
            if math.isnan(float(res[0])):
                raise ValueError('loss={}, policy_loss={}, entropy_loss={}, value_loss={}'.format(
                    float(res[0]), float(res[1]), float(res[2]), float(res[3])))
            raise ValueError('grad_norm={}'.format(float(res[_lib.LOSS_SLOTS])))
        losses = {'loss': res[0], 'policy_loss': res[1], 'entropy_loss': res[2], 'value_loss': res[3]}
        entropies = {k: res[4 + h] for h, k in enumerate(keys)}
        return losses, entropies, {'unclipped': res[_lib.LOSS_SLOTS], 'clipped': res[_lib.LOSS_SLOTS + 1]}

    @property
    def last_vtrace_stats(self):
        """Diagnostics of the last experience prep with ``advantage_estimator='vtrace'`` (None before one), over the rollouts'
        real steps (padding excluded): ``mean_log_rho`` (the mean log importance weight, log pi/mu), ``mean_clipped_rho``
        (the mean truncated weight), ``rho_clip_fraction`` and ``c_clip_fraction`` (the share of steps whose weight exceeds
        ``vtrace_rho_clip`` / ``vtrace_c_clip``).  Read back from the device, which waits for the prep, when accessed."""
        if self._vtrace_seg_stats is None:
            return None
        s = self._vtrace_seg_stats.sum(dim=0).tolist()
        n = max(s[0], 1.0)
        return {'mean_log_rho': s[1] / n, 'mean_clipped_rho': s[2] / n, 'rho_clip_fraction': s[3] / n,
                'c_clip_fraction': s[4] / n}

    @property
    def last_upgo_stats(self):
        """Diagnostics of the last experience prep that ran with ``upgo_coef > 0`` (None before one, or when the last prep
        ran without), over the rollouts' real steps (padding excluded): ``through_fraction`` (the share of steps whose
        upgoing return went on through the next step's, because that step's TD error was >= 0) and ``mean_advantage`` (the
        mean UPGO advantage A^U, before the coefficient).  Read back from the device, which waits for the prep."""
        if self._upgo_prep is None:
            return None
        s = self._upgo_prep[1].sum(dim=0).tolist()
        n = max(s[0], 1.0)
        return {'through_fraction': s[1] / n, 'mean_advantage': s[2] / n}

    def _upgo_coef_now(self):
        """``upgo_coef`` as prep and the advantage refresh read it, checked again: it may be assigned at any time."""
        check_upgo_coef(self.upgo_coef, self.value_heads)
        return float(self.upgo_coef)

    def _value_norm_moments(self):
        return value_norm_moments(self._value_norm, self.VALUE_NORM_MIN_STD)

    @property
    def value_norm_stats(self):
        """With ``value_norm``: ``{'mean': mu, 'std': sigma, 'weight': w}`` of the value statistics the next step trains
        under (w = 0: no update yet, identity); None when the feature is off."""
        if not self.value_norm:
            return None
        mu, sigma = self._value_norm_moments()
        return {'mean': mu, 'std': sigma, 'weight': self._value_norm[2]}

    def _update_value_norm(self, ret, valid):
        """The end of experience prep under ``value_norm``: the batch's (n, sum R, sum R^2) over the tokens the value loss
        averages over (``valid`` rows, or all), summed over the ranks with one all-reduce when data-parallel (a collective:
        every rank's prep must reach it), one host sync, the statistics update, and the POP rescale of the value head."""
        st = ops.value_norm_stats(ret, valid)
        if is_distributed():
            dist.all_reduce(st)
        n, s1, s2 = st.tolist()
        old = self._value_norm_moments()
        self._value_norm = value_norm_update(self._value_norm, n, s1, s2, self.value_norm_decay)
        new = self._value_norm_moments()
        if new != old:
            head = self.policy_base.affine_value
            ops.value_head_rescale(head.weight.data, head.bias.data, old, new)

    @staticmethod
    def _ppo_stats_dict(st, joint=False, kl=False, bc=False):
        if bc:                      # no ratio, so no approximate KL or clip fraction
            return {'explained_variance': st[_lib.STAT_EXPLAINED_VAR]}
        out = {'approx_kl': st[_lib.STAT_APPROX_KL], 'clip_fraction': st[_lib.STAT_CLIP_FRACTION]}
        for h, k in enumerate(ops.HEAD_KEYS):
            out['approx_kl/' + k] = st[_lib.STAT_APPROX_KL + 1 + h]
            out['clip_fraction/' + k] = st[_lib.STAT_CLIP_FRACTION + 1 + h]
        out['explained_variance'] = st[_lib.STAT_EXPLAINED_VAR]
        if joint:                   # the ratio the joint objective clips, over the steps with an action
            out['approx_kl/joint'] = st[_lib.STAT_JOINT_APPROX_KL]
            out['clip_fraction/joint'] = st[_lib.STAT_JOINT_CLIP_FRACTION]
        if kl:                      # the exact KL to the prep-time policy (this rank), per head, and the penalty beta KL
            out['kl'] = st[_lib.STAT_KL]
            for h, k in enumerate(ops.HEAD_KEYS):
                out['kl/' + k] = st[_lib.STAT_KL + 1 + h]
            out['kl_penalty'] = st[_lib.STAT_KL_PENALTY]
        return out

    def _upload_hparams(self):
        """Writes the current hyper-parameters into the device block the step's kernels read: one asynchronous copy on the
        current stream, before the step is launched or replayed (never inside a captured graph), and only when a value
        changed (with the value head's has-gradient flag, which follows vf_coef).  The pinned source is free to rewrite: the
        previous step's copy completed before that step's result was read back."""
        # value_norm: the statistics of the last prep (mu, sigma), which the loss normalises the raw targets with; off: 0, 0
        mu, sigma = self._value_norm_moments() if self.value_norm else (0.0, 0.0)
        # KL control: the penalty's beta and the early-stop limit (None: 0, no limit)
        # teacher: its coefficient, the double after the blocks (_teacher_coef_dev); dual clip: c, the double after that
        vals = (float(self.learning_rate), float(self.e_clip), float(self.entropy_coef), float(self.vf_coef),
                float(self.MAX_GRAD_NORM), float(self.value_clip or 0.0), mu, sigma, float(self.kl_coef),
                float(self.kl_stop or 0.0)) + ((float(self.teacher_coef),) if self.teacher_model is not None else ()) \
            + ((float(self.dual_clip),) if self._dual_clip_on else ())
        if vals == self._hparams_uploaded:
            return
        h = self._hparams_host.numpy()
        for slot, v in zip((_lib.HP_LR, _lib.HP_E_CLIP, _lib.HP_ENTROPY_COEF, _lib.HP_VF_COEF, _lib.HP_MAX_GRAD_NORM,
                            _lib.HP_VALUE_CLIP, _lib.HP_VALUE_NORM_MEAN, _lib.HP_VALUE_NORM_STD, _lib.HP_KL_COEF,
                            _lib.HP_KL_STOP), vals):
            h[slot] = v
        if self.value_heads is not None:    # the PPO loss's block: the same, its value term off
            self._hparams_host_all[1].copy_(self._hparams_host_all[0])
            hp = self._hparams_host_all[1].numpy()
            hp[_lib.HP_VF_COEF] = hp[_lib.HP_VALUE_CLIP] = 0.0
        if self.teacher_model is not None:
            self._teacher_coef_host[0] = float(self.teacher_coef)
        if self._dual_clip_on:
            self._dual_clip_host[0] = float(self.dual_clip)
        self._hparams_dev_flat.copy_(self._hparams_host_flat, non_blocking=True)
        # the value head has a gradient only while the value loss is on (optimizer.py:660-662): with vf_coef = 0 the
        # gradient finish skips its tensors (no Adam step, no share of the mean grad norm), like the reference's .grad = None
        self._n_actions[VALUE_SLOT:VALUE_SLOT + 1].fill_(1 if self.vf_coef > 0 else 0)
        self._hparams_uploaded = vals

    def _teacher_step(self, batch):
        """Whether a step on ``batch`` runs the teacher term: a teacher was given and the batch carries its rows (a batch
        prepared after the anneal retired it carries none, and runs the step without the term)."""
        return self.teacher_model is not None and batch.teacher_log_probs is not None

    def _enqueue_step(self, batch):
        """Launches one optimizer step (:581-689) on the current stream; returns the device result vectors (loss slots, metrics)."""
        keys = ops.HEAD_KEYS
        self.flat.zero_grad_detached()                                    # :671 (grads gathered into the flat buffer below)
        hidden = (batch.h0, batch.c0) if self.policy_base.cell == "lstm" else batch.h0
        batch.wait(batch.observations['env'], batch.h0, batch.c0, batch.reset_slot, batch.reset_h, batch.reset_c)
        # :619 on the module itself: the data-parallel wrapper's hook-driven reduction stays idle, the step reduces below
        # the attention layer and the target-unit head run only on the tokens whose target-unit row the loss reads (their
        # mask / action uploads are waited for right before the head), unless the batch is so small that the step is bound by
        # launches, which the row list adds
        active = None
        if batch.seq_len * batch.batch_size >= TARGET_ROWS_MIN_TOKENS:
            active = (batch.masks['target_unit'], batch.actions['target_unit'])
        packed, target_unit = self.policy_base._train_forward(batch.observations, hidden, wait=batch.wait, reset=batch.reset(),
                                                              active=active)
        valid = batch.valid if self.mask_padding else None
        old_log_probs = batch.old_log_probs if self.kl_control else None
        teacher_log_probs = batch.teacher_log_probs if self._teacher_step(batch) else None
        batch.wait(batch.old_logp, batch.advantages, batch.returns, batch.old_values, valid, old_log_probs,
                   teacher_log_probs, *batch.masks.values(), *batch.actions.values(), *batch.observations.values())
        # e_clip / entropy_coef / vf_coef / value_clip are read from the device block (_upload_hparams); padded tokens
        # (valid = False) count for nothing under mask_padding; the policy ratio is fixed per optimizer, so a captured
        # graph of the step keeps it
        heads = self.value_heads is not None
        # value heads: the PPO loss runs with its value term off (_hparams_dev_ppo); the value target it is handed then
        # feeds only an explained variance that dc_value_heads_loss overwrites, so the advantages stand in for it
        # teacher: the KL term to its rows with the coefficient after the hyper-parameter blocks (_upload_hparams)
        # bc: the NLL of the demonstrated actions in place of the surrogate (old_logp is not read)
        # dual clip: the floor c A under negative-advantage surrogates, c after the teacher's coefficient (_upload_hparams)
        bc = self.objective == 'bc'
        out, n_actions, d_packed, d_tu = ops.ppo_loss_packed(
            packed, target_unit, [batch.masks[k] for k in keys], [batch.actions[k] for k in keys],
            batch.old_logp, batch.advantages, batch.advantages if heads else batch.returns, self.e_clip,
            self.entropy_coef, self.vf_coef, hparams=self._hparams_dev_ppo, old_value=None if heads else batch.old_values,
            stats=self._ppo_stats, valid=valid, joint=self.policy_ratio == 'joint', old_log_probs=old_log_probs,
            kl_out=self.flat.kl_tail, teacher_log_probs=teacher_log_probs,
            teacher_coef=self._teacher_coef_dev if teacher_log_probs is not None else None,
            teacher_stats=self._teacher_stats if teacher_log_probs is not None else None, bc=bc,
            bc_stats=self._bc_stats, dual_clip=self._dual_clip_dev if self._dual_clip_on else None,
            dual_clip_stats=self._dual_clip_stats)[:4]
        if heads:
            ops.value_heads_loss(packed, d_packed, batch.returns, self._hparams_dev, out, self._value_head_stats,
                                 old_value=batch.old_values, valid=valid, stats=self._ppo_stats)
        self._n_actions[:5].copy_(n_actions)
        torch.autograd.backward([packed, target_unit], [d_packed, d_tu])                                # :672
        # drop every reference into this step's autograd graph before the gradient finish: it holds the saved activations
        del packed, target_unit, d_packed, d_tu
        self.flat.gather_grads()
        # distributed.py:29-57 -> flags + ONE all-reduce; divide fused into the finish kernel
        ops.grad_flags(self.flat.grad_full, self.flat.total, self.flat.seg_head, self._n_actions)
        if self.policy is not self.policy_base:
            self.policy.allreduce_gradients(divide=False, flags_ready=True)
        ops.grad_finish(self.flat.param, self.flat.grad_full, self.exp_avg, self.exp_avg_sq, self.adam_steps,
                        self.flat.seg_lo, self.flat.seg_hi, self.flat.seg_head, self.flat.total, self.learning_rate, self.ADAM_BETAS,
                        self.ADAM_EPS, self.MAX_GRAD_NORM, out, self._metrics, self._finish_ws,
                        hparams=self._hparams_dev, kl=self.kl_control)                              # :674-681
        return out, self._metrics

    # -- CUDA graph of the step ----------------------------------------------------------------------
    def _replay_step(self, batch):
        """Replays the captured step for this batch shape (captures it the second time the shape is seen: the first call of
        a shape runs launch by launch, which also warms every kernel up).  Inputs are copied into the graph's static
        buffers (device to device) -- or, for a batch that ``prefetch`` uploaded into an input slot (the graph's static
        inputs are then the batch itself), are already there; parameters, gradients, Adam state and step counters are the
        same device buffers the eager path uses, so eager and graphed steps can be mixed freely."""
        key = batch.graph_key() if batch._slot is None else batch.graph_key() + (id(batch._slot),)
        entry = self._graphs.get(key)
        if entry == "seen":
            for k in [k for k, v in self._graphs.items() if isinstance(v, _CapturedStep)][:-1]:
                del self._graphs[k]            # at most two captured shapes alive: a graph pins its step's activations
            entry = self._graphs[key] = self._capture_step(batch)
        if not isinstance(entry, _CapturedStep):   # first sight of this shape, or its capture failed
            self._graphs.setdefault(key, "seen")
            return self._enqueue_step(batch)
        if entry.static is not batch:
            torch._foreach_copy_([v for _, _, v in entry.static.tensors()], [v for _, _, v in batch.tensors()])
        entry.graph.replay()
        return entry.out, self._metrics

    def _capture_step(self, batch):
        static = batch if batch._slot is not None else batch.map(lambda v: v.detach().clone())
        graph = torch.cuda.CUDAGraph()
        # A garbage collection during the capture would free unreachable objects -- among them the captured graphs of an
        # optimizer nobody references any more -- and destroying a graph is not permitted while a stream is capturing: it
        # invalidates this capture.  So collect first and keep the cyclic collector off until the capture has ended.
        gc.collect()
        gc_was_enabled = gc.isenabled()
        gc.disable()
        try:
            torch.cuda.synchronize()
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                out, _ = self._enqueue_step(static)
        except Exception as e:                      # same kernels either way: fall back to launch-by-launch for this shape
            logger.warning('CUDA graph capture of the step failed (%s); this shape keeps running launch by launch', e)
            torch.cuda.synchronize()
            self.flat.rebind()
            return "eager"
        finally:
            if gc_was_enabled:
                gc.enable()
        return _CapturedStep(static, graph, out)

    def prefetch(self, experiences):
        """Starts the asynchronous upload of a pinned-host ``ExperienceBatch`` on the copy stream and returns the device batch
        at once (every tensor carries its own ready-event; ``train`` waits per tensor at first use).  Called while the previous
        step is still computing, it hides the PCIe transfer behind that step (double buffering) -- raw rollout data does not
        depend on the weights, so an optimizer fed from the experience queue can always upload one batch ahead."""
        if not isinstance(experiences, ExperienceBatch):
            experiences = ExperienceBatch.from_sequences(experiences, torch.device("cpu")).pin_memory()
        if experiences.advantages.is_cuda:
            return experiences
        if self.use_cuda_graph and experiences.advantages.is_pinned():
            staged = self._stage_into_slot(experiences)
            if staged is not None:
                return staged
        return experiences.to(self.device, prefetch=True)

    def _stage_into_slot(self, host):
        """Double-buffered graph inputs: every batch shape owns TWO sets of static device input buffers; ``prefetch`` copies
        the pinned host batch into the set that is not being trained on (copy stream, behind the replay that last read that
        set) and ``train`` replays the graph captured over that set -- so the upload of step k+1 overlaps the graph of step k.
        Returns None (caller falls back to per-tensor uploads) when both sets are still waiting to be trained on."""
        slots = self._input_slots.setdefault(host.graph_key(), [])
        slot = next((sl for sl in slots if not sl["busy"]), None)
        if slot is None:
            if len(slots) >= 2:
                return None
            dev_batch = host.map(lambda v: torch.empty(v.shape, dtype=v.dtype, device=self.device))
            slot = {"batch": dev_batch, "busy": False, "ready": torch.cuda.Event(), "done": torch.cuda.Event()}
            slot["done"].record()
            dev_batch._slot = slot
            slots.append(slot)
        side = _copy_stream(self.device)
        side.wait_event(slot["done"])                    # the replay that last read these buffers has finished
        with torch.cuda.stream(side):
            dsts = [v for _, _, v in slot["batch"].tensors()]
            srcs = [v for _, _, v in host.tensors()]
            for d, src in zip(dsts, srcs):
                d.copy_(src, non_blocking=True)
            slot["ready"].record(side)
        slot["busy"] = True
        return slot["batch"]

    def mean_gradient_norm(self):
        """Mean per-tensor L2 norm over parameters that got a gradient in the last step (:691-695)."""
        has = self.flat.flags > 0
        norms = torch.stack([self.flat.grad[lo:hi].norm(2) for lo, hi in
                             zip(self.flat.starts, self.flat.ends)])
        return norms[has].mean()

    def train_epochs(self, batch):
        """The PPO epochs of one iteration on ``batch`` (an ``ExperienceBatch``): ``epochs`` passes, each split into
        ``num_minibatches`` minibatches of whole sequences (``minibatch_indices`` with ``minibatch_rng``), one ``train`` step
        per minibatch -- forward, loss (advantages normalised over the minibatch), backward, all-reduce, clip, Adam.  With
        one minibatch every epoch trains on ``batch`` itself, as the reference does (:469).  Returns the per-step lists
        ``(losses, entropies, grad_norms, ppo_stats)``.  Raises ``ValueError`` when the batch has fewer sequences than
        minibatches.  Under ``kl_stop`` the first step whose all-ranks KL exceeds the limit is skipped and ends the
        iteration's updates (the shuffles of the epochs not run are not drawn); its results are the last in the lists, and
        ``last_kl_updates`` holds (updates run, updates skipped).

        With ``recompute_advantages`` every epoch after the first starts with ``_refresh_advantages``, which rewrites
        ``batch.advantages`` and ``batch.returns`` in place; no refresh follows a step that ``kl_stop`` skipped.  The batch
        must then come from ``batch_from_rollouts`` (``ExperienceBatch.refresh``), else ``ValueError`` before any launch.
        With ``recompute_states`` the same epochs start with ``_refresh_states`` instead, which rewrites the batch's
        recurrent start states (and, with ``recompute_advantages``, its advantages and returns from the same forward); the
        batch must carry ``ExperienceBatch.state_refresh``."""
        M = self.num_minibatches
        if batch.batch_size < M:
            raise ValueError("the batch has %d sequences, fewer than num_minibatches=%d" % (batch.batch_size, M))
        refresh = (self.recompute_advantages or self.recompute_states) and self.epochs > 1
        if refresh and self.recompute_advantages and batch.refresh is None:
            raise ValueError("recompute_advantages=True needs the scan inputs of experience prep, and this batch has none "
                             "(ExperienceBatch.refresh): train on a batch from batch_from_rollouts")
        if refresh and self.recompute_states and batch.state_refresh is None:
            raise ValueError("recompute_states=True needs the rollout layout of experience prep, and this batch has none "
                             "(ExperienceBatch.state_refresh): train on a batch from batch_from_rollouts")
        self._state_refresh_sums = []
        if M > 1 and not batch.advantages.is_cuda:
            batch = batch.to(self.device)                  # uploaded once; the minibatches are gathered on the device
        losses, entropies, grad_norms, ppo_stats = [], [], [], []
        stopped = False
        for ep in range(self.epochs):                                      # :469
            self.mq.process_data_events()
            if refresh and ep > 0:
                if self.recompute_states:
                    self._refresh_states(batch)
                else:
                    self._refresh_advantages(batch)
            for idx in minibatch_indices(batch.batch_size, M, self.minibatch_rng):
                loss_d, entropy_d, grad_norm_d = self.train(experiences=batch if M == 1 else batch.gather(idx))
                losses.append(loss_d)
                entropies.append(entropy_d)
                grad_norms.append(grad_norm_d)
                ppo_stats.append(self.last_ppo_stats)
                if self.kl_control and self.last_ppo_stats['kl_skipped']:
                    stopped = True
                    break
            if stopped:
                break
        if self.kl_control:
            run = len(losses) - (1 if stopped else 0)
            self.last_kl_updates = (run, self.epochs * M - run)
        return losses, entropies, grad_norms, ppo_stats

    def _refresh_advantages(self, batch):
        """Recomputes ``batch.advantages`` and ``batch.returns`` in place with the current weights (``recompute_advantages``;
        Andrychowicz et al. 2021, section 3.5): a no-grad training forward over the whole batch gives V for every token
        (denormalised with the current statistics under ``value_norm``) and, for V-trace, the current policy's log-probs of
        the taken actions, the new target; then prep's segmented scan runs again over prep's rollout-major rewards,
        segments and bootstraps, reading and writing the batch's tokens (``ops.gae_scan_indexed`` /
        ``vtrace_scan_indexed``, ``refresh_token_map``).  Rows that prep zeroed are not written.  Everything else in the
        batch -- the old log-probs, the old values, the initial and reset states -- stays as prep made it.

        The forward is the training step's (``Policy._train_forward``: encoder, recurrence with the batch's resets, heads),
        run over blocks of ``max(1, REFRESH_CHUNK_TOKENS // B)`` time steps with the recurrent
        state carried from block to block, so its transient memory is bounded by the block, not by the batch."""
        r, pol, keys = batch.refresh, self.policy_base, ops.HEAD_KEYS
        S, B = batch.seq_len, batch.batch_size
        vtrace = self.advantage_estimator == 'vtrace'
        hidden = (batch.h0, batch.c0) if pol.cell == "lstm" else batch.h0
        reset = batch.reset()
        T = max(1, self.REFRESH_CHUNK_TOKENS // B)
        col = ops.PACK_COLS["value"][0]
        c0, c1 = ops.pack_cols(self.n_value_heads)["value"]
        heads = self.value_heads is not None          # then every head's value, [S, B, K] (K = 1 included)
        values = None if T >= S else torch.empty((S, B) + ((c1 - c0,) if heads else ()), dtype=torch.float32,
                                                  device=self.device)
        target = torch.empty((S * B, 5), dtype=torch.float32, device=self.device) if vtrace else None
        with torch.no_grad():
            for t0 in range(0, S, T):
                t1 = min(S, t0 + T)
                x, unit_embedding = pol._encode(batch.observations['env'][t0:t1],
                                                [batch.observations[k][t0:t1] for k in Policy.INPUT_KEYS[1:]])
                y, hidden = pol._recur(x.contiguous(), hidden, None if reset is None else (reset[0][t0:t1],) + reset[1:])
                packed, target_unit = pol._head_outputs(y, unit_embedding)
                v = packed[..., c0:c1] if heads else packed[..., col]
                if values is None:                  # one block: the scan reads the value column where the GEMM wrote it
                    values = v
                else:
                    values[t0:t1] = v
                if vtrace:
                    logits = [target_unit if k == "target_unit" else packed[..., ops.PACK_COLS[k][0]:ops.PACK_COLS[k][1]]
                              for k in keys]
                    target[t0 * B:t1 * B] = ops.selected_logp(logits, [batch.masks[k][t0:t1] for k in keys],
                                                              [batch.actions[k][t0:t1] for k in keys])
                del x, unit_embedding, y, packed, target_unit
            if self.value_norm:
                values = ops.value_denorm(values, *self._value_norm_moments())
            self._rescan(batch, values, target, r.boot)

    def _rescan(self, batch, values, target, boot):
        """Prep's segmented GAE or V-trace scan over prep's rollout-major rewards and segments, reading the raw values
        (and for V-trace the target log-probs ``[S * B, 5]``) at the batch's tokens and writing ``batch.advantages`` /
        ``batch.returns`` there (``ops.gae_scan_indexed`` / ``vtrace_scan_indexed``), ending the segments on ``boot``;
        with ``upgo_coef > 0`` then prep's UPGO term over the same operands (``ops.upgo_scan_indexed``)."""
        r = batch.refresh
        if self.value_heads is not None:
            vh = self.value_heads
            ops.gae_scan_heads_indexed(r.rewards, values.reshape(-1, self.n_value_heads), r.tok, r.seg_off,
                                       batch.advantages, batch.returns, vh.group, vh.gammas, self.gae_lambda,
                                       boot_value=boot, boot_reward=boot)
        elif self.advantage_estimator == 'vtrace':
            ops.vtrace_scan_indexed(r.rewards, values, target, r.behaviour_logp, r.tok, r.seg_off, batch.advantages,
                                    batch.returns, self.gamma, self.gae_lambda, self.vtrace_rho_clip, self.vtrace_c_clip,
                                    boot_value=boot, valid_len=r.valid_len)
        else:
            ops.gae_scan_indexed(r.rewards, values, r.tok, r.seg_off, batch.advantages, batch.returns, self.gamma,
                                 self.gae_lambda, boot_value=boot, boot_reward=boot)
        upgo = self._upgo_coef_now()
        if upgo > 0.0:                          # + c A^U, as prep adds it
            ops.upgo_scan_indexed(r.rewards, values, r.tok, r.seg_off, batch.advantages, self.gamma, upgo, boot_value=boot,
                                  logp_target=target, logp_behaviour=r.behaviour_logp, rho_clip=self.vtrace_rho_clip)

    def _refresh_states(self, batch):
        """Recomputes the recurrent states entering the batch's chunks with the current weights (``recompute_states``;
        Kapturowski et al. 2019, section 3): every rollout runs again whole, in sequence, over its padded length, from the
        state prep started it from (zeros or its ``'initial_hidden'``), as experience prep runs it (``_rollout_forward``),
        with the observations gathered from the batch (``ExperienceBatch.state_refresh``, ``state_refresh_layout``; rows the
        batch does not hold are zeros, as in prep).  Every layer's state at each chunk start after a rollout's first is
        written over ``batch.h0`` / ``c0`` or the reset tables, in place (``ops.refresh_states``), and the drift sums go to
        ``last_state_refresh_stats``.  A rollout's first chunk keeps prep's start state.

        With ``recompute_advantages`` the same forward gives the values of every row (denormalised with the current
        statistics under ``value_norm``) and, for V-trace, the current policy's log-probs of the taken actions; a cut
        rollout's V(s_L) is recomputed from the refreshed state after its last step and its extra observation row; then
        prep's scan runs again (``_rescan``).  Everything else in the batch stays as prep made it.

        The forward runs over blocks of ``max(1, REFRESH_CHUNK_TOKENS // R)`` time steps of the ``R`` rollouts, with the
        state carried from block to block, so its transient memory is bounded by the block, not by the batch."""
        st, pol, keys = batch.state_refresh, self.policy_base, ops.HEAD_KEYS
        lay, dev = st.layout, self.device
        R, Lmax = lay.R, lay.L_max
        lstm = pol.cell == "lstm"
        adv = self.recompute_advantages
        vtrace = adv and self.advantage_estimator == 'vtrace'
        cut = adv and st.cut_len is not None
        T = max(1, self.REFRESH_CHUNK_TOKENS // R)
        if st.h0 is not None:
            h, c = st.h0, st.c0
        else:
            h = torch.zeros((pol.num_layers, R, pol.hidden_size), dtype=torch.float32, device=dev)
            c = torch.zeros_like(h) if lstm else None
        acc = torch.zeros(2, dtype=torch.float64, device=dev)
        values = torch.empty((Lmax, R) + self._vh_shape, dtype=torch.float32, device=dev) if adv else None
        target = torch.empty((Lmax * R, 5), dtype=torch.float32, device=dev) if vtrace else None
        if cut:                                # the state after each cut rollout's last step, taken from its block
            hb = torch.empty((pol.num_layers, st.cut_len.size, pol.hidden_size), dtype=torch.float32, device=dev)
            cb = torch.empty_like(hb) if lstm else None
            cut_block = (st.cut_len - 1) // T
        srcs = dict(batch.observations)
        if vtrace:
            srcs.update({('m', k): batch.masks[k] for k in keys})
            srcs.update({('a', k): batch.actions[k] for k in keys})
        with torch.no_grad():
            for blk, t0 in enumerate(range(0, Lmax, T)):
                t1 = min(Lmax, t0 + T)
                n = t1 - t0
                ins = {k: torch.empty((n, R) + tuple(v.shape[2:]), dtype=v.dtype, device=dev) for k, v in srcs.items()}
                ops.gather_columns_fill([(v.view((1, -1) + tuple(v.shape[2:])), ins[k].view((1, n * R) + tuple(v.shape[2:])))
                                         for k, v in srcs.items()], st.obs_token[t0 * R:t1 * R])
                ybufs, cbufs, logits, v = self._rollout_forward(ins, h, c)
                lo, hi = np.searchsorted(lay.step, [t0, t1])
                if hi > lo:
                    ops.refresh_states(ybufs, cbufs if lstm else None, t0, st.step[lo:hi], st.rollout[lo:hi],
                                       st.slot[lo:hi], batch.h0, batch.c0, batch.reset_h, batch.reset_c, acc)
                if adv:
                    values[t0:t1] = v.reshape((n, R) + self._vh_shape)
                if vtrace:
                    target[t0 * R:t1 * R] = ops.selected_logp([logits[k] for k in keys], [ins[('m', k)] for k in keys],
                                                              [ins[('a', k)] for k in keys])
                if cut and (cut_block == blk).any():
                    sel = np.flatnonzero(cut_block == blk)
                    ij = torch.from_numpy(np.stack([st.cut_len[sel] - t0, st.cut_rollout[sel], sel])).to(dev)
                    for k in range(pol.num_layers):
                        hb[k, ij[2]] = ybufs[k][ij[0], ij[1]]
                        if lstm:
                            cb[k, ij[2]] = cbufs[k][ij[0], ij[1]]
                h = ops.stack_layers([yb[n] for yb in ybufs])
                c = ops.stack_layers([cf[n] for cf in cbufs]) if lstm else None
                del ins, ybufs, cbufs, logits, v
            self._state_refresh_sums.append((acc, int(lay.step.size)))
            if not adv:
                return
            vn = self._value_norm_moments() if self.value_norm else None
            boot = batch.refresh.boot
            if cut:                            # V(s_L) from the refreshed state after the last step
                bootstrap = self._rollout_forward(st.obs_next, hb, cb)[3].reshape((-1,) + self._vh_shape)
                if vn is not None:
                    bootstrap = ops.value_denorm(bootstrap, *vn)
                boot = torch.cat([bootstrap.new_zeros((1,) + self._vh_shape), bootstrap])[st.boot_slot]
            if vn is not None:
                values = ops.value_denorm(values, *vn)
            vals_b = ops.gather_rows_fill([values.reshape((-1,) + self._vh_shape)], st.token_row)[0]
            target_b = ops.gather_rows_fill([target], st.token_row)[0] if vtrace else None
            self._rescan(batch, vals_b, target_b, boot)

    @property
    def last_state_refresh_stats(self):
        """The last state refresh of ``train_epochs`` (``recompute_states``): ``{'drift': sqrt(sum (new - old)^2 /
        sum old^2), 'states': n}`` over the ``n`` (rollout, chunk start) states it replaced, every layer's h and, for the
        LSTM, c, summed in float64 in a fixed order (bitwise reproducible; 0 when nothing was replaced).  None before the
        first.  Reading it waits for the device."""
        if not self._state_refresh_sums:
            return None
        acc, n = self._state_refresh_sums[-1]
        return {'drift': _drift(*acc.tolist()), 'states': n}

    # -- iteration driver (:436-579) ----------------------------------------------------------------
    def run(self):
        for it in range(self.iteration_start, self.iterations):
            self.run_iteration(it)

    def _pulled_sequences(self, rollout_lens, n_seq):
        """The training sequences of the rollouts pulled so far (``rollout_lens``, the last one just pulled; ``n_seq`` the
        count before it): the reference's ``ceil(L / seq_len)`` per rollout, or with ``pack_sequences`` the columns of the
        packed layout -- computed only once the unpacked count reaches ``min_seq_per_epoch``, as it can only be smaller."""
        S = self.seq_len
        if not self.pack_sequences:
            return n_seq + (rollout_lens[-1] + S - 1) // S
        unpacked = sequence_count(rollout_lens, S)
        return unpacked if unpacked < self.min_seq_per_epoch else sequence_count(rollout_lens, S, pack=True)

    def teacher_anneal(self):
        """With ``teacher_anneal_iterations`` N: sets ``teacher_coef`` to the constructor's value times max(0, 1 - n / N),
        n = ``teacher_iterations``, and retires the teacher once that is 0.  ``run_iteration`` calls it first."""
        if self.teacher_model is None or self.teacher_anneal_iterations is None:
            return
        self.teacher_coef = self._teacher_coef0 * max(0.0, 1.0 - self.teacher_iterations / self.teacher_anneal_iterations)
        if self.teacher_coef == 0.0:
            self._retire_teacher()

    def run_iteration(self, it):
        logger.info('iteration {}/{}'.format(it, self.iterations))
        self.teacher_anneal()
        teacher_on = self.teacher is not None
        experiences, subrewards, rollout_lens, weight_ages = [], [], [], []
        start_xp = time.time()
        xp_waits = 0
        # The reference pulls and prepares rollouts one at a time until it holds min_seq_per_epoch sequences (:448-466).  The
        # number of sequences a rollout yields is known from its length alone, so the SAME rollouts are pulled here first and
        # then prepared together in one batched pass (experiences_from_rollouts).  With pack_sequences the count is that of
        # the packed layout, so every rank still holds at least min_seq_per_epoch sequences.
        rollouts, n_seq = [], 0
        while n_seq < self.min_seq_per_epoch:                             # :448
            start_xp_wait = time.time()
            rollout, rollout_subrewards, rollout_len, weight_version, _ = self._next_rollout()
            xp_waits += time.time() - start_xp_wait
            rollouts.append(rollout)
            subrewards.append(rollout_subrewards)
            rollout_lens.append(rollout_len)
            weight_ages.append(it - weight_version)
            n_seq = self._pulled_sequences(rollout_lens, n_seq)
        batch = self.batch_from_rollouts(rollouts)                        # prepared + stacked once, reused by every epoch
        time_xp = time.time() - start_xp
        # a stream of rollouts gives every iteration its own batch size: capturing a graph per shape would cost more than the
        # `epochs` replays return, so the graph path is used only while consecutive iterations keep the same shape.  The
        # minibatch shapes follow from (S, B, num_minibatches): at most two, ceil and floor, and _replay_step keeps two
        # captured graphs alive, so the same rule serves minibatches
        shape = (batch.seq_len, batch.batch_size)
        graph_setting, self.use_cuda_graph = self.use_cuda_graph, self.use_cuda_graph and shape == self._last_iteration_shape
        self._last_iteration_shape = shape

        start_optimizing = time.time()
        try:
            losses, entropies, grad_norms, ppo_stats = self.train_epochs(batch)
        finally:
            self.use_cuda_graph = graph_setting
        time_optimizing = time.time() - start_optimizing

        losses = self.list_of_dicts_to_dict_of_lists(losses)
        entropies = self.list_of_dicts_to_dict_of_lists(entropies)
        grad_norms = self.list_of_dicts_to_dict_of_lists(grad_norms)
        n_steps = batch.batch_size * self.seq_len                          # :486 (len(experiences) * seq_len)
        subrewards_per_sec = np.stack(subrewards) / n_steps * Policy.OBSERVATIONS_PER_SECOND
        reward_dict = dict(zip(REWARD_KEYS, subrewards_per_sec.sum(axis=0)))
        time_it = time.time() - self.time_last_it
        self.time_last_it = time.time()
        metrics = {
            self.SPEED_KEY: n_steps / time_it,                             # :501,505 (environment steps per second)
            'reward_per_sec/sum': subrewards_per_sec.sum(axis=1).sum(),
            'loss/sum': losses['loss'].mean(),
            'loss/bc' if self.objective == 'bc' else 'loss/policy': losses['policy_loss'].mean(),
            'loss/entropy': losses['entropy_loss'].mean(),
            'loss/value': losses['value_loss'].mean(),
            'entropy': torch.stack(list(entropies.values())).sum(dim=0).mean(),
            'avg_rollout_len': torch.tensor(rollout_lens, dtype=torch.float32).mean(),
            'avg_weight_age': torch.tensor(weight_ages, dtype=torch.float32).mean(),
            'timing/it': time_it, 'timing/xp_total': time_xp, 'timing/xp_mq_wait': xp_waits,
            'timing/optimizer': time_optimizing,
        }
        for k, v in entropies.items():
            metrics['entropy/{}'.format(k)] = v.mean()
        for k, v in grad_norms.items():
            metrics['grad_norm/{}'.format(k)] = v.mean()
        for k, v in reward_dict.items():
            metrics['reward_per_sec/{}'.format(k)] = v
        # means over the steps.  Under kl_stop they include the step that was skipped: its losses, grad norms and statistics were
        # measured at the parameters it left unchanged, and its KL is the measurement that stopped the iteration
        for k in ppo_stats[0]:
            if k not in ('kl_all_ranks', 'kl_skipped'):     # value heads: 'loss/value/<name>' next to 'loss/value'
                metrics[k if k.startswith(('loss/', 'teacher/', 'bc/')) else 'ppo/{}'.format(k)] = \
                    float(np.mean([s[k] for s in ppo_stats]))
        if self.kl_control:
            # d: the mean over the steps (a skipped one included) of the all-ranks KL, the same number on every rank, so
            # the adaptive coefficient stays identical across ranks
            d = float(np.mean([s['kl_all_ranks'] for s in ppo_stats]))
            metrics['kl/coef'], metrics['kl/all_ranks'] = self.kl_coef, d
            if self.kl_stop is not None:
                metrics['kl/updates_run'], metrics['kl/updates_skipped'] = self.last_kl_updates
            if self.kl_target is not None:                                 # for the next iteration (saved with the model)
                self.kl_coef = kl_coef_update(self.kl_coef, d, self.kl_target)
        if self._dual_clip_on:                                             # the constant this iteration trained with
            metrics['dual_clip/coef'] = self.dual_clip
        if self.teacher_model is not None:                                 # the coefficient this iteration trained with
            metrics['teacher/coef'] = self.teacher_coef
            if teacher_on:
                self.teacher_iterations += 1
        if self.mask_padding:                                              # share of the trained tokens that were padding
            metrics['padding_fraction'] = (n_steps - sum(rollout_lens)) / n_steps
        if self.pack_sequences:                                            # share of the sequences packing saved
            metrics['packing_saved_fraction'] = 1.0 - batch.batch_size / sequence_count(rollout_lens, self.seq_len)
        n_cut = sum(not r.get('terminal', True) for r in rollouts)
        if n_cut:                                                          # share of the rollouts cut from a game that goes on
            metrics['non_terminal_fraction'] = n_cut / len(rollouts)
        if self.advantage_estimator == 'vtrace':                           # read now: the steps have synced the device
            for k, v in self.last_vtrace_stats.items():
                metrics['vtrace/{}'.format(k)] = v
        if self._upgo_prep is not None:                                    # UPGO of this iteration's prep
            metrics['upgo/coef'] = self._upgo_prep[0]
            for k, v in self.last_upgo_stats.items():
                metrics['upgo/{}'.format(k)] = v
        if self.value_norm:                                                # the statistics this iteration trained under
            st = self.value_norm_stats
            metrics['value_norm/mean'], metrics['value_norm/std'] = st['mean'], st['std']
        if self.recompute_states:                                          # how far the refreshes moved the start states
            drifts = [_drift(*acc.tolist()) for acc, _ in self._state_refresh_sums]
            metrics['refresh/state_drift'] = float(np.mean(drifts)) if drifts else 0.0
        logger.info('steps_per_s={:.2f}, avg_weight_age={:.1f}, loss={:.4f}, entropy={:.3f}'.format(
            metrics[self.SPEED_KEY], float(metrics['avg_weight_age']), float(metrics['loss/sum']), float(metrics['entropy'])))
        if self.checkpoint:
            self.upload_model(version=it)                                  # :575
        self.last_metrics = metrics
        return metrics


class _ParamGroup(collections.abc.MutableMapping):
    """The one torch-style parameter group of ``_FusedAdamHandle``.  Its ``'lr'`` is the owner's ``learning_rate``, read
    and written through, so the usual ``optimizer.param_groups[0]['lr'] = x`` sets the learning rate of the next step."""

    def __init__(self, owner, entries):
        self._owner = owner
        self._entries = {k: v for k, v in entries.items() if k != 'lr'}

    def __getitem__(self, key):
        return self._owner.learning_rate if key == 'lr' else self._entries[key]

    def __setitem__(self, key, value):
        if key == 'lr':
            self._owner.learning_rate = value
        else:
            self._entries[key] = value

    def __delitem__(self, key):
        if key == 'lr':
            raise KeyError("'lr' is the optimizer's learning_rate and cannot be removed")
        del self._entries[key]

    def __iter__(self):
        yield 'lr'
        yield from self._entries

    def __len__(self):
        return 1 + len(self._entries)

    def __repr__(self):
        return repr(dict(self))


class _FusedAdamHandle:
    """Minimal ``optimizer``-attribute stand-in: the Adam update itself is fused into ``dc_grad_finish``."""

    def __init__(self, owner):
        self._owner = owner
        self.defaults = {'lr': owner.learning_rate, 'betas': owner.ADAM_BETAS, 'eps': owner.ADAM_EPS, 'weight_decay': 0}
        self._param_groups = [_ParamGroup(owner, dict(self.defaults, params=list(owner.flat.params)))]

    @property
    def param_groups(self):
        """Persistent groups: writes to ``param_groups[0]['lr']`` reach the owner's ``learning_rate``."""
        return self._param_groups

    def zero_grad(self, set_to_none=False):
        self._owner.flat.zero_grad()

    def state_dict(self):
        """``torch.optim.Adam.state_dict()`` layout (per-parameter ``step`` / ``exp_avg`` / ``exp_avg_sq`` keyed by the
        parameter's index in ``named_parameters()`` order; tensors that never received a gradient have no entry, as in torch),
        so the checkpoint loads into a stock ``torch.optim.Adam`` over the same module and vice versa."""
        o = self._owner
        steps = o.adam_steps.cpu()
        state = {}
        for i, (p, lo, hi) in enumerate(zip(o.flat.params, o.flat.starts, o.flat.ends)):
            if int(steps[i]) > 0:
                state[i] = {'step': torch.tensor(float(steps[i])),
                            'exp_avg': o.exp_avg[lo:hi].view(p.shape).detach().cpu().clone(),
                            'exp_avg_sq': o.exp_avg_sq[lo:hi].view(p.shape).detach().cpu().clone()}
        group = dict(self.defaults, lr=o.learning_rate, amsgrad=False, maximize=False, foreach=None, capturable=False,
                     differentiable=False, fused=None, decoupled_weight_decay=False, params=list(range(o.flat.n_seg)))
        return {'state': state, 'param_groups': [group]}

    def load_state_dict(self, sd):
        """Restores the moments and step counters.  A state saved for another parameter layout (another number of tensors,
        or another shape at the same index -- e.g. a model with another ``num_layers``) raises ``ValueError`` before anything
        is changed: the state is keyed by parameter index, so it cannot be applied to a different layout."""
        o = self._owner
        if 'state' not in sd:                      # round-1 flat layout
            if (sd['exp_avg'].numel(), sd['exp_avg_sq'].numel(), sd['step'].numel()) != \
                    (o.exp_avg.numel(), o.exp_avg_sq.numel(), o.adam_steps.numel()):
                raise ValueError("Adam state was saved for another parameter layout (flat buffer of %d elements, %d tensors; "
                                 "this model: %d, %d)" % (sd['exp_avg'].numel(), sd['step'].numel(), o.exp_avg.numel(),
                                                          o.adam_steps.numel()))
            o.exp_avg.copy_(sd['exp_avg']); o.exp_avg_sq.copy_(sd['exp_avg_sq']); o.adam_steps.copy_(sd['step'])
            return
        n_saved = sum(len(g['params']) for g in sd['param_groups'])
        if n_saved != o.flat.n_seg:
            raise ValueError("Adam state was saved for %d parameter tensors; this model has %d" % (n_saved, o.flat.n_seg))
        for i, st in sd['state'].items():
            p = o.flat.params[int(i)]
            if st['exp_avg'].shape != p.shape or st['exp_avg_sq'].shape != p.shape:
                raise ValueError("Adam state of parameter %d (%s) has shape %s; the parameter is %s"
                                 % (int(i), o.flat.names[int(i)], tuple(st['exp_avg'].shape), tuple(p.shape)))
        o.exp_avg.zero_(); o.exp_avg_sq.zero_(); o.adam_steps.zero_()
        steps = torch.zeros(o.flat.n_seg, dtype=torch.int32)
        for i, st in sd['state'].items():
            i = int(i)
            lo, hi = o.flat.starts[i], o.flat.ends[i]
            o.exp_avg[lo:hi].copy_(st['exp_avg'].reshape(-1))
            o.exp_avg_sq[lo:hi].copy_(st['exp_avg_sq'].reshape(-1))
            steps[i] = int(st['step'])
        o.adam_steps.copy_(steps)


# ------------------------------------------------------------------------------------------ process entry
def init_distribution(backend='nccl'):
    """``env://`` rendezvous (:726-734); NCCL over NVLink instead of the reference's gloo over TCP."""
    assert 'WORLD_SIZE' in os.environ
    world_size = int(os.environ['WORLD_SIZE'])
    if world_size < 2:
        logger.warning('skipping distribution: world size too small ({})'.format(world_size))
        return
    if backend == 'nccl':
        torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', 0)))
    dist.init_process_group(backend=backend)
    logger.info("Distribution initialized.")


def main(rmq_host, rmq_port, epochs, min_seq_per_epoch, seq_len, learning_rate,
         pretrained_model, mq_prefetch_count, log_dir, entropy_coef, vf_coef, run_local,
         hidden_size=256, cell="gru", num_layers=1, gamma=GAMMA, gae_lambda=LAMBDA, clip_range=0.1, max_grad_norm=0.5,
         value_clip=None, advantage_estimator='gae', vtrace_rho_clip=1.0, vtrace_c_clip=1.0, num_minibatches=1,
         mask_padding=False, pack_sequences=False, policy_ratio='per_head', value_norm=False, value_norm_decay=0.99,
         kl_coef=0.0, kl_target=None, kl_stop=None, recompute_advantages=False, recompute_states=False, value_heads=None,
         value_gammas=None, teacher_model=None, teacher_coef=1.0, teacher_anneal_iterations=None, upgo_coef=0.0,
         objective='ppo', dual_clip=None):
    check_ppo_settings(gamma, gae_lambda, clip_range, max_grad_norm, value_clip, advantage_estimator=advantage_estimator,
                       vtrace_rho_clip=vtrace_rho_clip, vtrace_c_clip=vtrace_c_clip, num_minibatches=num_minibatches,
                       mask_padding=mask_padding, pack_sequences=pack_sequences,
                       policy_ratio=policy_ratio, value_norm=value_norm,
                       value_norm_decay=value_norm_decay, kl_coef=kl_coef, kl_target=kl_target,
                       kl_stop=kl_stop, recompute_advantages=recompute_advantages,
                       recompute_states=recompute_states, value_heads=value_heads,
                       value_gammas=value_gammas, teacher_model=teacher_model, teacher_coef=teacher_coef,
                       teacher_anneal_iterations=teacher_anneal_iterations,
                       upgo_coef=upgo_coef, objective=objective,
                       dual_clip=dual_clip)                                              # before any process-group setup
    check_minibatch_count(num_minibatches, min_seq_per_epoch)
    if dist.is_available() and 'WORLD_SIZE' in os.environ:
        init_distribution()
    dota_optimizer = DotaOptimizer(
        rmq_host=rmq_host, rmq_port=rmq_port, epochs=epochs, min_seq_per_epoch=min_seq_per_epoch, seq_len=seq_len,
        learning_rate=learning_rate, checkpoint=is_master(), pretrained_model=pretrained_model,
        mq_prefetch_count=mq_prefetch_count, log_dir=log_dir, entropy_coef=entropy_coef, vf_coef=vf_coef,
        run_local=run_local, hidden_size=hidden_size, cell=cell, num_layers=num_layers, gamma=gamma,
        gae_lambda=gae_lambda, clip_range=clip_range, max_grad_norm=max_grad_norm, value_clip=value_clip,
        advantage_estimator=advantage_estimator, vtrace_rho_clip=vtrace_rho_clip, vtrace_c_clip=vtrace_c_clip,
        num_minibatches=num_minibatches, mask_padding=mask_padding, pack_sequences=pack_sequences,
        policy_ratio=policy_ratio, value_norm=value_norm, value_norm_decay=value_norm_decay, kl_coef=kl_coef,
        kl_target=kl_target, kl_stop=kl_stop, recompute_advantages=recompute_advantages,
        recompute_states=recompute_states, value_heads=value_heads, value_gammas=value_gammas,
        teacher_model=teacher_model, teacher_coef=teacher_coef, teacher_anneal_iterations=teacher_anneal_iterations,
        upgo_coef=upgo_coef, objective=objective, dual_clip=dual_clip)
    if isinstance(dota_optimizer.mq, MessageQueue):
        logger.warning('the built-in MessageQueue is an IN-PROCESS broker (the AMQP transport is out of scope): with no producer '
                       'thread publishing to it in this process run() will wait forever; pass mq=<your pika-backed queue> to '
                       'DotaOptimizer for a RabbitMQ deployment (--ip/--port are accepted for CLI compatibility only)')
    dota_optimizer.run()


def default_log_dir():
    return '{}_{}'.format(datetime.now().strftime('%b%d_%H-%M-%S'), socket.gethostname())


def build_arg_parser():
    """The reference's flags and defaults (:777-794) plus ``--hidden-size``, ``--cell``, ``--num-layers`` and the PPO
    settings ``--gamma``, ``--gae-lambda``, ``--clip-range``, ``--max-grad-norm``, ``--value-clip``,
    ``--advantage-estimator``, ``--vtrace-rho-clip``, ``--vtrace-c-clip``, ``--num-minibatches``, ``--mask-padding``,
    ``--pack-sequences``, ``--policy-ratio``, ``--value-norm``, ``--value-norm-decay``, ``--kl-coef``, ``--kl-target``,
    ``--kl-stop``, ``--value-heads``, ``--value-gammas``, ``--teacher-model``, ``--teacher-coef``,
    ``--teacher-anneal-iterations``, ``--upgo-coef``, ``--objective`` and ``--dual-clip``."""
    p = argparse.ArgumentParser(formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("--log-dir", type=str, help="log and job dir name", default=default_log_dir())
    p.add_argument("--ip", type=str, help="mq ip", default='127.0.0.1')
    p.add_argument("--port", type=int, help="mq port", default=5672)
    p.add_argument("--epochs", type=int, help="amount of epochs", default=4)
    p.add_argument("--min-seq-per-epoch", type=int, help="minimum amount of sequences per epoch", default=1024)
    p.add_argument("--seq-len", type=int, help="sequence length (truncated BPTT window)", default=16)
    p.add_argument("--learning-rate", type=float, help="learning rate", default=5e-5)
    p.add_argument("--entropy-coef", type=float, help="entropy coef", default=5e-4)
    p.add_argument("--vf-coef", type=float, help="value fn coef", default=0.5)
    p.add_argument("--pretrained-model", type=str, help="pretrained model file", default=None)
    p.add_argument("--mq-prefetch-count", type=int, help="experience messages to prefetch from mq", default=1)
    p.add_argument("-l", "--log", dest="log_level", help="Set the logging level",
                   choices=['DEBUG', 'INFO', 'WARNING', 'ERROR', 'CRITICAL'], default='INFO')
    p.add_argument("--run-local", type=bool, help="set to true to run locally (not using GCP)", default=False)
    p.add_argument("--hidden-size", type=int, help="recurrent width, a multiple of 32 (reference: 256)", default=256)
    p.add_argument("--cell", type=str, choices=['gru', 'lstm'], help="recurrent cell (reference: gru)", default='gru')
    p.add_argument("--num-layers", type=int, help="recurrent layers (reference: 1)", default=1)
    p.add_argument("--gamma", type=float, help="discount factor, in (0, 1] (reference: 0.98)", default=GAMMA)
    p.add_argument("--gae-lambda", type=float, help="GAE lambda, in [0, 1] (reference: 0.97)", default=LAMBDA)
    p.add_argument("--clip-range", type=float, help="PPO ratio clip range (reference: 0.1)", default=0.1)
    p.add_argument("--max-grad-norm", type=float, help="global gradient-norm clip (reference: 0.5)", default=0.5)
    p.add_argument("--value-clip", type=float, default=None,
                   help="PPO2 value-loss clip range around the prep-time values (default: no value clipping)")
    p.add_argument("--advantage-estimator", type=str, choices=ADVANTAGE_ESTIMATORS, default='gae',
                   help="'vtrace' corrects for actors that played with older weights (rollouts must carry behaviour_logp)")
    p.add_argument("--vtrace-rho-clip", type=float, help="V-trace truncation rho-bar of the importance weights", default=1.0)
    p.add_argument("--vtrace-c-clip", type=float, help="V-trace truncation c-bar of the trace coefficients", default=1.0)
    p.add_argument("--num-minibatches", type=int, default=1,
                   help="shuffled minibatches of sequences per epoch, one optimizer step each (reference: 1)")
    p.add_argument("--mask-padding", action="store_true",
                   help="leave the zero padding of each rollout's last chunk out of GAE / V-trace and the loss "
                        "(reference: padding is trained on)")
    p.add_argument("--pack-sequences", action="store_true",
                   help="pack the rollouts' last partial chunks into shared sequences with recurrent-state resets, so "
                        "padding is not trained on (needs --mask-padding)")
    p.add_argument("--policy-ratio", type=str, choices=POLICY_RATIOS, default='per_head',
                   help="'joint' clips one PPO ratio per step, of the whole hierarchical action, instead of one per head "
                        "(reference: per_head)")
    p.add_argument("--value-norm", action="store_true",
                   help="PopArt: train the critic on returns normalised by running statistics, rescaling the value head "
                        "so that its unnormalised output is preserved (reference: raw returns)")
    p.add_argument("--value-norm-decay", type=float, default=0.99,
                   help="decay of the running value statistics per prepared batch, in [0, 1)")
    p.add_argument("--kl-coef", type=float, default=0.0,
                   help="coefficient of a penalty on the exact KL to the policy that prepared the batch (0: off)")
    p.add_argument("--kl-target", type=float, default=None,
                   help="adapt --kl-coef once per iteration: doubled above 1.5x this KL, halved below it / 1.5")
    p.add_argument("--kl-stop", type=float, default=None,
                   help="skip a step whose KL to the prep-time policy exceeds this, and the rest of the iteration's steps")
    p.add_argument("--recompute-advantages", action="store_true",
                   help="recompute the batch's advantages and returns with the current critic before every epoch after "
                        "the first")
    p.add_argument("--recompute-states", action="store_true",
                   help="rerun every rollout with the current network before every epoch after the first and replace the "
                        "recurrent states its training sequences start from")
    p.add_argument("--value-heads", type=parse_value_heads, default=None,
                   help="one value head per reward group, 'name=key,key;name=key,...' holding every reward key once "
                        "(default: one critic of the summed reward)")
    p.add_argument("--value-gammas", type=parse_value_gammas, default=None,
                   help="discounts of some value heads, 'name=0.999;...' (the others take --gamma)")
    p.add_argument("--teacher-model", type=str, default=None,
                   help="a Policy state_dict file (any width, cell or depth) whose policy the run is kickstarted from: "
                        "the loss adds --teacher-coef times the KL from it (default: no teacher)")
    p.add_argument("--teacher-coef", type=float, default=1.0,
                   help="coefficient of the KL to the teacher (needs --teacher-model)")
    p.add_argument("--teacher-anneal-iterations", type=int, default=None,
                   help="anneal --teacher-coef linearly to 0 over this many iterations, then retire the teacher "
                        "(needs --teacher-model; default: a fixed coefficient)")
    p.add_argument("--upgo-coef", type=float, default=0.0,
                   help="add this times the upgoing (UPGO) advantage, which follows a rollout's return only while the "
                        "next step does at least as well as the critic expects, to the GAE / V-trace advantage (0: off)")
    p.add_argument("--objective", type=str, choices=OBJECTIVES, default='ppo',
                   help="'bc' trains the policy on the log-likelihood of the actions of demonstrations (behaviour "
                        "cloning) instead of the PPO surrogate (reference: ppo)")
    p.add_argument("--dual-clip", type=float, default=None, metavar="C",
                   help="dual-clip PPO: floor the surrogate of every action with a negative advantage A at C * A, C > 1 "
                        "(Ye et al. 2020 use 3), so that a ratio that has run away stops driving the update (default: off)")
    return p


if __name__ == '__main__':
    args = build_arg_parser().parse_args()
    logger.setLevel(args.log_level)
    try:
        main(rmq_host=args.ip, rmq_port=args.port, epochs=args.epochs, min_seq_per_epoch=args.min_seq_per_epoch,
             seq_len=args.seq_len, learning_rate=args.learning_rate, pretrained_model=args.pretrained_model,
             mq_prefetch_count=args.mq_prefetch_count, log_dir=args.log_dir, entropy_coef=args.entropy_coef,
             vf_coef=args.vf_coef, run_local=args.run_local, hidden_size=args.hidden_size, cell=args.cell,
             num_layers=args.num_layers, gamma=args.gamma, gae_lambda=args.gae_lambda, clip_range=args.clip_range,
             max_grad_norm=args.max_grad_norm, value_clip=args.value_clip, advantage_estimator=args.advantage_estimator,
             vtrace_rho_clip=args.vtrace_rho_clip, vtrace_c_clip=args.vtrace_c_clip, num_minibatches=args.num_minibatches,
             mask_padding=args.mask_padding, pack_sequences=args.pack_sequences, policy_ratio=args.policy_ratio,
             value_norm=args.value_norm, value_norm_decay=args.value_norm_decay, kl_coef=args.kl_coef,
             kl_target=args.kl_target, kl_stop=args.kl_stop, recompute_advantages=args.recompute_advantages,
             recompute_states=args.recompute_states, value_heads=args.value_heads, value_gammas=args.value_gammas,
             teacher_model=args.teacher_model, teacher_coef=args.teacher_coef,
             teacher_anneal_iterations=args.teacher_anneal_iterations, upgo_coef=args.upgo_coef,
             objective=args.objective, dual_clip=args.dual_clip)
    except KeyboardInterrupt:
        pass
