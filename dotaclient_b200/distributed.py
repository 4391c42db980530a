"""Data-parallel gradient synchronisation -- drop-in for the reference's ``distributed.py``.

``DistributedDataParallelSparseParamCPU(module)`` keeps the reference's name and surface
(``.module``, ``.sync_parameters()``, ``.forward``; ``distributed.py:16-79``) but

* broadcasts ONE flat parameter buffer from rank 0 instead of 34 tensors (``distributed.py:71-74``),
* synchronises gradients with ONE all-reduce of ``[all grads | per-parameter has-grad flags]``
  (NCCL over NVLink when the buffer is on a GPU) instead of 68 gloo collectives
  (``distributed.py:29-57``), and
* forwards ``init_hidden`` / ``sequence`` / ``single`` / ``forward_time_major`` to the wrapped module,
  which the reference's wrapper lacks (its multi-optimizer path raises ``AttributeError`` at
  ``optimizer.py:340,385``; SURVEY.md 0.4).

Sparse-parameter semantics: a parameter's gradient is divided by the number of ranks that had one
(``distributed.py:36-37,57``).  Deliberate fix: the averaged gradient is applied on EVERY rank, including
ranks that had none locally -- the reference discards it there (``distributed.py:50-56`` writes into a
temporary), which silently de-synchronises replicas.  Documented in DESIGN.md.
"""
import logging

import torch
import torch.distributed as dist
from torch.autograd import Variable
from torch.nn.modules import Module

from .flat import FlatParameterSpace

logger = logging.getLogger(__name__)


def is_distributed():
    return dist.is_available() and dist.is_initialized()


class DistributedDataParallelSparseParamCPU(Module):
    """Name kept for drop-in compatibility; the buffers live wherever the module lives (GPU here)."""

    def __init__(self, module, flat_space=None):
        super().__init__()
        self.module = module
        self.flat = flat_space if flat_space is not None else FlatParameterSpace.of(module)
        self.needs_reduction = False
        # A caller that runs a backward through the wrapper's forward but reduces by itself (allreduce_gradients) sets
        # this to False.  DotaOptimizer.train does not need it: it runs the module directly, so needs_reduction stays False.
        self.auto_reduce = True
        self.sync_parameters()

        def reduce_after_backward():
            if self.needs_reduction and self.auto_reduce:
                self.needs_reduction = False
                self.allreduce_gradients(divide=True)

        for p in self.flat.params:
            def hook(*unused):
                Variable._execution_engine.queue_callback(reduce_after_backward)     # distributed.py:63-69
            p.register_hook(hook)

    # -- reference surface -------------------------------------------------------------------
    def sync_parameters(self):
        """Rank 0's parameters everywhere (``distributed.py:71-74``), one broadcast."""
        if is_distributed():
            dist.broadcast(self.flat.param, 0)

    def forward(self, *inputs, **kwargs):
        self.needs_reduction = True                                                   # distributed.py:76-79
        return self.module(*inputs, **kwargs)

    # -- forwarded module API (fixes SURVEY.md 0.4) ----------------------------------------------
    def init_hidden(self):
        return self.module.init_hidden()

    def sequence(self, hidden, **kwargs):
        return self.module.sequence(hidden, **kwargs)

    def single(self, hidden, **kwargs):
        return self.module.single(hidden, **kwargs)

    def forward_time_major(self, observations, hidden):
        self.needs_reduction = True
        return self.module.forward_time_major(observations, hidden)

    # -- gradient synchronisation ----------------------------------------------------------------
    def set_local_flags(self, has_grad=None):
        """Writes this rank's has-grad flags (1/0 per parameter) behind the gradients."""
        if has_grad is None:
            self.flat.flags.fill_(1.0)
        else:
            self.flat.flags.copy_(torch.as_tensor(has_grad, dtype=torch.float32, device=self.flat.flags.device))

    def allreduce_gradients(self, divide=True, flags_ready=False):
        """ONE all-reduce(SUM) of gradients + flags; optionally the count-divide (``distributed.py:56-57``)."""
        flat = self.flat
        if not flags_ready:
            self.set_local_flags()
        if is_distributed():
            dist.all_reduce(flat.grad_full, op=dist.ReduceOp.SUM)
        if divide:
            counts = flat.flags.clamp(min=1.0)
            lengths = torch.tensor([hi - lo for lo, hi in zip(flat.offsets[:-1], flat.offsets[1:])],
                                   device=flat.grad.device)      # padded extents: the padding holds zeros
            flat.grad.div_(torch.repeat_interleave(counts, lengths))
