"""One flat fp32 buffer for all parameters, one for all gradients (+ per-parameter has-grad slots).

The reference synchronises gradients with 68 blocking collectives per step (``distributed.py:29-57``)
and then walks the 34 tensors three more times (two norm passes, clip, Adam: ``optimizer.py:674-681``).
Re-homing every ``nn.Parameter`` as a view into one contiguous buffer turns that into ONE all-reduce
over NVLink and one fused finish kernel (``csrc/grad_finish.cu``).  ``state_dict()`` is unaffected
(same keys, shapes, values), so checkpoints stay byte-compatible with the reference's agents.
"""
import torch

# Parameters that only receive a gradient when a particular action head was used in the batch
# (``optimizer.py:627-630`` skips unused heads, so their .grad stays None in the reference):
# affine_unit_eth reaches the loss only through the target_unit head because of the
# ``eth_embedding_max`` quirk at ``policy.py:127``.
HEAD_INDEX = {"enum": 0, "x": 1, "y": 2, "target_unit": 3, "ability": 4}
VALUE_SLOT = 5     # pseudo-head: 1 when vf_coef > 0 (value loss present), else 0
PARAM_HEAD = {
    "affine_head_enum": 0, "affine_move_x": 1, "affine_move_y": 2,
    "affine_unit_attention": 3, "affine_unit_eth": 3, "affine_head_ability": 4,
    "affine_value": VALUE_SLOT,
}


def head_dependency(param_name):
    """-1 if the parameter always has a gradient, else the index of the head it depends on."""
    return PARAM_HEAD.get(param_name.split(".")[0], -1)


class FlatParameterSpace:
    """Re-homes ``module``'s parameters (in ``named_parameters()`` order == the reference's all-reduce order).

    ``kl_tail=True`` (KL control) gives ``grad_full`` two more floats after the has-grad flags, ``kl_tail``: the PPO loss
    writes the rank's (sum_t KL_t, T_a) there, so the one gradient all-reduce also sums them over the ranks."""
    ALIGN = 64      # floats
    KL_TAIL = 2

    def __init__(self, module, device=None, kl_tail=False):
        named = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        if not named:
            raise ValueError("module has no trainable parameters")
        device = torch.device(device) if device is not None else named[0][1].device
        self.names = [n for n, _ in named]
        self.params = [p for _, p in named]
        sizes = [p.numel() for p in self.params]
        # every tensor starts on a 256-byte boundary (16-byte alignment is required by the tensor-core GEMM and by
        # vectorised loads); the padding elements stay zero and are never touched by the finish kernels.
        starts, cursor = [], 0
        for s in sizes:
            starts.append(cursor)
            cursor = (cursor + s + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        self.total = cursor
        self.n_seg = len(sizes)
        self.starts = starts
        self.ends = [a + s for a, s in zip(starts, sizes)]
        offs = starts + [cursor]                       # kept for compatibility: offs[i] = start of tensor i
        self.param = torch.zeros(self.total, dtype=torch.float32, device=device)
        # gradient buffer carries n_seg extra slots: per-parameter has-grad flags / counts (distributed.py:36-37)
        extra = self.KL_TAIL if kl_tail else 0
        self.grad_full = torch.zeros(self.total + self.n_seg + extra, dtype=torch.float32, device=device)
        self.grad = self.grad_full[:self.total]
        self.flags = self.grad_full[self.total:self.total + self.n_seg]
        self.kl_tail = self.grad_full[self.total + self.n_seg:] if kl_tail else None
        for p, lo, hi in zip(self.params, self.starts, self.ends):
            self.param[lo:hi].copy_(p.data.reshape(-1))
            p.data = self.param[lo:hi].view(p.shape)
            p.grad = self.grad[lo:hi].view(p.shape)
        self.offsets = offs
        self.seg_lo = torch.tensor(self.starts, dtype=torch.int64, device=device)
        self.seg_hi = torch.tensor(self.ends, dtype=torch.int64, device=device)
        self.seg_head = torch.tensor([head_dependency(n) for n in self.names], dtype=torch.int32, device=device)
        module._dc_flat_space = self

    @staticmethod
    def of(module, device=None):
        space = getattr(module, "_dc_flat_space", None)
        if space is None or (device is not None and space.param.device != torch.device(device)):
            space = FlatParameterSpace(module, device)
        return space

    def rebind(self):
        """Re-attach ``.grad`` views (``optimizer.zero_grad()`` / ``set_to_none`` detaches them)."""
        for p, lo, hi in zip(self.params, self.starts, self.ends):
            if p.grad is None or p.grad.data_ptr() != self.grad[lo:hi].data_ptr():
                p.grad = self.grad[lo:hi].view(p.shape)

    def zero_grad(self):
        self.grad_full.zero_()
        self.rebind()

    def zero_grad_detached(self):
        """Zeroes the flat gradient buffer and DETACHES every ``.grad`` (sets it to None): autograd then hands each parameter
        its gradient tensor as is instead of launching one ``grad += new`` kernel per parameter (34 small launches per step);
        ``gather_grads`` moves them into the flat buffer with one multi-tensor copy and re-attaches the views."""
        self.grad_full.zero_()
        for p in self.params:
            p.grad = None

    def gather_grads(self):
        dsts, srcs = [], []
        for p, lo, hi in zip(self.params, self.starts, self.ends):
            g = p.grad
            view = self.grad[lo:hi].view(p.shape)
            if g is not None and g.data_ptr() != view.data_ptr():
                dsts.append(view)
                srcs.append(g.detach())
            p.grad = view
        if dsts:
            torch._foreach_copy_(dsts, srcs)

    def grad_of(self, name):
        i = self.names.index(name)
        return self.grad[self.starts[i]:self.ends[i]].view(self.params[i].shape)
