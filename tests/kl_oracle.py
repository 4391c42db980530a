"""CPU oracle of KL control (``DotaOptimizer(kl_coef=..., kl_target=..., kl_stop=...)``) in float64.

For a token t that counts (``valid``, or every token), S_t is the set of heads with an action row at t and T_a the number of
counting tokens with S_t not empty.  p_old is the masked softmax of experience prep, p the current one (the reference's
form, normalised over the legal entries of the mask):
    KL_t = sum_{h in S_t} sum_{a legal} p_old(a) (log p_old(a) - log p(a)),     KL = (1 / T_a) sum_t KL_t  (0 if T_a = 0)
    loss = (the per-head or joint PPO loss) + beta KL
The gradient of beta KL is taken by autograd.  The beta rule and the skip decision are restated from their definitions.
"""
import torch

import joint_ratio_oracle as JO
import padding_oracle as PO
from oracle.ref_policy import masked_softmax

HEADS = PO.HEADS
SIZES = (4, 9, 9, 40, 3)
ROW = sum(SIZES)


def masked_log_rows(logits, masks):
    """``[N, 65]`` float64: every head's masked log-softmax row side by side in head order, 0 at illegal entries."""
    parts = []
    for k in HEADS:
        m = masks[k].bool()
        lp = masked_softmax(logits[k].double(), m, dim=1)
        parts.append(torch.where(m, lp, torch.zeros_like(lp)))
    return torch.cat(parts, dim=1)


def exact_kl(logits, actions, masks, old_rows, valid=None):
    """``(KL, sum_t KL_t, T_a, per_head)``: the exact KL of section 1 (differentiable in ``logits``), its numerator, T_a, and
    per head the sum of its rows' KL over its action rows divided by their count (0 for a head without any)."""
    n = old_rows.shape[0]
    use = torch.ones(n, dtype=torch.bool) if valid is None else valid.reshape(-1).bool()
    total = torch.zeros([], dtype=torch.float64)
    has = torch.zeros(n, dtype=torch.bool)
    per_head, col = {}, 0
    for k, size in zip(HEADS, SIZES):
        m = masks[k].bool()
        in_s = actions[k].bool().any(dim=1) & use
        lo = old_rows[:, col:col + size].double()
        col += size
        lp = masked_softmax(logits[k].double(), m, dim=1)
        po = torch.exp(lo)
        terms = torch.where(m & in_s[:, None], po * (lo - lp), torch.zeros_like(lp))
        row = terms.sum(dim=1)
        s = row.sum()
        total = total + s
        has |= in_s
        cnt = int(in_s.sum())
        per_head[k] = float(s.detach()) / cnt if cnt else 0.0
    t_a = int(has.sum())
    kl = total / t_a if t_a else torch.zeros([], dtype=torch.float64)
    return kl, total, t_a, per_head


def kl_ppo_loss(logits, values, actions, masks, dense_old, old_rows, adv_raw, returns, entropy_coef, vf_coef, e_clip,
                kl_coef, joint=False, valid=None, old_values=None, value_clip=None):
    """The PPO loss of the chosen ratio mode plus ``kl_coef * KL``.  Returns (loss, policy_loss, entropy_loss, value_loss,
    entropies, kl), float64, differentiable in logits and values."""
    if joint:
        base = JO.joint_ppo_loss(logits, values, actions, masks, dense_old, adv_raw, returns, entropy_coef, vf_coef, e_clip,
                                 valid=valid, old_values=old_values, value_clip=value_clip)
    else:
        v = torch.ones(dense_old.shape[0], dtype=torch.bool) if valid is None else valid
        base = PO.masked_ppo_loss(logits, values, actions, masks, dense_old, adv_raw, returns, v, entropy_coef, vf_coef,
                                  e_clip, old_values=old_values, value_clip=value_clip)
    kl, _, _, _ = exact_kl(logits, actions, masks, old_rows, valid)
    loss, p_loss, e_loss, v_loss, ents = base
    return loss + kl_coef * kl, p_loss, e_loss, v_loss, ents, kl


def kl_coef_update(kl_coef, kl, kl_target):
    """beta <- 2 beta if kl > 1.5 kl_target; beta / 2 if kl < kl_target / 1.5; else beta."""
    if kl > 1.5 * kl_target:
        return 2.0 * kl_coef
    if kl < kl_target / 1.5:
        return 0.5 * kl_coef
    return kl_coef


def kl_skip(kl_sum, t_a, kl_stop):
    """Whether a step is skipped: the all-ranks KL (sum over the ranks of sum_t KL_t, over the sum of T_a; 0 when that is
    0) exceeds a limit > 0.  ``kl_stop`` None or <= 0 is no limit."""
    kl = kl_sum / t_a if t_a > 0 else 0.0
    return bool(kl_stop is not None and kl_stop > 0 and kl > kl_stop)


def temper_rows(rows, legal):
    """A different prep-time policy over the same legal sets: each head's masked log-prob row tilted by 1.5 cos(j) on entry
    j and renormalised over the legal entries, 0 at illegal ones.  The tilt moves even a uniform row (an untrained policy's)
    far enough for the KL term to matter.  ``legal`` [..., 65] bool is the heads' masks side by side.  The transform is per
    row, so a batch and its sequences, chunked, gathered or packed, all get the same rows.  Computed in float64, returned in
    the dtype of ``rows``."""
    out, col = [], 0
    r, legal = rows.double(), legal.bool()
    for size in SIZES:
        part, m = r[..., col:col + size], legal[..., col:col + size]
        tilt = 1.5 * torch.cos(torch.arange(size, dtype=torch.float64, device=r.device))
        x = torch.where(m, part + tilt, torch.full_like(part, -torch.inf))
        lp = x - torch.logsumexp(x, dim=-1, keepdim=True)
        out.append(torch.where(m, lp, torch.zeros_like(lp)))
        col += size
    return torch.cat(out, dim=-1).to(rows.dtype)


class KLRefOptimizer(PO.MaskedRefOptimizer):
    """The reference optimizer training the per-head (``joint=False``) or joint PPO loss plus ``kl_coef * KL`` on sequences
    that carry ``old_log_probs [S, 65]`` (and ``valid`` when ``masked``)."""

    def __init__(self, policy, seq_len, kl_coef, joint=False, masked=True, **kw):
        super().__init__(policy, seq_len, **kw)
        self.kl_coef, self.joint, self.masked = kl_coef, joint, masked

    def loss_only(self, experiences):
        from oracle import ref_optimizer as RO
        adv, ret, hidden, actions, masks, obs, _ = RO.stack_batch(experiences)
        valid = torch.stack([e.valid for e in experiences]).reshape(-1) if self.masked else None
        logits, values, _ = self.policy(**obs, hidden=hidden)
        dense_old = torch.stack([PO.seq_dense_old(e) for e in experiences]).reshape(-1, 5)
        rows = torch.stack([torch.as_tensor(e.old_log_probs) for e in experiences]).reshape(-1, ROW)
        flat = {k: t.reshape(-1, t.shape[-1]) for k, t in logits.items()}
        loss, p_loss, e_loss, v_loss, ents, kl = kl_ppo_loss(
            flat, values.reshape(-1), {k: a.reshape(flat[k].shape) for k, a in actions.items()},
            {k: m.reshape(flat[k].shape) for k, m in masks.items()}, dense_old, rows, adv.reshape(-1), ret.reshape(-1),
            self.entropy_coef, self.vf_coef, self.e_clip, self.kl_coef, joint=self.joint, valid=valid)
        self.last_kl = float(kl.detach())
        return (loss, p_loss, e_loss, v_loss, ents), logits, values
