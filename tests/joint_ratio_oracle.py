"""CPU oracle of ``DotaOptimizer(policy_ratio='joint')``: the PPO loss with one clipped ratio per step, of the whole
hierarchical action, and its diagnostics, in float64.

Per token t that counts (``valid``, or every token), S_t is the set of heads with an action row at t and T_a the number of
counting tokens with S_t not empty:
    log r_t = sum_{h in S_t} (logp_new[t, h, a_h] - old_logp[t, h])
    policy  = -(1 / T_a) sum_t min(r_t A_t, clamp(r_t, 1 - eps, 1 + eps) A_t)            (0 when T_a = 0)
The advantage normalisation, the per-head entropy terms, the value loss (clipped or not) and the skipping of a head without
action rows are those of the default objective (``padding_oracle.masked_ppo_loss``).
"""
import torch

import padding_oracle as PO
import ppo_controls_oracle as PC
from oracle import ref_optimizer as RO
from oracle.ref_policy import masked_softmax

HEADS = PC.HEADS


def _counting(n, valid):
    return torch.ones(n, dtype=torch.bool) if valid is None else valid.reshape(-1).bool()


def joint_log_ratio(logits, actions, masks, dense_old, valid=None):
    """``(log_r [N] float64, has [N] bool, lp)``: the joint log-ratio of every token (0 where S_t is empty), whether S_t is
    not empty on a counting token, and each head's float64 masked log-softmax.  Differentiable in the logits."""
    n = dense_old.shape[0]
    use = _counting(n, valid)
    log_r = torch.zeros(n, dtype=torch.float64)
    has = torch.zeros(n, dtype=torch.bool)
    lps = {}
    for h, k in enumerate(HEADS):
        act = actions[k].bool() & use[:, None]
        step = act.any(dim=1)
        if not bool(step.any()):                       # a head nobody used: skipped, as in the default objective
            continue
        lp = masked_softmax(logits[k].double(), masks[k].bool(), dim=1)
        lps[k] = lp
        sel = lp.masked_fill(~act, 0.0).sum(dim=1)      # lp[t, a_h] on the rows of S_t, 0 elsewhere
        log_r = log_r + torch.where(step, sel - dense_old[:, h].double(), torch.zeros_like(sel))
        has |= step
    return log_r, has, lps


def joint_ppo_loss(logits, values, actions, masks, dense_old, adv_raw, returns, entropy_coef, vf_coef, e_clip, valid=None,
                   old_values=None, value_clip=None):
    """Flat tokens: ``logits`` / ``actions`` / ``masks`` dicts of ``[N, n_h]``, ``values`` / ``adv_raw`` / ``returns`` /
    ``valid`` / ``old_values`` ``[N]``, ``dense_old`` ``[N, 5]``.  Returns (loss, policy_loss, entropy_loss, value_loss,
    entropies), float64, differentiable in logits and values."""
    n = dense_old.shape[0]
    use = _counting(n, valid)
    a = adv_raw.reshape(-1).double()
    adv = ((a - a[use].mean()) / (a[use].std() + RO.EPS)).detach()
    log_r, has, lps = joint_log_ratio(logits, actions, masks, dense_old, valid)
    entropies = {}
    for k in HEADS:
        if k not in lps:
            entropies[k] = torch.zeros([], dtype=torch.float64)
            continue
        n_h = (actions[k].bool() & use[:, None]).any(dim=1).sum()
        lp_m = torch.masked_select(lps[k], masks[k].bool() & use[:, None])
        entropies[k] = -(torch.exp(lp_m) * lp_m).sum() / n_h
    t_a = int(has.sum())
    if t_a == 0:
        p_loss = torch.zeros([], dtype=torch.float64)
    else:
        r = torch.exp(log_r[has])
        surr1 = r * adv[has]
        surr2 = torch.clamp(r, 1.0 - e_clip, 1.0 + e_clip) * adv[has]
        p_loss = -torch.min(surr1, surr2).sum() / t_a
    e_loss = -entropy_coef * torch.stack(list(entropies.values())).sum() if entropy_coef > 0 \
        else torch.zeros([], dtype=torch.float64)
    v = values.reshape(-1)[use].double()
    ret = returns.reshape(-1)[use].double()
    if vf_coef <= 0:
        v_loss = torch.zeros([], dtype=torch.float64)
    elif value_clip:
        v_loss = PC.clipped_value_loss(v, old_values.reshape(-1)[use].double(), ret, vf_coef, value_clip)
    else:
        v_loss = vf_coef * (0.5 * (ret - v).pow(2).mean())
    return p_loss + e_loss + v_loss, p_loss, e_loss, v_loss, entropies


def joint_stats(logits, actions, masks, dense_old, e_clip, valid=None):
    """``approx_kl/joint`` (k3: (r - 1) - log r) and ``clip_fraction/joint`` (share of |r - 1| > e_clip) over the T_a
    tokens; 0 when T_a = 0."""
    with torch.no_grad():
        log_r, has, _ = joint_log_ratio(logits, actions, masks, dense_old, valid)
    if not bool(has.any()):
        return {"approx_kl/joint": 0.0, "clip_fraction/joint": 0.0}
    lr = log_r[has]
    return {"approx_kl/joint": float((torch.expm1(lr) - lr).mean()),
            "clip_fraction/joint": float(((torch.exp(lr) - 1.0).abs() > e_clip).double().mean())}


class JointRefOptimizer(RO.RefOptimizer):
    """``oracle.ref_optimizer.RefOptimizer`` training the joint objective on sequences that carry their own advantages,
    returns, dense-able old log-probs and, optionally, ``valid``."""

    def loss_only(self, experiences):
        adv, ret, hidden, actions, masks, obs, _ = RO.stack_batch(experiences)
        logits, values, _ = self.policy(**obs, hidden=hidden)
        valid = None
        if getattr(experiences[0], "valid", None) is not None:
            valid = torch.stack([e.valid for e in experiences]).reshape(-1)
        dense_old = torch.stack([PO.seq_dense_old(e) for e in experiences]).reshape(-1, 5)
        flat = {k: t.reshape(-1, t.shape[-1]) for k, t in logits.items()}
        out = joint_ppo_loss(flat, values.reshape(-1), {k: a.reshape(flat[k].shape) for k, a in actions.items()},
                             {k: m.reshape(flat[k].shape) for k, m in masks.items()}, dense_old, adv.reshape(-1),
                             ret.reshape(-1), self.entropy_coef, self.vf_coef, self.e_clip, valid=valid)
        return out, logits, values
