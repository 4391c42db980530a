"""CPU oracle of the PPO diagnostics (approximate KL, clip fraction, explained variance) and of the PPO2 clipped value loss,
for the tests of ``DotaOptimizer``'s schedulable PPO settings.  Sums run in float64."""
import math

import torch

from oracle import ref_optimizer as RO
from oracle.ref_policy import masked_softmax

HEADS = ("enum", "x", "y", "target_unit", "ability")


def ppo_stats(logits, masks, actions, old, values, returns, e_clip):
    """``logits`` / ``masks`` / ``actions``: dicts of ``[N, n_h]`` tensors; ``old``: dict of the compact old log-probs of
    each head's action rows (row order); ``values`` / ``returns``: ``[N]``.  Returns the dict of ``last_ppo_stats``.

    Per head over its action rows: KL ~ mean((r - 1) - log r) (k3), clip fraction = share of |r - 1| > e_clip, with
    log r = new log-prob - old log-prob.  A head without action rows reports 0 and is left out of the means.  Explained
    variance 1 - Var(ret - v) / Var(ret) over all N rows (NaN for constant returns)."""
    out, kls, clips = {}, [], []
    for k in HEADS:
        step = actions[k].bool().any(dim=-1)
        if not bool(step.any()):
            out["approx_kl/" + k] = 0.0
            out["clip_fraction/" + k] = 0.0
            continue
        lp = masked_softmax(logits[k].float(), masks[k].bool(), dim=-1)
        log_r = (lp[actions[k].bool()] - old[k].float()).double()
        r = torch.exp(log_r)
        out["approx_kl/" + k] = float(((r - 1.0) - log_r).mean())
        out["clip_fraction/" + k] = float(((r - 1.0).abs() > e_clip).double().mean())
        kls.append(out["approx_kl/" + k])
        clips.append(out["clip_fraction/" + k])
    out["approx_kl"] = sum(kls) / len(kls) if kls else 0.0
    out["clip_fraction"] = sum(clips) / len(clips) if clips else 0.0
    ret = returns.reshape(-1).double()
    d = ret - values.reshape(-1).double()
    var_r = float(ret.var(unbiased=False))
    out["explained_variance"] = math.nan if var_r == 0.0 else 1.0 - float(d.var(unbiased=False)) / var_r
    return out


def clipped_value_loss(values, old_values, returns, vf_coef, value_clip):
    """PPO2: ``0.5 * vf_coef * mean(max((v - R)^2, (v_old + clip(v - v_old, -eps, eps) - R)^2))`` (differentiable in v)."""
    v_clipped = old_values + torch.clamp(values - old_values, -value_clip, value_clip)
    return vf_coef * (0.5 * torch.maximum((values - returns).pow(2), (v_clipped - returns).pow(2)).mean())


def ppo_loss(logits, values, actions, masks, old, adv_raw, returns, entropy_coef, vf_coef, e_clip, old_values=None,
             value_clip=None):
    """``oracle.ref_optimizer.ppo_loss`` with the value loss optionally clipped against ``old_values`` (shape of
    ``returns``).  Returns (loss, policy_loss, entropy_loss, value_loss, entropies)."""
    if not value_clip:
        return RO.ppo_loss(logits, values, actions, masks, old, adv_raw, returns, entropy_coef, vf_coef, e_clip)
    loss, p_loss, e_loss, _, ents = RO.ppo_loss(logits, values, actions, masks, old, adv_raw, returns, entropy_coef, 0.0,
                                                e_clip)
    v = values.squeeze(-1)
    v_loss = clipped_value_loss(v, old_values.reshape(v.shape), returns.reshape(v.shape), vf_coef, value_clip) \
        if vf_coef > 0 else torch.tensor(0.0)
    return loss + v_loss, p_loss, e_loss, v_loss, ents
