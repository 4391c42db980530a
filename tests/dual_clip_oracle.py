"""CPU oracle of dual-clip PPO (``DotaOptimizer(dual_clip=c)``) in float64.

A_t is the token's normalised advantage (mean and unbiased std over the counting tokens, + eps, as every loss normalises
it), r a row's ratio (per head, or the joint ratio of the token) and s = min(r A_t, clamp(r, 1 - eps, 1 + eps) A_t) the
clipped surrogate.  Dual clip (Ye et al. 2020) replaces each row's s with
    term = s                 if A_t >= 0
    term = max(s, c A_t)     if A_t <  0
and the policy loss is today's mean of -term: per head, over the head's action rows, averaged over the five heads (a head
without action rows counts 0); joint, over the T_a counting tokens with an action row.  The gradient is the autograd of
``torch.where(A < 0, torch.maximum(s, c * A), s)``.  A row binds where A_t < 0 and s < c A_t.  The entropy and value terms
are ``padding_oracle.masked_ppo_loss``'s / ``joint_ratio_oracle.joint_ppo_loss``'s, the KL penalty and the teacher term
``kl_oracle.exact_kl``'s.
"""
import torch

import joint_ratio_oracle as JO
import kl_oracle as KO
import padding_oracle as PO
from oracle import ref_optimizer as RO
from oracle.ref_policy import masked_softmax

HEADS = PO.HEADS


def _counting(n, valid):
    return torch.ones(n, dtype=torch.bool) if valid is None else valid.reshape(-1).bool()


def normalised_advantage(adv_raw, valid=None):
    """A_t [N] float64: (a - mean) / (std + eps) over the counting tokens (every token's value, counting or not)."""
    a = adv_raw.reshape(-1).double()
    use = _counting(a.shape[0], valid)
    return ((a - a[use].mean()) / (a[use].std() + RO.EPS)).detach()


def dual_clip_term(r, adv, e_clip, c):
    """``(term, bound)``: each row's dual-clipped surrogate (differentiable in ``r``) and whether its floor binds."""
    s = torch.min(r * adv, torch.clamp(r, 1.0 - e_clip, 1.0 + e_clip) * adv)
    floor = c * adv
    return torch.where(adv < 0, torch.maximum(s, floor), s), (adv < 0) & (s < floor)


def policy_loss(logits, actions, masks, dense_old, adv, e_clip, c, joint=False, valid=None):
    """``(policy_loss, fractions)``: -mean of the dual-clipped terms in the chosen ratio mode (float64, differentiable in
    ``logits``), and the shares of bound rows as ``dc_ppo_loss_fwd_bwd_dual_clip`` reports them: ``'fraction'``,
    ``'fraction/<head>'`` (0 under the joint ratio) and ``'fraction/joint'`` (0 with per-head ratios)."""
    n = dense_old.shape[0]
    use = _counting(n, valid)
    fr = {'fraction/' + k: 0.0 for k in HEADS}
    fr['fraction/joint'] = 0.0
    if joint:
        log_r, has, _ = JO.joint_log_ratio(logits, actions, masks, dense_old, valid)
        t_a = int(has.sum())
        if t_a == 0:
            return torch.zeros([], dtype=torch.float64), dict(fr, fraction=0.0)
        term, bound = dual_clip_term(torch.exp(log_r[has]), adv[has], e_clip, c)
        fr['fraction/joint'] = float(bound.sum()) / t_a
        return -term.sum() / t_a, dict(fr, fraction=0.0)
    total = torch.zeros([], dtype=torch.float64)
    used = []
    for h, k in enumerate(HEADS):
        act = actions[k].bool() & use[:, None]
        rows = act.any(dim=1)
        n_h = int(rows.sum())
        if n_h == 0:                            # a head nobody used: 0, and left out of the mean fraction
            continue
        lp = masked_softmax(logits[k].double(), masks[k].bool(), dim=1)
        lpa = lp.masked_fill(~act, 0.0).sum(dim=1)[rows]
        term, bound = dual_clip_term(torch.exp(lpa - dense_old[rows, h].double()), adv[rows], e_clip, c)
        total = total - term.sum() / n_h
        fr['fraction/' + k] = float(bound.sum()) / n_h
        used.append(fr['fraction/' + k])
    return total / len(HEADS), dict(fr, fraction=sum(used) / len(used) if used else 0.0)


def dual_clip_ppo_loss(logits, values, actions, masks, dense_old, adv_raw, returns, entropy_coef, vf_coef, e_clip, c,
                       joint=False, valid=None, old_rows=None, kl_coef=0.0, teacher_rows=None, teacher_coef=0.0,
                       old_values=None, value_clip=None):
    """Flat tokens as ``joint_ratio_oracle.joint_ppo_loss``.  The dual-clipped policy loss plus the entropy and value terms
    of the chosen ratio mode, plus ``kl_coef * KL`` when ``old_rows`` is given and ``teacher_coef * KL_T`` when
    ``teacher_rows`` is.  Returns (loss, policy_loss, entropy_loss, value_loss, entropies, fractions), float64,
    differentiable in logits and values."""
    if joint:
        base = JO.joint_ppo_loss(logits, values, actions, masks, dense_old, adv_raw, returns, entropy_coef, vf_coef, e_clip,
                                 valid=valid, old_values=old_values, value_clip=value_clip)
    else:
        v = torch.ones(dense_old.shape[0], dtype=torch.bool) if valid is None else valid
        base = PO.masked_ppo_loss(logits, values, actions, masks, dense_old, adv_raw, returns, v, entropy_coef, vf_coef,
                                  e_clip, old_values=old_values, value_clip=value_clip)
    _, _, e_loss, v_loss, ents = base
    p_loss, fractions = policy_loss(logits, actions, masks, dense_old, normalised_advantage(adv_raw, valid), e_clip, c,
                                    joint, valid)
    loss = p_loss + e_loss + v_loss
    if old_rows is not None:
        loss = loss + kl_coef * KO.exact_kl(logits, actions, masks, old_rows, valid)[0]
    if teacher_rows is not None:
        loss = loss + teacher_coef * KO.exact_kl(logits, actions, masks, teacher_rows, valid)[0]
    return loss, p_loss, e_loss, v_loss, ents, fractions
