"""CPU oracle of the kickstarting term (``DotaOptimizer(teacher_model=..., teacher_coef=...)``) in float64.

For a token t that counts (``valid``, or every token), S_t is the set of heads with an action row at t and T_a the number of
counting tokens with S_t not empty.  p_T is the teacher's masked softmax and p the current one, both over the legal entries
of the stored mask, in the reference's form:
    KL_T = (1 / T_a) sum_t sum_{h in S_t} sum_{a legal} p_T(a) (log p_T(a) - log p(a))     (0 when T_a = 0)
    loss = (the per-head or joint PPO loss) + beta KL(p_old || p) + lambda KL_T
This is the definition of KL control with the teacher's rows in place of the prep-time ones, so ``kl_oracle.exact_kl`` and
``kl_oracle.masked_log_rows`` serve both.  The gradient is taken by autograd.  The anneal is restated from its definition.
"""
import torch

import kl_oracle as KO

masked_log_rows = KO.masked_log_rows


def teacher_kl(logits, actions, masks, teacher_rows, valid=None):
    """``(KL_T, sum_t KL_t, T_a, per_head)`` of ``kl_oracle.exact_kl`` on the teacher's rows."""
    return KO.exact_kl(logits, actions, masks, teacher_rows, valid)


def teacher_ppo_loss(logits, values, actions, masks, dense_old, old_rows, teacher_rows, adv_raw, returns, entropy_coef,
                     vf_coef, e_clip, kl_coef, teacher_coef, joint=False, valid=None, old_values=None, value_clip=None):
    """The PPO loss of the chosen ratio mode, plus ``kl_coef * KL`` when ``old_rows`` is given, plus
    ``teacher_coef * KL_T``.  Returns (loss, policy_loss, entropy_loss, value_loss, entropies, kl_t), float64,
    differentiable in logits and values."""
    rows = old_rows if old_rows is not None else teacher_rows
    beta = kl_coef if old_rows is not None else 0.0
    loss, p_loss, e_loss, v_loss, ents, _ = KO.kl_ppo_loss(
        logits, values, actions, masks, dense_old, rows, adv_raw, returns, entropy_coef, vf_coef, e_clip, beta,
        joint=joint, valid=valid, old_values=old_values, value_clip=value_clip)
    kl_t = teacher_kl(logits, actions, masks, teacher_rows, valid)[0]
    return loss + teacher_coef * kl_t, p_loss, e_loss, v_loss, ents, kl_t


def anneal(teacher_coef, n, n_anneal):
    """lambda before an iteration with ``n`` iterations already trained with the teacher: teacher_coef max(0, 1 - n / N)
    (``n_anneal`` = N), or teacher_coef without an anneal (N None)."""
    if n_anneal is None:
        return teacher_coef
    return teacher_coef * max(0.0, 1.0 - n / n_anneal)
