"""The loss terms of KL control, kickstarting, behaviour cloning, value heads and PopArt written for any dtype and device,
on top of ``test_gpu_ppo_fp64.reference`` (the per-head / joint PPO loss with its closed-form dlogits and dvalue), for
the whole-step float64 suite ``test_gpu_objectives_fp64``.

For a token t that counts (``valid``), S_t is the set of heads with an action row at t and T_a the number of counting
tokens with S_t not empty.  p is the masked softmax of the current logits, over the legal entries of the stored mask:
    KL control     + beta KL,        KL   = (1 / T_a) sum_t sum_{h in S_t} sum_{a legal} p_old(a) (log p_old(a) - log p(a))
    kickstarting   + lambda KL_T,    KL_T = the same with the teacher's rows
    behaviour      the surrogate replaced by NLL = (1 / T_a) sum_t sum_{h in S_t} -log p(a_{t,h})
    cloning        (the advantages are not read: the PPO reference runs with advantages 0, whose surrogate is exactly 0)
    value heads    the PPO value term off; vf_coef sum_k 0.5 mean_t l_k,t with l the squared or PPO2-clipped error of
                   head k against its own returns and old values
    PopArt         the value term on fp32((R - mu) / sigma) and fp32((V_old - mu) / sigma), computed in float64
The extra terms are differentiated by autograd in ``dtype``; the KL terms as the loss above (gradient
(beta / T_a)(p sum p_old - p_old), which is (beta / T_a)(p - p_old) up to the rounding of the stored rows), so that in
float64 the result is the definition ``kl_oracle`` / ``teacher_oracle`` / ``bc_oracle`` / ``value_heads_oracle`` /
``value_norm_oracle`` use (``test_gpu_objectives_fp64.test_reference_and_bound_on_the_cpu``).
"""
import math

import torch

import test_gpu_ppo_fp64 as PF

HEADS = PF.HEADS
SIZES = PF.SIZES
ROW = sum(SIZES)
TIE_MARGIN = 1e-4          # a row whose top two masked logits lie closer than this has an arg-max fp32 may decide either way


def normalised(x, norm):
    """fp32((x - mu) / sigma) from float64, as the loss kernel reads a raw target under PopArt."""
    mu, sigma = norm
    return ((x.double() - mu) / sigma).float()


def _log_softmax(lg, mask):
    e = torch.where(mask, lg, torch.zeros_like(lg)).exp() * mask
    return lg - e.sum(1, keepdim=True).log()


def kl_to_rows(lg, masks, actions, use, rows, dtype):
    """-> (KL differentiable in ``lg``, per head {name: sum of its action rows' KL / their count}, T_a)."""
    n = use.shape[0]
    total = torch.zeros([], dtype=dtype, device=use.device)
    has = torch.zeros(n, dtype=torch.bool, device=use.device)
    per_head, col = {}, 0
    for h, (k, size) in enumerate(zip(HEADS, SIZES)):
        m = masks[h]
        in_s = actions[h].any(1) & use
        lo = rows[:, col:col + size].to(dtype)
        col += size
        lp = _log_softmax(lg[h], m)
        s = torch.where(m & in_s[:, None], lo.exp() * (lo - lp), torch.zeros_like(lp)).sum()
        total = total + s
        has |= in_s
        cnt = int(in_s.sum())
        per_head[k] = float(s.detach()) / cnt if cnt else 0.0
    t_a = int(has.sum())
    return (total / t_a if t_a else total * 0.0), per_head, t_a


def nll(lg, masks, actions, use, dtype):
    """-> (NLL differentiable in ``lg``, per head {name: sum of -log p(a) over its action rows / their count}, T_a)."""
    n = use.shape[0]
    total = torch.zeros([], dtype=dtype, device=use.device)
    has = torch.zeros(n, dtype=torch.bool, device=use.device)
    per_head = {}
    for h, k in enumerate(HEADS):
        act = actions[h] & use[:, None]
        in_s = act.any(1)
        s = -torch.where(act, _log_softmax(lg[h], masks[h]), torch.zeros_like(lg[h])).sum()
        total = total + s
        has |= in_s
        cnt = int(in_s.sum())
        per_head[k] = float(s.detach()) / cnt if cnt else 0.0
    t_a = int(has.sum())
    return (total / t_a if t_a else total * 0.0), per_head, t_a


def accuracy(logits, masks, actions, use):
    """-> (token accuracy, per head accuracy, near, rows): the arg-max decisions of ``bc_oracle.accuracy`` on ``logits``
    (lowest index on ties); ``near`` / ``rows`` {name: count} per 'bc/accuracy/<head>' the action rows whose top two masked
    logits lie within ``TIE_MARGIN`` / all its action rows, and for 'bc/accuracy' the tokens with such a row / T_a."""
    n = use.shape[0]
    has = torch.zeros(n, dtype=torch.bool, device=use.device)
    wrong = torch.zeros(n, dtype=torch.bool, device=use.device)
    near_tok = torch.zeros(n, dtype=torch.bool, device=use.device)
    per_head, near, rows = {}, {}, {}
    for h, k in enumerate(HEADS):
        in_s = actions[h].any(1) & use
        x = logits[h].double().masked_fill(~masks[h], -math.inf)
        right = in_s & (x.argmax(1) == actions[h].int().argmax(1))
        tie = torch.zeros_like(in_s)
        if x.shape[1] > 1:
            top = x.topk(2, dim=1).values
            tie = in_s & ((top[:, 0] - top[:, 1]) < TIE_MARGIN)
        has |= in_s
        wrong |= in_s & ~right
        near_tok |= tie
        cnt = int(in_s.sum())
        per_head[k] = int(right.sum()) / cnt if cnt else 0.0
        near["bc/accuracy/" + k], rows["bc/accuracy/" + k] = int(tie.sum()), cnt
    t_a = int(has.sum())
    near["bc/accuracy"], rows["bc/accuracy"] = int(near_tok.sum()), t_a
    return (int((has & ~wrong).sum()) / t_a if t_a else 0.0), per_head, near, rows


def explained_variance(ret, v):
    var_r = float(ret.var(unbiased=False))
    return math.nan if var_r == 0.0 else 1.0 - float((ret - v).var(unbiased=False)) / var_r


def reference(inp, dtype, joint, value_clip=None, old_rows=None, beta=0.0, teacher_rows=None, lam=0.0, bc=False,
              head_names=None, norm=None, entropy_coef=5e-4, vf_coef=0.5):
    """``test_gpu_ppo_fp64.reference`` with the terms above.  ``inp`` as there; with ``head_names`` (K value heads)
    ``values`` / ``ret`` / ``old_values`` are [N, K].  ``old_rows`` / ``teacher_rows`` [N, 65] are the prep-time / teacher
    log-prob rows, ``norm`` = (mu, sigma).  -> the dict of ``reference`` (dvalue [N, K] with value heads) plus 'kl',
    'kl/<head>', 'kl_penalty', 'teacher/kl', 'teacher/kl/<head>', 'loss/teacher', 'bc/nll/<head>', 'bc/accuracy',
    'bc/accuracy/<head>', 'near_ties/<accuracy>', 'rows/<accuracy>', 'loss/value/<head>', 'explained_variance/<head>' as they apply."""
    n = inp["adv"].shape[0]
    use = inp["valid"] if inp["valid"] is not None else torch.ones(n, dtype=torch.bool, device=inp["adv"].device)
    base = dict(inp)
    if norm is not None:
        base["ret"] = normalised(inp["ret"], norm)
        base["old_values"] = None if inp["old_values"] is None else normalised(inp["old_values"], norm)
    if bc:
        base["adv"] = torch.zeros_like(inp["adv"])
    if head_names is not None:          # the PPO loss with its value term off; the heads' term below
        base.update(values=inp["values"][:, 0], ret=inp["ret"][:, 0], old_values=None)
    out = PF.reference(base, dtype, joint, entropy_coef=entropy_coef, vf_coef=0.0 if head_names else vf_coef,
                       value_clip=None if head_names else value_clip)
    lg = [l.to(dtype, copy=True).requires_grad_(True) for l in inp["logits"]]
    extra = torch.zeros([], dtype=dtype, device=use.device)
    if old_rows is not None:
        kl, per_head, _ = kl_to_rows(lg, inp["masks"], inp["actions"], use, old_rows, dtype)
        extra = extra + beta * kl
        out["kl"] = out["kl_all_ranks"] = float(kl.detach())
        out["kl_penalty"] = beta * out["kl"]
        out.update({"kl/" + k: v for k, v in per_head.items()})
    if teacher_rows is not None:
        kl_t, per_head, _ = kl_to_rows(lg, inp["masks"], inp["actions"], use, teacher_rows, dtype)
        extra = extra + lam * kl_t
        out["teacher/kl"] = float(kl_t.detach())
        out["loss/teacher"] = lam * out["teacher/kl"]
        out.update({"teacher/kl/" + k: v for k, v in per_head.items()})
    if bc:
        l_nll, per_head, _ = nll(lg, inp["masks"], inp["actions"], use, dtype)
        extra = extra + l_nll
        out["policy"] = float(l_nll.detach())
        out.update({"bc/nll/" + k: v for k, v in per_head.items()})
        acc, per_acc, near, rows = accuracy(inp["logits"], inp["masks"], inp["actions"], use)
        out["bc/accuracy"] = acc
        out.update({"bc/accuracy/" + k: v for k, v in per_acc.items()})
        out.update({"near_ties/" + k: v for k, v in near.items()})
        out.update({"rows/" + k: v for k, v in rows.items()})
    if extra.requires_grad:
        extra.backward()
        out["dlogits"] = [d + (x.grad if x.grad is not None else 0.0) for d, x in zip(out["dlogits"], lg)]
    out["loss"] = out["loss"] + float(extra.detach())
    if head_names is not None:
        v = inp["values"].to(dtype, copy=True).requires_grad_(True)
        ret, vu = inp["ret"].to(dtype)[use], v[use]
        l = (vu - ret).pow(2)
        if value_clip:
            vo = inp["old_values"].to(dtype)[use]
            l = torch.maximum(l, (vo + (vu - vo).clamp(-value_clip, value_clip) - ret).pow(2))
        heads = vf_coef * 0.5 * l.mean(0)
        heads.sum().backward()
        out["dvalue"] = v.grad
        out["value_loss"] = float(heads.sum().detach())
        out["loss"] = out["loss"] + out["value_loss"]
        with torch.no_grad():
            for k, name in enumerate(head_names):
                out["loss/value/" + name] = float(heads[k])
                out["explained_variance/" + name] = explained_variance(ret[:, k], vu[:, k])
            out["explained_variance"] = explained_variance(ret.sum(1), vu.sum(1))
    return out
