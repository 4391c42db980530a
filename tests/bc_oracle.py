"""CPU oracle of behaviour cloning (``DotaOptimizer(objective='bc')``) in float64.

For a token t that counts (``valid``, or every token), S_t is the set of heads with an action row at t, a_{t,h} the action of
row (t, h), and T_a the number of counting tokens with S_t not empty.  p is the masked softmax over the legal entries of the
stored mask, in the reference's form:
    NLL  = (1 / T_a) sum_t sum_{h in S_t} -log p(a_{t,h})                                   (0 when T_a = 0)
    loss = NLL + the entropy term + the value term of the default objective
    d NLL / d logit[t, h, j] = (1 / T_a)(p(j) - [j == a_{t,h}])  for h in S_t and j legal, 0 elsewhere
The entropy and value terms are those of ``padding_oracle.masked_ppo_loss``.  With every advantage 0 the normalised
advantage is 0, so that loss's policy term and its gradient are exactly 0 and one call gives the other two terms alone.
The accuracy of a row is whether the arg-max of its masked logits (the lowest index on ties) is its action.
"""
import torch

import padding_oracle as PO
from oracle.ref_policy import masked_softmax

HEADS = PO.HEADS


def _counting(n, valid):
    return torch.ones(n, dtype=torch.bool) if valid is None else valid.reshape(-1).bool()


def nll(logits, actions, masks, valid=None):
    """``(NLL, T_a, per_head_sum, per_head_count)``: the NLL (differentiable in ``logits``), T_a, and per head the sum of
    -log p(a) over its action rows on counting tokens and the number of those rows."""
    n = actions[HEADS[0]].shape[0]
    use = _counting(n, valid)
    total = torch.zeros([], dtype=torch.float64)
    has = torch.zeros(n, dtype=torch.bool)
    sums, counts = {}, {}
    for k in HEADS:
        act = actions[k].bool() & use[:, None]
        in_s = act.any(dim=1)
        lp = masked_softmax(logits[k].double(), masks[k].bool(), dim=1)
        s = -lp.masked_fill(~act, 0.0).sum()
        total = total + s
        has |= in_s
        sums[k], counts[k] = float(s.detach()), int(in_s.sum())
    t_a = int(has.sum())
    return (total / t_a if t_a else torch.zeros([], dtype=torch.float64)), t_a, sums, counts


def accuracy(logits, actions, masks, valid=None):
    """``(token_accuracy, per_head)``: the share of the T_a tokens whose every row in S_t is right, and per head the share
    of its action rows that are right (0 for a head without any)."""
    n = actions[HEADS[0]].shape[0]
    use = _counting(n, valid)
    has = torch.zeros(n, dtype=torch.bool)
    wrong = torch.zeros(n, dtype=torch.bool)
    per_head = {}
    for k in HEADS:
        m = masks[k].bool()
        in_s = actions[k].bool().any(dim=1) & use
        best = logits[k].double().masked_fill(~m, float("-inf")).argmax(dim=1)    # torch: the first of equal maxima
        right = in_s & (best == actions[k].int().argmax(dim=1))
        has |= in_s
        wrong |= in_s & ~right
        cnt = int(in_s.sum())
        per_head[k] = int(right.sum()) / cnt if cnt else 0.0
    t_a = int(has.sum())
    return (int((has & ~wrong).sum()) / t_a if t_a else 0.0), per_head


def nll_dlogits(logits, actions, masks, valid=None):
    """The closed form of d NLL / d logits, per head ``[N, n_h]`` float64."""
    n = actions[HEADS[0]].shape[0]
    use = _counting(n, valid)
    t_a = int((torch.stack([actions[k].bool().any(dim=1) for k in HEADS], 1).any(dim=1) & use).sum())
    out = {}
    for k in HEADS:
        m = masks[k].bool()
        in_s = actions[k].bool().any(dim=1) & use
        p = torch.exp(masked_softmax(logits[k].double(), m, dim=1)).masked_fill(~m, 0.0)
        g = (p - actions[k].double()) / max(t_a, 1)
        out[k] = torch.where(in_s[:, None] & m, g, torch.zeros_like(g))
    return out


def bc_loss(logits, values, actions, masks, returns, entropy_coef, vf_coef, valid=None, old_values=None, value_clip=None):
    """Flat tokens: ``logits`` / ``actions`` / ``masks`` dicts of ``[N, n_h]``, ``values`` / ``returns`` / ``valid`` /
    ``old_values`` ``[N]``.  Returns (loss, NLL, entropy_loss, value_loss, entropies), float64, differentiable in logits and
    values."""
    n = values.reshape(-1).shape[0]
    use = _counting(n, valid)
    zeros = torch.zeros(n, dtype=torch.float64)
    _, _, e_loss, v_loss, ents = PO.masked_ppo_loss(logits, values, actions, masks, torch.zeros(n, 5, dtype=torch.float64),
                                                    zeros, returns, use, entropy_coef, vf_coef, 0.2,
                                                    old_values=old_values, value_clip=value_clip)
    l_nll = nll(logits, actions, masks, valid)[0]
    return l_nll + e_loss + v_loss, l_nll, e_loss, v_loss, ents
