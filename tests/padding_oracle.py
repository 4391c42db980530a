"""CPU oracle of ``DotaOptimizer(mask_padding=True)``, for the padding tests.

A padded step counts for nothing, so the masked loss over N tokens is the reference loss over the valid tokens alone:
``masked_ppo_loss`` selects the valid rows and hands them to ``oracle.ref_optimizer.ppo_loss`` (or to the clipped-value
form of ``ppo_controls_oracle``), which makes the compaction identity the definition.  Gradients flow back through the
selection, so padded rows get exactly zero.  ``experiences_from_rollout`` is the reference prep with the terminal
bootstrap after the rollout's real last step instead of after its padding, and zero advantages / returns on padded rows.
"""
import numpy as np
import torch

import ppo_controls_oracle as PC
from oracle import ref_optimizer as RO

HEADS = PC.HEADS


def compact_old(dense_old, actions):
    """Dense ``[N, 5]`` old log-probs -> the reference's per-head vectors over each head's action rows, in row order."""
    return {k: dense_old[actions[k].bool().any(dim=-1), h] for h, k in enumerate(HEADS)}


def masked_ppo_loss(logits, values, actions, masks, dense_old, adv_raw, returns, valid, entropy_coef, vf_coef, e_clip,
                    old_values=None, value_clip=None):
    """Flat tokens: ``logits`` / ``actions`` / ``masks`` dicts of ``[N, n_h]``, ``values`` / ``adv_raw`` / ``returns`` /
    ``valid`` / ``old_values`` ``[N]``, ``dense_old`` ``[N, 5]``.  The reference loss over the rows where ``valid`` is
    True.  Returns (loss, policy_loss, entropy_loss, value_loss, entropies), differentiable in logits and values."""
    v = valid.reshape(-1).bool()
    lg = {k: logits[k][v].unsqueeze(0) for k in HEADS}
    act = {k: actions[k].bool()[v].unsqueeze(0) for k in HEADS}
    msk = {k: masks[k].bool()[v].unsqueeze(0) for k in HEADS}
    old = compact_old(dense_old[v], {k: a[0] for k, a in act.items()})
    ov = None if old_values is None else old_values.reshape(-1)[v].view(1, -1)
    return PC.ppo_loss(lg, values.reshape(-1)[v].view(1, -1, 1), act, msk, old, adv_raw.reshape(-1)[v].view(1, -1),
                       returns.reshape(-1)[v].view(1, -1), entropy_coef, vf_coef, e_clip, old_values=ov,
                       value_clip=value_clip)


def masked_stats(logits, actions, masks, dense_old, values, returns, valid, e_clip):
    """``last_ppo_stats`` over the valid rows (``ppo_controls_oracle.ppo_stats`` of the compacted tokens)."""
    v = valid.reshape(-1).bool()
    act = {k: actions[k].bool()[v] for k in HEADS}
    return PC.ppo_stats({k: logits[k][v] for k in HEADS}, {k: masks[k].bool()[v] for k in HEADS}, act,
                        compact_old(dense_old[v], act), values.reshape(-1)[v], returns.reshape(-1)[v], e_clip)


def real_advantage_returns(rewards, values, gamma=RO.GAMMA, lam=RO.LAMBDA):
    """GAE of one rollout's real steps: ``rewards`` ``[L]`` (summed sub-rewards) and ``values`` ``[L]``, each with the
    terminated rollout's trailing 0 appended after step L."""
    r = np.append(np.asarray(rewards, dtype=np.float32), np.float32(0.0))
    v = np.append(np.asarray(values, dtype=np.float32), np.float32(0.0))
    return RO.advantage_returns(r, v, gamma, lam)


def experiences_from_rollout(policy, data, seq_len):
    """The reference prep (``oracle.ref_optimizer.experiences_from_rollout``) with GAE over the real steps only; every
    sequence also carries ``valid`` ``[seq_len]`` bool."""
    seqs = RO.experiences_from_rollout(policy, data, seq_len)
    L = int(data["rewards"].shape[0])
    values = torch.cat([s.values.reshape(-1) for s in seqs]).numpy()
    rewards = np.concatenate([np.sum(s.rewards, axis=1).ravel() for s in seqs])          # optimizer.py:397
    adv, ret = real_advantage_returns(rewards[:L], values[:L])
    pad = len(seqs) * seq_len - L
    adv = np.concatenate([adv, np.zeros(pad, np.float32)])
    ret = np.concatenate([ret, np.zeros(pad, np.float32)])
    for j, s in enumerate(seqs):
        s.advantages = torch.from_numpy(adv[j * seq_len:(j + 1) * seq_len].copy())
        s.returns = torch.from_numpy(ret[j * seq_len:(j + 1) * seq_len].copy())
        s.valid = torch.arange(seq_len) < L - j * seq_len
    return seqs


class MaskedRefOptimizer(RO.RefOptimizer):
    """``oracle.ref_optimizer.RefOptimizer`` whose prep and loss leave padded steps out (any RefPolicy, stacked too)."""

    def experiences_from_rollout(self, data):
        return experiences_from_rollout(self.policy_base, data, self.seq_len)

    def loss_only(self, experiences):
        adv, ret, hidden, actions, masks, obs, _ = RO.stack_batch(experiences)
        valid = torch.stack([e.valid for e in experiences]).reshape(-1)
        logits, values, _ = self.policy(**obs, hidden=hidden)
        dense_old = torch.stack([seq_dense_old(e) for e in experiences]).reshape(-1, 5)
        flat = {k: t.reshape(-1, t.shape[-1]) for k, t in logits.items()}
        out = masked_ppo_loss(flat, values.reshape(-1), {k: a.reshape(flat[k].shape) for k, a in actions.items()},
                              {k: m.reshape(flat[k].shape) for k, m in masks.items()}, dense_old, adv.reshape(-1),
                              ret.reshape(-1), valid, self.entropy_coef, self.vf_coef, self.e_clip)
        return out, logits, values


def seq_dense_old(seq):
    """``[S, 5]`` dense old log-probs of a reference sequence (0 where a head took no action)."""
    S = seq.actions[HEADS[0]].shape[0]
    dense = torch.zeros(S, 5)
    for h, k in enumerate(HEADS):
        dense[seq.actions[k].bool().any(dim=-1), h] = seq.log_probs_sel[k]
    return dense
