"""Oracles of experience prep on rollouts cut from a longer game (``'initial_hidden'``, ``'terminal': False``).

``gae`` is a float64 numpy GAE with a bootstrap: the advantages bootstrap from ``boot_value`` (V of the state after the
last row) and the returns go on past the last row as ``gamma^(n-t) * boot_reward``; V-trace with a bootstrap is
``vtrace_oracle.vtrace(..., boot=)``.  ``experiences_from_rollout`` is the reference prep (``oracle.ref_optimizer``)
started from the rollout's initial state, whose real steps bootstrap from the reference policy's value of the extra
observation row when the rollout is not terminal; its padding is scanned on its own and ends on 0.
"""
import numpy as np
import torch

import padding_oracle as PO
from oracle import ref_optimizer as RO


def gae(rewards, values, gamma, lam, boot_value=0.0, boot_reward=0.0):
    """One segment -> float64 ``(advantages, returns)``.  ``rewards`` / ``values`` ``[n]``."""
    r = np.asarray(rewards, dtype=np.float64)
    v = np.append(np.asarray(values, dtype=np.float64), float(boot_value))
    n = r.shape[0]
    adv, ret = np.zeros(n), np.zeros(n)
    a, q = 0.0, float(boot_reward)
    for t in range(n - 1, -1, -1):
        a = r[t] + gamma * v[t + 1] - v[t] + gamma * lam * a
        q = r[t] + gamma * q
        adv[t], ret[t] = a, q
    return adv, ret


def initial_hidden(policy, data):
    """The state the rollout starts from, as the reference policy takes it: ``'initial_hidden'`` or the zero state."""
    h = data.get("initial_hidden")
    if h is None:
        return policy.init_hidden()
    return tuple(torch.as_tensor(x).float() for x in h) if isinstance(h, (tuple, list)) else torch.as_tensor(h).float()


def bootstrap_value(policy, data):
    """V(s_L) of a non-terminal rollout: the reference policy run over its L steps from its initial state, then one
    step on observation row L.  fp32."""
    L = int(data["rewards"].shape[0])
    obs = data["observations"]
    with torch.no_grad():
        _, _, h = policy.sequence(hidden=initial_hidden(policy, data), **{k: v[:L] for k, v in obs.items()})
        _, value, _ = policy.sequence(hidden=h, **{k: v[L:L + 1] for k, v in obs.items()})
    return np.float32(value.reshape(-1)[0])


def experiences_from_rollout(policy, data, seq_len, mask_padding=False):
    """Reference prep of a rollout of the wire format with the two optional keys: the chunk-by-chunk forward of
    ``oracle.ref_optimizer.experiences_from_rollout`` from ``initial_hidden``, then GAE over the real steps ending on the
    bootstrap (0 when terminal) and over the padding ending on 0 -- one scan of both when the rollout is terminal and
    ``mask_padding`` is off, as the reference.  With ``mask_padding`` padded rows get 0 and sequences carry ``valid``."""
    L = int(data["rewards"].shape[0])
    terminal = data.get("terminal", True)
    real = dict(data, observations={k: v[:L] for k, v in data["observations"].items()})
    init = initial_hidden(policy, data)
    saved = policy.init_hidden
    policy.init_hidden = lambda: init                   # RO's chunk loop starts from policy.init_hidden()
    try:
        seqs = RO.experiences_from_rollout(policy, real, seq_len)
    finally:
        policy.init_hidden = saved
    values = torch.cat([s.values.reshape(-1) for s in seqs]).numpy()
    rewards = np.concatenate([np.sum(s.rewards, axis=1).ravel() for s in seqs])           # optimizer.py:397
    if terminal and not mask_padding:
        return seqs                                                                         # RO's own scan
    b = np.float32(0.0) if terminal else bootstrap_value(policy, data)
    adv, ret = RO.advantage_returns(np.append(rewards[:L], b), np.append(values[:L], b))
    pad = len(seqs) * seq_len - L
    if pad and not mask_padding:
        a2, r2 = RO.advantage_returns(np.append(rewards[L:], np.float32(0)), np.append(values[L:], np.float32(0)))
    else:
        a2, r2 = np.zeros(pad, np.float32), np.zeros(pad, np.float32)
    adv, ret = np.concatenate([adv, a2]), np.concatenate([ret, r2])
    for j, s in enumerate(seqs):
        s.advantages = torch.from_numpy(adv[j * seq_len:(j + 1) * seq_len].copy())
        s.returns = torch.from_numpy(ret[j * seq_len:(j + 1) * seq_len].copy())
        if mask_padding:
            s.valid = torch.arange(seq_len) < L - j * seq_len
    return seqs


class ContinuationRefOptimizer(RO.RefOptimizer):
    """``oracle.ref_optimizer.RefOptimizer`` with this prep; with ``mask_padding`` the loss leaves padded steps out
    (``padding_oracle``)."""

    def __init__(self, policy, seq_len, mask_padding=False, **kw):
        super().__init__(policy, seq_len, **kw)
        self.mask_padding = mask_padding

    def experiences_from_rollout(self, data):
        return experiences_from_rollout(self.policy_base, data, self.seq_len, self.mask_padding)

    def loss_only(self, experiences):
        if self.mask_padding:
            return PO.MaskedRefOptimizer.loss_only(self, experiences)
        return super().loss_only(experiences)
