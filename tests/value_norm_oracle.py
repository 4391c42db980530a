"""CPU / float64 oracle of ``DotaOptimizer(value_norm=True)`` (PopArt), for the value-normalisation tests.

The statistics are three float64 EMAs (m, q, w) of the value targets' mean and mean square and of their debias weight;
(mu, sigma) = (m / w, max(sqrt(q / w - mu^2), MIN_STD)), or (0, 1) before the first update.  One update per prepared
batch, from (n, sum R, sum R^2) over the tokens the value loss averages over.  After every update the value head is
rescaled so that sigma v + mu does not move (POP).  Prep reads the critic as V = mu + sigma v; the loss trains v on
(R - mu) / sigma with the statistics current at the step.  ``ValueNormRefOptimizer`` puts that on top of
``oracle.ref_optimizer.RefOptimizer``: GAE or V-trace prep of terminal rollouts, with or without the padding mask, and the
value loss clipped or not.
"""
import math

import numpy as np
import torch

import padding_oracle as PO
import vtrace_oracle as VT
from oracle import ref_optimizer as RO

HEADS = PO.HEADS
MIN_STD = 1e-2


def moments(state, min_std=MIN_STD):
    m, q, w = state
    if w == 0.0:
        return 0.0, 1.0
    mu = m / w
    var = q / w - mu * mu
    return mu, max(math.sqrt(var if var > 0.0 else 0.0), min_std)


def update(state, n, s1, s2, decay):
    if n == 0:
        return state
    m, q, w = state
    return (decay * m + (1.0 - decay) * (s1 / n), decay * q + (1.0 - decay) * (s2 / n), decay * w + (1.0 - decay))


def batch_sums(targets, valid=None):
    """(n, sum, sum of squares) in float64 of the fp32 ``targets`` where ``valid`` is True (all when None)."""
    x = np.asarray(targets, dtype=np.float32).reshape(-1).astype(np.float64)
    if valid is not None:
        x = x[np.asarray(valid, dtype=bool).reshape(-1)]
    return float(x.size), float(np.sum(x)), float(np.sum(x * x))


def rescale(weight, bias, old, new):
    """The POP step: fp32 (W sigma_old / sigma_new, (sigma_old b + mu_old - mu_new) / sigma_new) from float64."""
    w = np.asarray(weight, dtype=np.float32).astype(np.float64)
    b = np.asarray(bias, dtype=np.float32).astype(np.float64)
    return (w * old[1] / new[1]).astype(np.float32), ((old[1] * b + old[0] - new[0]) / new[1]).astype(np.float32)


def denorm(v, mu, sigma):
    """fp32(mu + sigma v) from float64."""
    return (mu + sigma * np.asarray(v, dtype=np.float32).astype(np.float64)).astype(np.float32)


def normalise(x, mu, sigma):
    """fp32((x - mu) / sigma) from float64: a raw target in the units of the normalised head."""
    return ((np.asarray(x, dtype=np.float32).astype(np.float64) - mu) / sigma).astype(np.float32)


class ValueNormRefOptimizer(RO.RefOptimizer):
    """``RefOptimizer`` with value normalisation.  ``prepare(rollouts)`` is one iteration's prep (and statistics update);
    ``train(sequences)`` one step.  ``estimator`` 'gae' or 'vtrace' (rollouts then carry ``behaviour_logp``),
    ``mask_padding`` leaves the padding of each rollout's last chunk out, ``value_clip`` clips the value loss."""

    def __init__(self, policy, seq_len, decay=0.99, estimator="gae", mask_padding=False, value_clip=None,
                 gamma=RO.GAMMA, lam=RO.LAMBDA, **kw):
        super().__init__(policy, seq_len, **kw)
        self.decay, self.estimator, self.mask_padding, self.value_clip = decay, estimator, mask_padding, value_clip
        self.gamma, self.lam = gamma, lam
        self.state = (0.0, 0.0, 0.0)

    @property
    def stats(self):
        return moments(self.state)

    def _prepare_one(self, data, mu, sigma):
        S = self.seq_len
        seqs = RO.experiences_from_rollout(self.policy_base, data, S)      # the forward; its targets are recomputed below
        L = int(data["rewards"].shape[0])
        Lp = len(seqs) * S
        for s in seqs:
            s.values = torch.from_numpy(denorm(s.values.numpy(), mu, sigma))
        values = np.concatenate([s.values.numpy().ravel() for s in seqs])
        rewards = np.concatenate([np.sum(s.rewards, axis=1).ravel() for s in seqs]).astype(np.float32)
        n = L if self.mask_padding else Lp                                  # the scan's rows, ending on the bootstrap of 0
        if self.estimator == "vtrace":
            dense = torch.cat([PO.seq_dense_old(s) for s in seqs]).numpy()
            acted = np.stack([np.concatenate([s.actions[k].numpy().reshape(S, -1).any(axis=1) for s in seqs])
                              for k in HEADS], axis=1)
            behaviour = np.zeros((Lp, 5), np.float32)
            behaviour[:L] = np.asarray(data["behaviour_logp"], np.float32)
            logrho = VT.log_rho(dense[:n], np.where(acted, behaviour, 0.0)[:n])
            adv, ret = VT.vtrace(rewards[:n], values[:n], logrho, self.gamma, self.lam)
            adv, ret = adv.astype(np.float32), ret.astype(np.float32)
        else:
            adv, ret = RO.advantage_returns(np.append(rewards[:n], np.float32(0)), np.append(values[:n], np.float32(0)),
                                            self.gamma, self.lam)
        adv = np.concatenate([adv, np.zeros(Lp - n, np.float32)])
        ret = np.concatenate([ret, np.zeros(Lp - n, np.float32)])
        for j, s in enumerate(seqs):
            s.advantages = torch.from_numpy(adv[j * S:(j + 1) * S].copy())
            s.returns = torch.from_numpy(ret[j * S:(j + 1) * S].copy())
            s.valid = torch.arange(S) < (L - j * S) if self.mask_padding else torch.ones(S, dtype=torch.bool)
        return seqs

    def prepare(self, rollouts):
        """Prep of one batch: values read under the current statistics, then the statistics update and the POP rescale.
        Returns the sequences, rollout by rollout."""
        mu, sigma = self.stats
        seqs = [s for r in rollouts for s in self._prepare_one(r, mu, sigma)]
        rets = np.concatenate([s.returns.numpy() for s in seqs])
        valid = np.concatenate([s.valid.numpy() for s in seqs])
        old = self.stats
        self.state = update(self.state, *batch_sums(rets, valid), self.decay)
        new = self.stats
        head = self.policy_base.affine_value
        w, b = rescale(head.weight.detach().numpy(), head.bias.detach().numpy(), old, new)
        with torch.no_grad():
            head.weight.copy_(torch.from_numpy(w))
            head.bias.copy_(torch.from_numpy(b))
        return seqs

    def loss_only(self, experiences):
        mu, sigma = self.stats
        adv, ret, hidden, actions, masks, obs, _ = RO.stack_batch(experiences)
        valid = torch.stack([e.valid for e in experiences]).reshape(-1)
        old_values = torch.stack([e.values.reshape(-1) for e in experiences]).reshape(-1)
        logits, values, _ = self.policy(**obs, hidden=hidden)
        dense_old = torch.stack([PO.seq_dense_old(e) for e in experiences]).reshape(-1, 5)
        flat = {k: t.reshape(-1, t.shape[-1]) for k, t in logits.items()}
        ret_n = torch.from_numpy(normalise(ret.reshape(-1).numpy(), mu, sigma))
        ov_n = torch.from_numpy(normalise(old_values.numpy(), mu, sigma))
        out = PO.masked_ppo_loss(flat, values.reshape(-1), {k: a.reshape(flat[k].shape) for k, a in actions.items()},
                                 {k: m.reshape(flat[k].shape) for k, m in masks.items()}, dense_old, adv.reshape(-1),
                                 ret_n, valid, self.entropy_coef, self.vf_coef, self.e_clip, old_values=ov_n,
                                 value_clip=self.value_clip)
        return out, logits, values
