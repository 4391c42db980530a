"""Float64 oracle of the advantage refresh between PPO epochs (``DotaOptimizer(recompute_advantages=True)``), on top of the
reference optimizer.

Before each epoch after the first, every chunk's values (and for V-trace the taken actions' log-probs) are recomputed with
the current network in float64, chunk by chunk from the chunk's stored initial state, as the reference's prep forward
runs them; then each rollout's GAE or V-trace runs again in float64, with the segments and bootstraps of prep: the real
steps end on prep's bootstrap (0 for a terminal rollout), and the padding is its own segment ending on 0 (or, for a
terminal rollout without ``mask_padding``, part of the one segment).  Under ``mask_padding`` padded rows stay 0.

``RefreshRefOptimizer`` is ``value_norm_oracle.ValueNormRefOptimizer`` (GAE or V-trace prep, ``mask_padding``, the masked
loss) with the value statistics optional and, for GAE, rollouts cut from a longer game (``continuation_oracle``: prep from
``'initial_hidden'``, the real steps of a non-terminal rollout bootstrapped from V(s_L) at prep, which the refresh keeps).
``train_epochs`` runs one iteration's epochs and minibatches with the refresh and, with ``kl_stop``, the early stop: a step
whose exact KL to the prep-time policy (``kl_oracle.exact_kl``, before its update) exceeds the limit is not applied and ends
the iteration, so no refresh follows it."""
import copy

import numpy as np
import torch

import continuation_oracle as CO
import kl_oracle as KO
import value_norm_oracle as VO
import vtrace_oracle as VT
from oracle import ref_optimizer as RO
from oracle.ref_policy import masked_softmax

HEADS = VO.HEADS


def gae(rewards, values, gamma, lam, boot=0.0):
    """One segment's GAE advantages and rewards-to-go in float64; the bootstrap ends both recursions."""
    r = VT.reward_sum(rewards).astype(np.float64)
    v = np.asarray(values, dtype=np.float64)
    n = v.shape[0]
    adv, ret = np.zeros(n), np.zeros(n)
    a, q, v_next = 0.0, float(boot), float(boot)
    for t in range(n - 1, -1, -1):
        a = r[t] + gamma * v_next - v[t] + gamma * lam * a
        q = r[t] + gamma * q
        adv[t], ret[t], v_next = a, q, v[t]
    return adv, ret


def chunk_forward(policy64, obs, masks, actions, hidden):
    """One ``S``-step chunk through a float64 copy of the network from its stored state: (values [S], the taken actions'
    log-probs [S, 5], 0 where a head took no action)."""
    hid = tuple(h.double() for h in hidden) if isinstance(hidden, tuple) else hidden.double()
    with torch.no_grad():
        logits, values, _ = policy64.sequence(**{k: v.double() for k, v in obs.items()}, hidden=hid)
        S = values.shape[1]
        dense = np.zeros((S, len(HEADS)))
        for h, k in enumerate(HEADS):
            lp = masked_softmax(logits[k], masks[k].bool().unsqueeze(0))[0]
            dense[:, h] = lp.masked_fill(~actions[k].bool(), 0.0).sum(dim=-1).numpy()
    return values.reshape(-1).numpy(), dense


def refresh_rollout(policy64, chunks, rewards, L, *, estimator, gamma, lam, mask_padding, terminal=True, boot=0.0,
                    behaviour=None, mu=0.0, sigma=1.0, rho_clip=1.0, c_clip=1.0):
    """The refreshed ``(advantages, returns)`` of one rollout, fp32 ``[Lp]``.  ``chunks``: ``(obs, masks, actions, hidden)``
    per chunk, rows ``[S, ...]``; ``rewards`` ``[>= L, n_sub]``; ``behaviour`` ``[L, 5]`` (V-trace); ``(mu, sigma)`` the value
    statistics the network's value head is normalised with (identity without value normalisation)."""
    vals, target, acted = [], [], []
    for obs, masks, actions, hidden in chunks:
        v, lp = chunk_forward(policy64, obs, masks, actions, hidden)
        vals.append(v)
        target.append(lp)
        acted.append(np.stack([actions[k].numpy().reshape(v.shape[0], -1).any(axis=1) for k in HEADS], axis=1))
    v = mu + sigma * np.concatenate(vals)
    target, acted = np.concatenate(target), np.concatenate(acted)
    Lp = v.shape[0]
    r = np.zeros((Lp, np.asarray(rewards).shape[1]), np.float32)
    r[:L] = np.asarray(rewards, np.float32)[:L]
    if estimator == "vtrace":
        b = np.zeros((Lp, len(HEADS)))
        b[:L] = np.asarray(behaviour, np.float64)[:L]
        logrho = VT.log_rho(target, np.where(acted, b, 0.0))

        def scan(lo, hi, bt):
            return VT.vtrace(r[lo:hi], v[lo:hi], logrho[lo:hi], gamma, lam, rho_clip, c_clip, bt)
    else:
        def scan(lo, hi, bt):
            return gae(r[lo:hi], v[lo:hi], gamma, lam, bt)
    adv, ret = np.zeros(Lp), np.zeros(Lp)
    segs = [(0, Lp, 0.0)] if terminal and not mask_padding else [(0, L, 0.0 if terminal else boot), (L, Lp, 0.0)]
    for lo, hi, bt in segs:
        if hi > lo:
            adv[lo:hi], ret[lo:hi] = scan(lo, hi, bt)
    if mask_padding:
        adv[L:], ret[L:] = 0.0, 0.0
    return adv.astype(np.float32), ret.astype(np.float32)


class RefreshRefOptimizer(VO.ValueNormRefOptimizer):
    """The reference optimizer with prep as ``ValueNormRefOptimizer`` (``value_norm=False``: statistics fixed at the
    identity, no update) or, when a rollout carries ``'initial_hidden'`` or ``'terminal': False``, as
    ``continuation_oracle`` (GAE, no value statistics); one iteration's ``train_epochs`` with the refresh (``recompute``)
    and the KL early stop (``kl_stop``)."""

    def __init__(self, policy, seq_len, value_norm=False, recompute=True, kl_stop=None, **kw):
        super().__init__(policy, seq_len, **kw)
        self.value_norm, self.recompute, self.kl_stop = value_norm, recompute, kl_stop
        self._ends = None

    @property
    def stats(self):
        return VO.moments(self.state) if self.value_norm else (0.0, 1.0)

    def prepare(self, rollouts):
        S = self.seq_len
        # (terminal, the bootstrap of the real steps) per rollout, as prep computed it
        self._ends = [(bool(d.get("terminal", True)),
                       0.0 if d.get("terminal", True) else float(CO.bootstrap_value(self.policy_base, d))) for d in rollouts]
        if any("initial_hidden" in d or not d.get("terminal", True) for d in rollouts):
            assert not self.value_norm and self.estimator == "gae"
            seqs = [s for d in rollouts for s in CO.experiences_from_rollout(self.policy_base, d, S, self.mask_padding)]
            for s in seqs:
                if getattr(s, "valid", None) is None:
                    s.valid = torch.ones(S, dtype=torch.bool)
        elif self.value_norm:
            seqs = super().prepare(rollouts)
        else:
            seqs = [s for r in rollouts for s in self._prepare_one(r, 0.0, 1.0)]
        if self.kl_stop is not None:                    # the prep-time distribution the KL is measured against
            with torch.no_grad():
                for s in seqs:
                    logits, _, _ = self.policy_base.sequence(**s.observations, hidden=s.hidden)
                    s.old_rows = KO.masked_log_rows({k: v[0] for k, v in logits.items()}, s.masks)
        return seqs

    def refresh(self, seqs, rollouts):
        """Rewrites the advantages and returns of ``seqs`` (rollout by rollout, chunk by chunk) with the current weights."""
        policy64 = copy.deepcopy(self.policy_base).double()
        mu, sigma = self.stats
        S, j = self.seq_len, 0
        for data, (terminal, boot) in zip(rollouts, self._ends):
            L = int(data["rewards"].shape[0])
            n = (L + S - 1) // S
            mine = seqs[j:j + n]
            chunks = [(s.observations, s.masks, s.actions, s.hidden) for s in mine]
            adv, ret = refresh_rollout(policy64, chunks, data["rewards"], L, estimator=self.estimator, gamma=self.gamma,
                                       lam=self.lam, mask_padding=self.mask_padding, terminal=terminal, boot=boot,
                                       behaviour=data.get("behaviour_logp"), mu=mu, sigma=sigma)
            for c, s in enumerate(mine):
                s.advantages = torch.from_numpy(adv[c * S:(c + 1) * S].copy())
                s.returns = torch.from_numpy(ret[c * S:(c + 1) * S].copy())
            j += n

    def kl(self, experiences):
        """The exact KL of a minibatch to the prep-time policy at the current weights (float64)."""
        _, _, hidden, actions, masks, obs, _ = RO.stack_batch(experiences)
        with torch.no_grad():
            logits, _, _ = self.policy(**obs, hidden=hidden)
        flat = lambda d: {k: v.reshape(-1, v.shape[-1]) for k, v in d.items()}       # noqa: E731
        rows = torch.cat([e.old_rows for e in experiences])
        valid = torch.cat([e.valid.reshape(-1) for e in experiences])
        return float(KO.exact_kl(flat(logits), flat(actions), flat(masks), rows, valid)[0])

    def train_epochs(self, seqs, rollouts, epochs, num_minibatches, rng):
        """``epochs`` passes of ``num_minibatches`` minibatches (``minibatch_indices`` with ``rng``), the refresh before every
        pass after the first.  Returns the per-step ``(losses, entropies, grad_norms)``; a step that ``kl_stop`` stops is
        the last, with its losses at the weights it left unchanged and grad_norms None."""
        from dotaclient_b200.optimizer import minibatch_indices
        out = []
        for ep in range(epochs):
            if self.recompute and ep > 0:
                self.refresh(seqs, rollouts)
            for idx in minibatch_indices(len(seqs), num_minibatches, rng):
                batch = [seqs[i] for i in idx]
                if self.kl_stop is not None and self.kl(batch) > self.kl_stop:
                    (loss, p_loss, e_loss, v_loss, ents), _, _ = self.loss_only(batch)
                    out.append(({"loss": loss, "policy_loss": p_loss, "entropy_loss": e_loss, "value_loss": v_loss},
                                ents, None))
                    return out
                out.append(self.train(batch))
        return out
