"""Float64 oracle of the state refresh between PPO epochs (``DotaOptimizer(recompute_states=True)``), on top of
``refresh_oracle`` and ``continuation_oracle``.

Each rollout is rerun whole, in float64, with the current weights, from the state prep started it from (zeros or its
``'initial_hidden'``), over its padded length (zero observations after its real steps, as prep pads).  Its states at every
chunk start are the refreshed ``h0`` / ``c0`` / reset rows, and they feed both the chunks and, with
``recompute_advantages``, the scan (``refresh_oracle.refresh_rollout``); a cut rollout's V(s_L) comes from the state after
its last real step and its extra observation row."""
import copy

import numpy as np
import torch

import refresh_oracle as RF


def _double(h):
    return tuple(x.double() for x in h) if isinstance(h, tuple) else h.double()


def _padded_rows(t, L, Lp):
    t = torch.as_tensor(t)[:L]
    return torch.cat([t, torch.zeros((Lp - L,) + tuple(t.shape[1:]), dtype=t.dtype)])


def rollout_states(policy64, rollout, S, start):
    """The float64 states entering every ``S``-step chunk of ``rollout`` (its padded length) run whole from ``start``
    (``Policy.init_hidden()`` structure), and the state after its ``L`` real steps: ``(states, after_L)``."""
    L = int(rollout["rewards"].shape[0])
    Lp = (L + S - 1) // S * S
    obs = {k: _padded_rows(v, L, Lp).double() for k, v in rollout["observations"].items()}
    h = _double(start)
    states = []
    with torch.no_grad():
        for j in range(Lp // S):
            states.append(h)
            _, _, h = policy64.sequence(**{k: v[j * S:(j + 1) * S] for k, v in obs.items()}, hidden=h)
        h = _double(start)
        _, _, after = policy64.sequence(**{k: v[:L] for k, v in obs.items()}, hidden=h)
    return states, after


def refreshed_advantages(policy64, rollout, S, start, *, estimator, mask_padding, mu=0.0, sigma=1.0, gamma=0.98,
                         lam=0.97):
    """The advantages and returns of one rollout after the state refresh with ``recompute_advantages``: every chunk from
    its refreshed state, and for a cut rollout the bootstrap V(s_L) from the refreshed state after step L."""
    L = int(rollout["rewards"].shape[0])
    Lp = (L + S - 1) // S * S
    states, after = rollout_states(policy64, rollout, S, start)
    terminal = bool(rollout.get("terminal", True))
    boot = 0.0
    if not terminal:
        with torch.no_grad():
            _, v, _ = policy64.sequence(**{k: torch.as_tensor(v)[L:L + 1].double()
                                           for k, v in rollout["observations"].items()}, hidden=after)
        boot = mu + sigma * float(v.reshape(-1)[0])
    chunks = []
    for j in range(Lp // S):
        sl = slice(j * S, (j + 1) * S)
        chunks.append(({k: _padded_rows(v, L, Lp)[sl] for k, v in rollout["observations"].items()},
                       {k: _padded_rows(v, L, Lp)[sl] for k, v in rollout["masks"].items()},
                       {k: _padded_rows(v, L, Lp)[sl] for k, v in rollout["actions"].items()}, states[j]))
    return RF.refresh_rollout(policy64, chunks, rollout["rewards"], L, estimator=estimator, gamma=gamma, lam=lam,
                              mask_padding=mask_padding, terminal=terminal, boot=boot,
                              behaviour=rollout.get("behaviour_logp"), mu=mu, sigma=sigma)


def drift(new, old):
    """sqrt(sum (new - old)^2 / sum old^2) in float64 over matching tensors."""
    num = sum(float(((n.double() - o.double()) ** 2).sum()) for n, o in zip(new, old))
    den = sum(float((o.double() ** 2).sum()) for o in old)
    return float(np.sqrt(num / den)) if den > 0 else 0.0


class StateRefreshRefOptimizer(RF.RefreshRefOptimizer):
    """``refresh_oracle.RefreshRefOptimizer`` with the state refresh before every epoch after the first: each rollout is
    rerun whole in float64 with the current weights from its prep start state (``rollout_states``), and every chunk after
    its first starts from the refreshed state.  ``recompute_advantages``: the advantages and returns are recomputed from
    the same states, a cut rollout's V(s_L) from the refreshed state after step L (``refreshed_advantages``); otherwise
    they stay as prep made them.  The old log-probs, the prep-time rows of the KL and the value statistics stay."""

    def __init__(self, policy, seq_len, recompute_advantages=False, **kw):
        super().__init__(policy, seq_len, recompute=True, **kw)
        self.recompute_advantages = recompute_advantages

    def refresh(self, seqs, rollouts):
        policy64 = copy.deepcopy(self.policy_base).double()
        mu, sigma = self.stats
        S, j = self.seq_len, 0
        for data in rollouts:
            L = int(data["rewards"].shape[0])
            n = (L + S - 1) // S
            mine = seqs[j:j + n]
            start = data.get("initial_hidden", self.policy_base.init_hidden())
            states, _ = rollout_states(policy64, data, S, start)
            for c in range(1, n):                        # the first chunk keeps prep's start state
                old = mine[c].hidden
                if isinstance(old, tuple):
                    mine[c].hidden = tuple(s.to(o.dtype).reshape(o.shape) for s, o in zip(states[c], old))
                else:
                    mine[c].hidden = states[c].to(old.dtype).reshape(old.shape)
            if self.recompute_advantages:
                adv, ret = refreshed_advantages(policy64, data, S, start, estimator=self.estimator,
                                                mask_padding=self.mask_padding, mu=mu, sigma=sigma, gamma=self.gamma,
                                                lam=self.lam)
                for c, s in enumerate(mine):
                    s.advantages = torch.from_numpy(adv[c * S:(c + 1) * S].copy())
                    s.returns = torch.from_numpy(ret[c * S:(c + 1) * S].copy())
            j += n
