"""Float64 numpy UPGO (the upgoing policy update of AlphaStar, Vinyals et al. 2019): the CPU oracle of ``dc_upgo_scan``
and of experience prep with ``DotaOptimizer(upgo_coef=c)``.

One segment at a time, a plain backward loop over its rows lo .. hi-1, with V_hi = boot:
    delta_t   = r_t + gamma V_{t+1} - V_t                      float64, no FMA
    through_t = (t + 1 < hi) and (delta_{t+1} >= 0)
    G_t       = r_t + gamma * (through_t ? G_{t+1} : V_{t+1})
    A^U_t     = rhob_t * (G_t - V_t)
rhob_t = 1 (GAE) or V-trace's min(rho_clip, exp(log rho_t)) (``vtrace_oracle``).  Prep's advantage is then
fp32((double)A_base_t + c A^U_t).
"""
import numpy as np

import vtrace_oracle as VT

STATS_SLOTS = 3


def upgo(rewards, values, gamma, boot=0.0, logrho=None, rho_clip=1.0):
    """One segment -> ``(A^U, through)`` in float64 / bool.  ``rewards`` [n] or [n, n_sub] fp32, ``values`` [n] fp32,
    ``logrho`` [n] float64 or None (GAE: rhob = 1)."""
    r = VT.reward_sum(rewards).astype(np.float64)
    v = np.asarray(values, dtype=np.float32).astype(np.float64)
    n = v.shape[0]
    v_next = np.append(v[1:], float(np.float32(boot)))
    delta = (r + gamma * v_next) - v
    through = np.zeros(n, bool)
    through[:-1] = delta[1:] >= 0
    g = np.zeros(n)
    g_next = 0.0
    for t in range(n - 1, -1, -1):
        g[t] = r[t] + gamma * (g_next if through[t] else v_next[t])
        g_next = g[t]
    rhob = np.ones(n)
    if logrho is not None:
        with np.errstate(over='ignore'):
            rhob = VT._clip(np.exp(np.asarray(logrho, dtype=np.float64)), rho_clip)
    return rhob * (g - v), through


def advantages(base, au, coef):
    """Prep's advantage: the base scan's fp32 advantage plus ``coef`` A^U in float64, rounded once."""
    return (np.asarray(base, np.float32).astype(np.float64) + coef * np.asarray(au, np.float64)).astype(np.float32)


def stats(au, through):
    """The ``DC_UPGO_STATS_SLOTS`` sums of one segment's real steps: count, #through, sum A^U."""
    return np.array([au.size, np.sum(through), np.sum(au)], dtype=np.float64)


def discounted_return(rewards, gamma, boot=0.0):
    """sum_k gamma^k r_{t+k} + gamma^(n-t) boot per row, in float64."""
    r = VT.reward_sum(rewards).astype(np.float64)
    out = np.zeros(r.size)
    acc = float(np.float32(boot))
    for t in range(r.size - 1, -1, -1):
        acc = r[t] + gamma * acc
        out[t] = acc
    return out
