"""Float64 numpy V-trace (Espeholt et al. 2018): the CPU oracle of ``dc_vtrace_scan`` and of the V-trace experience prep.

One rollout (segment) at a time, a plain backward loop over its rows:
    log rho_t = sum_h (lp_target[t, h] - lp_behaviour[t, h])          heads in order, float64
    rhob_t    = min(rho_clip, rho_t),  c_t = lam * min(c_clip, rho_t)
    vs_t      = V_t + rhob_t (r_t + gamma V_{t+1} - V_t) + gamma c_t (vs_{t+1} - V_{t+1}),   vs_L = V_L = boot
    A_t       = rhob_t (r_t + gamma vs_{t+1} - V_t)
"""
import numpy as np

STATS_SLOTS = 8


def reward_sum(rewards):
    """The per-step reward of the scans: numpy's fp32 sum over the sub-rewards (``optimizer.py:397``)."""
    rewards = np.asarray(rewards, dtype=np.float32)
    return rewards if rewards.ndim == 1 else np.sum(rewards, axis=1)


def log_rho(lp_target, lp_behaviour):
    """float64 log importance weight per row from two dense ``[n, 5]`` log-prob arrays, summed over the heads in order."""
    d = np.asarray(lp_target, dtype=np.float64) - np.asarray(lp_behaviour, dtype=np.float64)
    out = np.zeros(d.shape[0])
    for h in range(d.shape[1]):
        out += d[:, h]
    return out


def _clip(rho, level):
    return np.where(rho > level, level, rho)          # min(level, rho) that keeps NaN, like the kernel


def vtrace(rewards, values, logrho, gamma, lam, rho_clip=1.0, c_clip=1.0, boot=0.0):
    """One segment -> ``(pg_adv, vs)`` in float64.  ``rewards`` [n] or [n, n_sub] fp32, ``values`` [n] fp32."""
    r = reward_sum(rewards).astype(np.float64)
    v = np.asarray(values, dtype=np.float32).astype(np.float64)
    with np.errstate(over='ignore'):
        rho = np.exp(np.asarray(logrho, dtype=np.float64))
    rhob, c = _clip(rho, rho_clip), lam * _clip(rho, c_clip)
    n = v.shape[0]
    boot = float(np.float32(boot))
    vs = np.zeros(n)
    pg = np.zeros(n)
    vs_next, v_next = boot, boot
    for t in range(n - 1, -1, -1):
        vs[t] = v[t] + rhob[t] * (r[t] + gamma * v_next - v[t]) + gamma * c[t] * (vs_next - v_next)
        pg[t] = rhob[t] * (r[t] + gamma * vs_next - v[t])
        vs_next, v_next = vs[t], v[t]
    return pg, vs


def stats(logrho, rho_clip=1.0, c_clip=1.0):
    """The ``DC_VTRACE_STATS_SLOTS`` sums of one segment's real steps: count, sum log rho, sum rhob, #(rho > rho_clip),
    #(rho > c_clip), then zeros."""
    logrho = np.asarray(logrho, dtype=np.float64)
    with np.errstate(over='ignore'):
        rho = np.exp(logrho)
    out = np.zeros(STATS_SLOTS)
    out[:5] = [logrho.size, logrho.sum(), _clip(rho, rho_clip).sum(), (rho > rho_clip).sum(), (rho > c_clip).sum()]
    return out


def summary(seg_stats):
    """``DotaOptimizer.last_vtrace_stats`` from per-segment sums."""
    s = np.sum(np.asarray(seg_stats, dtype=np.float64).reshape(-1, STATS_SLOTS), axis=0)
    n = max(s[0], 1.0)
    return {'mean_log_rho': s[1] / n, 'mean_clipped_rho': s[2] / n, 'rho_clip_fraction': s[3] / n,
            'c_clip_fraction': s[4] / n}
