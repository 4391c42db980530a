"""Float64 numpy restatement of the value heads (``DotaOptimizer(value_heads=...)``): the group rewards, the per-group GAE
scans over prep's segments with their bootstraps, the summed advantage, the K-head value loss with mask and clip and its
statistics, and the fold and split of the value head.  Test infrastructure only."""
import numpy as np

f32 = np.float32


def group_rewards(rewards, group, K):
    """[n, K] fp32: r_k = numpy's fp32 sum over the row of the group's columns, idx_k ascending, as np.sum(rewards, axis=1)
    reduces a row (pairwise).  The gathered columns are made C-contiguous first: ``rewards[:, idx]`` alone is laid out
    column-major, and numpy then sums its rows sequentially instead."""
    rewards = np.asarray(rewards, dtype=f32)
    return np.stack([np.ascontiguousarray(rewards[:, np.flatnonzero(np.asarray(group) == k)]).sum(axis=1)
                     for k in range(K)], axis=1)


def scan_heads(rewards, values, seg_off, group, gammas, lam, boot_value=None, boot_reward=None):
    """Per segment and group: delta in fp32 with numpy's three roundings, A_k = delta + g_k lam A_k', R_k = r + g_k R_k'
    in float64 from the segment's bootstraps.  Returns (adv [n] = fp32(sum_k A_k), ret [n, K] fp32) and the float64
    (adv, ret) before rounding."""
    values = np.asarray(values, dtype=f32)
    n, K = values.shape
    r = group_rewards(rewards, group, K)
    adv64, ret64 = np.zeros(n), np.zeros((n, K))
    for s in range(len(seg_off) - 1):
        lo, hi = int(seg_off[s]), int(seg_off[s + 1])
        for k in range(K):
            g = float(gammas[k])
            bv = f32(0.0) if boot_value is None else f32(np.asarray(boot_value, dtype=f32).reshape(-1, K)[s, k])
            br = 0.0 if boot_reward is None else float(np.asarray(boot_reward, dtype=f32).reshape(-1, K)[s, k])
            a, q, v_next = 0.0, br, bv
            for t in range(hi - 1, lo - 1, -1):
                delta = (r[t, k] + f32(g) * v_next) - values[t, k]        # fp32, three roundings
                a = float(delta) + g * lam * a
                q = float(r[t, k]) + g * q
                adv64[t] += a
                ret64[t, k] = q
                v_next = values[t, k]
    return adv64.astype(f32), ret64.astype(f32), adv64, ret64


def value_heads_loss(v, ret, vf_coef, old_value=None, value_clip=0.0, valid=None):
    """The K-head value loss in float64: (loss = vf_coef sum_k 0.5 mean (R_k - V_k)^2 or its PPO2-clipped form, dvalue
    [N, K] (0 where not valid), per-head losses [K], per-head explained variances [K], explained variance of the sums)."""
    v, ret = np.asarray(v, np.float64), np.asarray(ret, np.float64)
    N, K = v.shape
    m = np.ones(N, bool) if valid is None else np.asarray(valid, bool)
    n = m.sum()
    d = v - ret
    l = d * d
    g = d.copy()
    if old_value is not None and value_clip > 0:
        vo = np.asarray(old_value, np.float64)
        dv = v - vo
        dc = vo + np.clip(dv, -value_clip, value_clip) - ret
        l2 = dc * dc
        w1 = np.where(l > l2, 1.0, np.where(l == l2, 0.5, 0.0))
        w2 = np.where(l2 > l, 1.0, np.where(l == l2, 0.5, 0.0))
        g = w1 * d + w2 * ((dv >= -value_clip) & (dv <= value_clip)) * dc
        l = np.maximum(l, l2)
    heads = vf_coef * 0.5 * l[m].sum(axis=0) / n
    dvalue = np.where(m[:, None], vf_coef * g / n, 0.0)

    def ev(r, pred):
        var_r = r.var()
        return 1.0 - (r - pred).var() / var_r if var_r > 0 else np.nan
    ev_heads = np.array([ev(ret[m, k], v[m, k]) for k in range(K)])
    ev_total = ev(ret[m].sum(axis=1), v[m].sum(axis=1))
    return heads.sum(), dvalue, heads, ev_heads, ev_total


def fold(weight, bias):
    """The one-row head of K rows, float64: (sum_k W_k [1, H], sum_k b_k [1])."""
    return np.asarray(weight, np.float64).sum(axis=0, keepdims=True), np.asarray(bias, np.float64).sum(keepdims=True)[:1]


def split(weight, bias, K):
    """K rows of W / K and b / K from a one-row head, float64."""
    w, b = np.asarray(weight, np.float64), np.asarray(bias, np.float64)
    return np.repeat(w / K, K, axis=0), np.repeat(b / K, K)
