"""Experience prep (``DotaOptimizer._prepare_rollouts`` through ``batch_from_rollouts``, ``mask_padding=True``) at the
benchmark's scale, against a float64 reference over whole rollouts.

Prep has its own forward: the recurrence keeps every step's state (``rnn_stack_forward_states``), the encoder stores
nothing for backward, chunk-entry states are read at ``ybufs[k][j*S]``, a cut rollout's bootstrap value is one more step
from its state after the cut, then ``selected_logp`` and the segmented GAE or V-trace scan.  Two regimes, hidden 128
LSTM, S 512: 256 ragged rollouts of 300 to 512 steps, and 32 rollouts of 3585 to 4096 steps (256 chunks; the forward
runs B 32 x S 4096).  Every second rollout is cut mid-game (``split_rollout``) and starts from an ``initial_hidden``.

For 6 sampled rollouts (cut and terminal ones) the reference is ``StackedRefPolicy`` in float64 over the whole rollout,
chunk by chunk with the state carried, plus the extra step after a cut, followed by GAE (``advantage_returns``' recursions
in float64) or ``vtrace_oracle.vtrace``.  The same reference in fp32 calibrates the bound of ``test_gpu_step_fp64``:

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

K and FLOOR (``BOUNDS``): 32 and 2e-6 for values (a cut rollout's bootstrap V(s_L) appended), old log-probabilities,
advantages and returns; 32 and 1e-6 for the chunk-entry states.  Measured on one H100 80GB HBM3 (700 W power limit), the
largest ratio max|gpu - f64| / max|torch32 - f64|, values / old_logp / advantages / returns / h0 / c0, and the wall time:
    ragged-gae (and -packed)  11 /  8.3 /  9.7 / 33 /  -  /  -    4 s
    ragged-vtrace             12 /  9.1 /  11  / 14 /  -  /  -    4 s
    long-gae                  14 /  10  /  12  / 6.6 / 16 / 20    8 s
    long-vtrace               14 /  11  /  8.9 / 14 / 16 / 21    7 s
(A ragged rollout is one chunk: its entry state is its initial_hidden, exact.)  The returns' ratio of 33 is at
max|gpu - f64| = 6e-7 of max|f64|, inside the floor.
"""
import copy
import gc
import time
import uuid

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import vtrace_oracle as VT
from stacked_oracle import StackedRefPolicy
from test_gpu_encoder import _grid
from test_gpu_ppo_fp64 import HEADS, log_softmax
from test_gpu_rnn_fp64 import bound_check
from test_gpu_step_fp64 import grid_encoder

S, H, CELL = 512, 128, "lstm"
GAMMA, LAMBDA = 0.98, 0.97
# (K, FLOOR): critic values (a cut rollout's bootstrap value V(s_L) appended to its values) and old log-probabilities;
# advantages and returns; chunk-entry states
BOUNDS = {"forward": (32.0, 2e-6), "scan": (32.0, 2e-6), "state": (32.0, 1e-6)}
KINDS = {"values": "forward", "old_logp": "forward", "advantages": "scan", "returns": "scan", "h0": "state", "c0": "state"}

# (id, number of rollouts, length range, estimator, pack_sequences)
REGIMES = [
    ("ragged-gae", 256, (300, 512), "gae", False),
    ("ragged-vtrace", 256, (300, 512), "vtrace", False),
    ("ragged-gae-packed", 256, (300, 512), "gae", True),
    ("long-gae", 32, (3585, 4096), "gae", False),
    ("long-vtrace", 32, (3585, 4096), "vtrace", False),
]


def make_rollouts(n, lengths, seed, vtrace):
    """Rollouts with grid observations; every even one is cut mid-game (non-terminal, an extra observation row) and every
    one starts from a non-zero ``initial_hidden``."""
    from dotaclient_b200.synthetic import make_rollout, split_rollout
    rng = np.random.RandomState(seed)
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        L = int(rng.randint(lengths[0], lengths[1] + 1))
        cut = i % 2 == 0
        r = make_rollout(L + (1 if cut else 0), 1000 * seed + i, game_id=i)
        for k, v in r["observations"].items():
            r["observations"][k] = _grid(g, v.shape, 48, 16) if k == "env" else _grid(g, v.shape, 4, 4)
        if vtrace:
            r["behaviour_logp"] = -torch.rand(L + (1 if cut else 0), 5, generator=g).numpy()
        if cut:
            r = split_rollout(r, [L])[0]
        h = 0.5 * torch.randn(1, 1, H, generator=g)
        r["initial_hidden"] = (h, 0.5 * torch.randn(h.shape, generator=g))
        out.append(r)
    return out


def gae(rewards, values, boot):
    """float64 GAE-lambda and rewards-to-go of one rollout with ``boot`` after its last step (0 when terminal)."""
    r = np.append(np.sum(np.asarray(rewards, dtype=np.float32), axis=1).astype(np.float64), boot)
    v = np.append(np.asarray(values, dtype=np.float64), boot)
    deltas = r[:-1] + GAMMA * v[1:] - v[:-1]
    adv = lfilter([1], [1, -GAMMA * LAMBDA], deltas[::-1])[::-1]
    ret = lfilter([1], [1, -GAMMA], r[::-1])[::-1][:-1]
    return adv, ret


def ref_rollout(pol, data, dtype, vtrace):
    """One whole rollout under ``pol`` in ``dtype`` -> {values, old_logp [L, 5], advantages, returns, h0 / c0 entering
    every chunk [n_chunks, H], bootstrap (cut rollouts)}."""
    L = int(data["rewards"].shape[0])
    cut = not data.get("terminal", True)
    obs = {k: torch.as_tensor(v).to(dtype).unsqueeze(0) for k, v in data["observations"].items()}
    h, c = (t.to(dtype) for t in data["initial_hidden"])
    hs, cs, values, lps = [], [], [], []
    with torch.no_grad():
        for t0 in range(0, L, S):
            hs.append(h[0, 0])
            cs.append(c[0, 0])
            t1 = min(t0 + S, L)
            lg, v, (h, c) = pol(**{k: o[:, t0:t1] for k, o in obs.items()}, hidden=(h, c))
            values.append(v[0, :, 0])
            sel = []
            for k in HEADS:
                m = torch.as_tensor(data["masks"][k][t0:t1]).bool()
                a = torch.as_tensor(data["actions"][k][t0:t1]).bool()
                sel.append(torch.where(a, log_softmax(lg[k][0], m), torch.zeros((), dtype=dtype)).sum(1))
            lps.append(torch.stack(sel, 1))
        boot = float(pol(**{k: o[:, L:L + 1] for k, o in obs.items()}, hidden=(h, c))[1][0, 0, 0]) if cut else 0.0
    values, old = torch.cat(values), torch.cat(lps)
    if vtrace:
        acted = np.stack([np.asarray(data["actions"][k]).any(1) for k in HEADS], 1)
        beh = np.where(acted, np.asarray(data["behaviour_logp"], dtype=np.float32), 0.0)
        adv, ret = VT.vtrace(data["rewards"], values.double().numpy(), VT.log_rho(old.double().numpy(), beh), GAMMA,
                             LAMBDA, boot=boot)
    else:
        adv, ret = gae(data["rewards"], values.double().numpy(), boot)
    out = {"values": values, "old_logp": old, "advantages": torch.from_numpy(np.ascontiguousarray(adv)),
           "returns": torch.from_numpy(np.ascontiguousarray(ret)), "h0": torch.stack(hs), "c0": torch.stack(cs)}
    if cut:
        out["values"] = torch.cat([values, torch.tensor([boot], dtype=dtype)])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_prep_vs_fp64(regime, tmp_path):
    from dotaclient_b200.optimizer import DotaOptimizer
    name, n, lengths, estimator, packed = regime
    t0 = time.perf_counter()
    gc.collect()
    torch.cuda.empty_cache()
    opt = DotaOptimizer(rmq_host="prep-fp64", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=1,
                        seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                        log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H, cell=CELL,
                        mask_padding=True, advantage_estimator=estimator, pack_sequences=packed)
    grid_encoder(opt.policy_base, 17)
    rollouts = make_rollouts(n, lengths, n + lengths[0], estimator == "vtrace")
    captured = {}
    prepare = opt._prepare_rollouts

    def keep(datas):
        captured["p"] = prepare(datas)
        return captured["p"]
    opt._prepare_rollouts = keep
    batch = opt.batch_from_rollouts(copy.deepcopy(rollouts))
    p = captured["p"]
    Ls, Lps = p["Ls"], p["Lps"]
    assert int(batch.valid.sum()) == sum(Ls)
    if not packed:
        assert batch.batch_size == sum(lp // S for lp in Lps)
    cut = [i for i, d in enumerate(rollouts) if not d.get("terminal", True)]

    sampled = (0, 1, 2, n // 2 - 1, n // 2, n - 1)
    sd = {k: v.detach().cpu() for k, v in opt.policy_base.state_dict().items()}
    got, f64, f32 = {}, {}, {}
    for i in sampled:
        base = int(sum(Lps[:i]))
        L = Ls[i]
        g = {"values": p["values_lr"][:L, i], "old_logp": p["old_logp"][:L, i],
             "advantages": p["adv_c"][base:base + L], "returns": p["ret_c"][base:base + L],
             "h0": p["ybufs"][0][0:L:S, i], "c0": p["cbufs"][0][0:L:S, i]}
        if not packed:                              # the batch columns of the rollout's chunks carry the same states
            col = sum(lp // S for lp in Lps[:i])
            nc = Lps[i] // S
            assert torch.equal(batch.h0[0, col:col + nc], g["h0"]) and torch.equal(batch.c0[0, col:col + nc], g["c0"])
            assert torch.equal(batch.old_values[:, col:col + nc].t().reshape(-1)[:L], g["values"])
            assert torch.equal(batch.advantages[:, col:col + nc].t().reshape(-1)[:L], g["advantages"])
        if i in cut:
            g["values"] = torch.cat([g["values"], p["bootstrap"][cut.index(i)].reshape(1)])
        for dst, res in ((got, {k: v.cpu() for k, v in g.items()}),
                         (f64, ref_rollout(_policy(sd, torch.float64), rollouts[i], torch.float64, estimator == "vtrace")),
                         (f32, ref_rollout(_policy(sd, torch.float32), rollouts[i], torch.float32, estimator == "vtrace"))):
            for k, v in res.items():
                dst.setdefault(k, []).append(v.reshape(-1))
    got, f64, f32 = ({k: torch.cat(v) for k, v in d.items()} for d in (got, f64, f32))
    del batch, p, captured
    opt.close()
    del opt
    gc.collect()
    torch.cuda.empty_cache()
    ratios, over = {}, []
    for k, kind in KINDS.items():
        r, o = bound_check(got, f64, f32, [k], BOUNDS[kind])
        ratios.update(r)
        over += o
    print("\n%s: %s, %.1f s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items()), time.perf_counter() - t0))
    assert not over, over


def _policy(sd, dtype):
    pol = StackedRefPolicy(H, CELL, 1)
    pol.load_state_dict(sd)
    return pol.to(dtype)
