"""Experience prep under UPGO, value heads, PopArt, KL control and a teacher (``DotaOptimizer._prepare_rollouts`` through
``batch_from_rollouts``, ``mask_padding=True``) at the benchmark's scale, against a float64 reference over whole
rollouts, by the method of ``test_gpu_prep_fp64``, whose rollouts and bound this file imports: hidden 128 LSTM, S 512,
every second rollout cut mid-game, non-zero initial states, 6 sampled rollouts, and per output

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

with (K, FLOOR) = (32, 2e-6) for values, bootstraps, log-probabilities, advantages and returns and (32, 1e-6) for the
chunk-entry states (``test_gpu_prep_fp64.BOUNDS``).  The reference is ``StackedRefPolicy`` in float64 over each sampled
rollout, chunk by chunk with the state carried, plus the extra step after a cut; the same in fp32 calibrates the bound.
  ragged-gae-upgo,     256 rollouts of 300 to 512 steps, ``upgo_coef`` 0.5: GAE or V-trace plus 0.5 ``upgo_oracle.upgo``
  ragged-vtrace-upgo   on the float64 values with the bootstrap after a cut.  UPGO's ``through`` flag has a kink at
                       delta_{t+1} = 0, so before prep the sampled rollouts' rewards (data) are shifted so that no float64
                       |delta| is under 1e-4; the number of steps moved is reported.
  ragged-heads3        the three groups of ``test_gpu_value_heads.THREE`` with their own discounts: a 3-row float64 value
                       head, then ``value_heads_oracle.scan_heads``; values, bootstraps, advantages and [.., 3] returns.
  ragged-popart        statistics preset to mu = -1.3, sigma = 3.7: values and bootstraps are mu + sigma v of the float64
                       forward, advantages and returns GAE in raw units.  (The statistics update and the POP rescale are
                       ``test_gpu_value_norm``'s.)
  long-kl-teacher      32 rollouts of 3,585 to 4,096 steps, ``kl_coef`` 0.2, a GRU-256 teacher (grid encoder) for the
                       LSTM-128 student: every head's ``old_log_probs`` row (the chunk-crossing state) and the
                       ``teacher_log_probs`` rows on their legal entries, the masked log-softmax of each forward, the
                       teacher from the zero state over every whole rollout, cut ones included; illegal entries exactly 0.
Measured on one H100 80GB HBM3 (700 W power limit), the largest ratio max|gpu - f64| / max|torch32 - f64| per output,
values / old_logp / advantages / returns / h0 / c0 (/ old_log_probs / teacher_log_probs), the largest share of its bound
any output uses, the steps moved off delta = 0, and the wall time of the regime:
    ragged-gae-upgo      12 /  8.2 /  11 /  43 /  -  /  -               0.31   4 moved   5 s
    ragged-vtrace-upgo   13 /  7.8 /  10 /  14 /  -  /  -               0.35   5 moved   4 s
    ragged-heads3       8.1 /  8.2 / 6.5 /  27 /  -  /  -               0.31             5 s
    ragged-popart       8.3 /  8.2 / 8.5 /  35 /  -  /  -               0.40             5 s
    long-kl-teacher      15 /   11 /  13 /  58 /  15 /  19 / 9.4 / 17   0.42            19 s
(A ragged rollout is one chunk: its entry state is its initial_hidden, exact.)  long-kl-teacher checks 2,324,632 illegal
row entries to be exactly 0.  The whole file runs in about 55 s on the H100.
"""
import copy
import gc
import time
import uuid

import numpy as np
import pytest
import torch

import test_gpu_prep_fp64 as PR
import upgo_oracle as UP
import value_heads_oracle as VH
import vtrace_oracle as VT
from dotaclient_b200.policy import REWARD_KEYS
from stacked_oracle import StackedRefPolicy
from test_gpu_objectives_fp64 import NORM_STATE, HeadsRefPolicy
from test_gpu_ppo_fp64 import HEADS, log_softmax
from test_gpu_rnn_fp64 import bound_check
from test_gpu_step_fp64 import grid_encoder
from test_gpu_value_heads import GAMMAS3, THREE
from value_norm_oracle import moments

S, H, CELL = PR.S, PR.H, PR.CELL
GAMMA, LAMBDA = PR.GAMMA, PR.LAMBDA
BOUNDS = PR.BOUNDS
KINDS = dict(PR.KINDS, old_log_probs="forward", teacher_log_probs="forward")
UPGO_COEF, KL_COEF = 0.5, 0.2
DELTA_MARGIN = 1e-4           # least float64 |delta| of a sampled rollout under UPGO after the reward shift

# (id, number of rollouts, length range, estimator, options)
REGIMES = [
    ("ragged-gae-upgo", 256, (300, 512), "gae", dict(upgo_coef=UPGO_COEF)),
    ("ragged-vtrace-upgo", 256, (300, 512), "vtrace", dict(upgo_coef=UPGO_COEF)),
    ("ragged-heads3", 256, (300, 512), "gae", dict(value_heads=THREE, value_gammas=GAMMAS3)),
    ("ragged-popart", 256, (300, 512), "gae", dict(value_norm=True)),
    ("long-kl-teacher", 32, (3585, 4096), "gae", dict(kl_coef=KL_COEF)),
]


def rollout_forward(pol, data, dtype, zero_state=False):
    """``pol`` over one rollout in chunks of S with the state carried, from its ``initial_hidden`` (or the zero state)
    -> {logits {head: [L, n]}, values [L, K], boot [K] (after a cut, None otherwise; not with ``zero_state``), h0 / c0
    entering every chunk [n_chunks, H]}."""
    L = int(data["rewards"].shape[0])
    cut = not data.get("terminal", True)
    lstm = pol.cell == "lstm"
    obs = {k: torch.as_tensor(v).to(dtype).unsqueeze(0) for k, v in data["observations"].items()}
    if zero_state:
        h = torch.zeros(1, 1, pol.hidden_size, dtype=dtype)
        c = torch.zeros_like(h)
    else:
        h, c = (t.to(dtype) for t in data["initial_hidden"])
    hs, cs, lgs, vals = [], [], [], []
    with torch.no_grad():
        for t0 in range(0, L, S):
            hs.append(h[0, 0])
            cs.append(c[0, 0])
            lg, v, hid = pol(**{k: o[:, t0:min(t0 + S, L)] for k, o in obs.items()}, hidden=(h, c) if lstm else h)
            h, c = hid if lstm else (hid, c)
            lgs.append({k: x[0] for k, x in lg.items()})
            vals.append(v[0].reshape(v.shape[1], -1))            # [T, K] (HeadsRefPolicy returns [1, T, K, 1])
        boot = None
        if cut and not zero_state:
            boot = pol(**{k: o[:, L:L + 1] for k, o in obs.items()}, hidden=(h, c) if lstm else h)[1].reshape(-1)
    return {"logits": {k: torch.cat([x[k] for x in lgs]) for k in HEADS}, "values": torch.cat(vals), "boot": boot,
            "h0": torch.stack(hs), "c0": torch.stack(cs)}


def selected(logits, data, dtype):
    """[L, 5] selected log-probabilities (0 where a head took no action)."""
    sel = []
    for k in HEADS:
        m = torch.as_tensor(data["masks"][k]).bool()
        a = torch.as_tensor(data["actions"][k]).bool()
        sel.append(torch.where(a, log_softmax(logits[k], m), torch.zeros((), dtype=dtype)).sum(1))
    return torch.stack(sel, 1)


def deltas(data, values, boot):
    """float64 TD errors r_t + gamma V_{t+1} - V_t of one rollout (``values`` [L], ``boot`` after the last step)."""
    r = VT.reward_sum(data["rewards"]).astype(np.float64)
    v = np.asarray(values, np.float64)
    return r + GAMMA * np.append(v[1:], boot) - v


def shift_rewards(data, values, boot):
    """Moves every step whose float64 |delta| is under DELTA_MARGIN to 2 DELTA_MARGIN off 0 by shifting its first reward
    column (the rollout's data); returns the number of steps moved."""
    d = deltas(data, values, boot)
    near = np.abs(d) < DELTA_MARGIN
    rew = np.array(data["rewards"], dtype=np.float32, copy=True)
    rew[near, 0] += (np.where(d[near] >= 0, 2 * DELTA_MARGIN, -2 * DELTA_MARGIN) - d[near]).astype(np.float32)
    data["rewards"] = rew
    assert np.abs(deltas(data, values, boot)).min() >= DELTA_MARGIN
    return int(near.sum())


def reference(pol, teacher, data, dtype, estimator, opts, norm):
    """One sampled rollout in ``dtype`` -> the outputs prep writes for it (values with a cut's bootstrap appended)."""
    f = rollout_forward(pol, data, dtype)
    L = int(data["rewards"].shape[0])
    v, boot = f["values"], f["boot"]
    if norm is not None:
        v, boot = norm[0] + norm[1] * v, None if boot is None else norm[0] + norm[1] * boot
    old = selected(f["logits"], data, dtype)
    b = np.zeros(v.shape[1]) if boot is None else boot.double().numpy()
    out = {"values": v if boot is None else torch.cat([v, boot[None]]), "old_logp": old, "h0": f["h0"], "c0": f["c0"]}
    if opts.get("value_heads"):
        names = list(THREE)
        group = np.array([[k in THREE[n] for n in names].index(True) for k in REWARD_KEYS], np.int32)
        gammas = np.array([GAMMAS3.get(n, GAMMA) for n in names])
        _, _, adv, ret = VH.scan_heads(data["rewards"], v.double().numpy(), [0, L], group, gammas, LAMBDA,
                                       boot_value=b[None], boot_reward=b[None])
    else:
        v1 = v[:, 0].double().numpy()
        logrho = None
        if estimator == "vtrace":
            acted = np.stack([np.asarray(data["actions"][k]).any(1) for k in HEADS], 1)
            beh = np.where(acted, np.asarray(data["behaviour_logp"], dtype=np.float32), 0.0)
            logrho = VT.log_rho(old.double().numpy(), beh)
            adv, ret = VT.vtrace(data["rewards"], v1, logrho, GAMMA, LAMBDA, boot=float(b[0]))
        else:
            adv, ret = PR.gae(data["rewards"], v1, float(b[0]))
        if opts.get("upgo_coef"):
            adv = adv + opts["upgo_coef"] * UP.upgo(data["rewards"], v1, GAMMA, boot=float(b[0]), logrho=logrho)[0]
    out["advantages"] = torch.from_numpy(np.ascontiguousarray(adv))
    out["returns"] = torch.from_numpy(np.ascontiguousarray(ret))
    if opts.get("kl_coef"):
        masks = {k: torch.as_tensor(data["masks"][k]).bool() for k in HEADS}
        legal = torch.cat([masks[k] for k in HEADS], 1)
        t_logits = rollout_forward(teacher, data, dtype, zero_state=True)["logits"]
        for k, lg in (("old_log_probs", f["logits"]), ("teacher_log_probs", t_logits)):
            out[k] = torch.cat([log_softmax(lg[h], masks[h]) for h in HEADS], 1)[legal]      # in dtype, legal entries
    return out


def ref_policy(sd, dtype, K):
    pol = HeadsRefPolicy(H, CELL, 1, K) if K > 1 else StackedRefPolicy(H, CELL, 1)
    pol.load_state_dict(sd)
    return pol.to(dtype)


def save_teacher(tmp_path):
    """A GRU-256 teacher: the reference's seeded initialisation with the encoder on the grids of ``grid_encoder``."""
    from dotaclient_b200.policy import Policy
    torch.manual_seed(7)
    pol = Policy()
    grid_encoder(pol, 29)
    sd = {k: v.detach().cpu() for k, v in pol.state_dict().items()}
    path = str(tmp_path / "teacher_gru256.pt")
    torch.save(sd, path)
    return path, sd


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_prep_objectives_vs_fp64(regime, tmp_path):
    from dotaclient_b200.optimizer import DotaOptimizer
    name, n, lengths, estimator, opts = regime
    t0 = time.perf_counter()
    gc.collect()
    torch.cuda.empty_cache()
    kw, t_sd = dict(opts), None
    if opts.get("kl_coef"):
        kw["teacher_model"], t_sd = save_teacher(tmp_path)
    opt = DotaOptimizer(rmq_host="prep-objectives", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=1,
                        seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                        log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H, cell=CELL,
                        mask_padding=True, advantage_estimator=estimator, **kw)
    norm = None
    if opts.get("value_norm"):
        opt._value_norm = NORM_STATE
        norm = moments(NORM_STATE)
        assert opt._value_norm_moments() == norm
    K = opt.n_value_heads
    grid_encoder(opt.policy_base, 17)
    sd = {k: v.detach().cpu().clone() for k, v in opt.policy_base.state_dict().items()}    # before prep (PopArt rescales)
    rollouts = PR.make_rollouts(n, lengths, n + lengths[0] + 7, estimator == "vtrace")
    sampled = (0, 1, 2, n // 2 - 1, n // 2, n - 1)
    moved = 0
    if opts.get("upgo_coef"):
        p64 = ref_policy(sd, torch.float64, K)
        for i in sampled:
            f = rollout_forward(p64, rollouts[i], torch.float64)
            moved += shift_rewards(rollouts[i], f["values"][:, 0].numpy(),
                                   0.0 if f["boot"] is None else float(f["boot"][0]))
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
    cut = [i for i, d in enumerate(rollouts) if not d.get("terminal", True)]
    over, zero_off = [], 0
    got = {}
    for i in sampled:
        base, L = int(sum(Lps[:i])), Ls[i]
        g = {"values": p["values_lr"][:L, i].reshape(L, K), "old_logp": p["old_logp"][:L, i],
             "advantages": p["adv_c"][base:base + L], "returns": p["ret_c"][base:base + L],
             "h0": p["ybufs"][0][0:L:S, i], "c0": p["cbufs"][0][0:L:S, i]}
        if i in cut:
            g["values"] = torch.cat([g["values"], p["bootstrap"][cut.index(i)].reshape(1, K)])
        if opts.get("kl_coef"):
            legal = torch.cat([torch.as_tensor(rollouts[i]["masks"][k]).bool() for k in HEADS], 1).to(g["h0"].device)
            for k in ("old_log_probs", "teacher_log_probs"):
                rows = p[k][:L, i]
                if bool((rows[~legal] != 0).any()):
                    over.append("%s: non-zero at an illegal entry of rollout %d" % (k, i))
                zero_off += int((~legal).sum())
                g[k] = rows[legal]
        for k, v in g.items():
            got.setdefault(k, []).append(v.cpu().reshape(-1))
    del batch, p, captured
    opt.close()
    del opt
    gc.collect()
    torch.cuda.empty_cache()
    f64, f32 = {}, {}
    for dtype, dst in ((torch.float64, f64), (torch.float32, f32)):
        pol = ref_policy(sd, dtype, K)
        teacher = None
        if t_sd is not None:
            teacher = StackedRefPolicy(256, "gru", 1)
            teacher.load_state_dict(t_sd)
            teacher = teacher.to(dtype)
        for i in sampled:
            for k, v in reference(pol, teacher, rollouts[i], dtype, estimator, opts, norm).items():
                dst.setdefault(k, []).append(v.reshape(-1))
    got, f64, f32 = ({k: torch.cat(v) for k, v in d.items()} for d in (got, f64, f32))
    ratios, used = {}, 0.0
    for k in got:
        kind = KINDS[k]
        r, o = bound_check(got, f64, f32, [k], BOUNDS[kind])
        ratios.update(r)
        over += o
        err = float((got[k].double() - f64[k]).abs().max())
        kb, floor = BOUNDS[kind]
        used = max(used, err / (kb * float((f32[k].double() - f64[k]).abs().max()) + floor * float(f64[k].abs().max())))
    print("\n%s: %s, of bound %.3g, steps moved off delta = 0: %d, illegal entries checked zero: %d, %.1f s"
          % (name, ", ".join("%s %.3g" % kv for kv in ratios.items() if not kv[0].startswith("rel ")), used, moved,
             zero_off, time.perf_counter() - t0))
    assert not over, over
