"""Cost of ``value_heads`` on the device.

1. The loss at C2's token count (256 sequences x 512 steps = 131,072 tokens, clipped value loss): the default single
   ``dc_ppo_loss_fwd_bwd_dev`` call against the same call with its value term off followed by ``dc_value_heads_loss``, for
   K = 1, 2 and 10 heads, on the same preallocated inputs; every setting is timed between two CUDA events, the settings
   alternated call by call; median, min and max of ``--calls`` calls each.
2. The whole C2 training step (LSTM-128, S = 512, B = 256, replayed from its CUDA graph) on one batch: the default optimizer
   against K = 2 and K = 10 heads, steps alternated, each timed on the host around ``train()`` (which ends in the step's
   host sync).
3. ``batch_from_rollouts`` on 88 ragged rollouts of 1000-1400 steps (seq_len 16, GRU-256): default against K = 10,
   alternated.

Prints one JSON line with the card and its power limit.

    python tools/value_heads_bench.py [--calls 200] [--steps 30] [--preps 10]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dotaclient_b200 import _lib, ops  # noqa: E402
from dotaclient_b200.optimizer import DotaOptimizer  # noqa: E402
from dotaclient_b200.policy import REWARD_KEYS  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

S, B, H = 512, 256, 128


def heads(K):
    """K groups of the reward keys (None for the default critic): 'win' alone, then the rest spread over K - 1 heads."""
    if K is None:
        return None
    if K == 1:
        return {'all': list(REWARD_KEYS)}
    rest = [k for k in REWARD_KEYS if k != 'win']
    return {'win': ['win'], **{'g%d' % j: rest[j::K - 1] for j in range(K - 1)}}


def _optimizer(K, seq_len=S, hidden_size=H, cell="lstm"):
    vh = heads(K)
    return DotaOptimizer(rmq_host="value_heads_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1,
                         min_seq_per_epoch=4, seq_len=seq_len, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=hidden_size, cell=cell, value_clip=0.2, value_heads=vh,
                         value_gammas=None if vh is None or K == 1 else {'win': 0.999})


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _stats(xs):
    xs = sorted(xs)
    return {"median": float(np.median(xs)), "min": xs[0], "max": xs[-1], "n": len(xs)}


def _alternate(jobs, n):
    """Runs every ``(key, fn)`` of ``jobs`` n times, alternated, each timed on the host after a device sync; ms."""
    times = {k: [] for k, _ in jobs}
    for _ in range(n):
        for key, fn in jobs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[key].append(1e3 * (time.perf_counter() - t0))
    return times


def _loss_rows(calls):
    """The default packed loss call against the loss with its value term off plus the value-heads kernel, K = 1, 2, 10,
    on the same random C2-sized inputs, alternated; microseconds per call (both kernels for the value-heads rows)."""
    d = torch.device("cuda")
    N = S * B
    g = torch.Generator(device=d).manual_seed(0)
    packed = torch.randn(N, ops.PACK_WIDTH, generator=g, device=d)
    tu = torch.randn(N, 40, generator=g, device=d)
    masks, actions = [], []
    for n in ops.HEAD_SIZES:
        m = torch.rand(N, n, generator=g, device=d) < 0.7
        a = torch.zeros(N, n, dtype=torch.bool, device=d)
        a[torch.arange(N, device=d), torch.randint(0, n, (N,), generator=g, device=d)] = True
        masks.append(m)
        actions.append(a & m)
    old = torch.randn(N, 5, generator=g, device=d) - 2.0
    adv = torch.randn(N, generator=g, device=d)
    rets = {K: torch.randn(N, K, generator=g, device=d) for K in (1, 2, 10)}
    olds = {K: torch.randn(N, K, generator=g, device=d) for K in (1, 2, 10)}
    hp = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5, value_clip=0.2)
    hp_off = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4)
    stats = torch.empty(_lib.PPO_STATS_SLOTS, device=d)
    hs = torch.empty(_lib.VALUE_HEADS_STATS_SLOTS, device=d)

    def default():
        ops.ppo_loss_packed(packed, tu, masks, actions, old, adv, rets[1], 0, 0, 0, hparams=hp, old_value=olds[1],
                            stats=stats)

    def with_heads(K):
        out, _, dp, _, _ = ops.ppo_loss_packed(packed, tu, masks, actions, old, adv, adv, 0, 0, 0, hparams=hp_off,
                                               stats=stats)
        ops.value_heads_loss(packed, dp, rets[K], hp, out, hs, old_value=olds[K], stats=stats)
    fns = {"default": default, **{"heads_%d" % K: (lambda K=K: with_heads(K)) for K in (1, 2, 10)}}
    for _ in range(10):
        for f in fns.values():
            f()
    torch.cuda.synchronize()
    pairs = {k: [] for k in fns}
    for _ in range(calls):
        for k, f in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            pairs[k].append((e0, e1))
    torch.cuda.synchronize()
    res = {k: _stats([1000.0 * a.elapsed_time(b) for a, b in v]) for k, v in pairs.items()}
    res["tokens"] = N
    res["note"] = "each call includes its output allocations (d_packed zero-fill), as ppo_loss_packed makes them"
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed loss calls per setting (median; >= 200)")
    ap.add_argument("--steps", type=int, default=30, help="timed C2 steps per optimizer")
    ap.add_argument("--preps", type=int, default=10, help="timed batch_from_rollouts calls per optimizer")
    args = ap.parse_args()
    if args.calls < 200:
        ap.error("--calls must be >= 200")
    if not torch.cuda.is_available():
        raise SystemExit("value_heads_bench needs a CUDA device")
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls,
              "config": "C2: LSTM-128, seq_len 512, 256 sequences, value_clip 0.2"}
    result["loss_us"] = _loss_rows(args.calls)

    pool = [make_rollout(2 * S, 50_000 + i) for i in range(8)]
    rollouts = [pool[i % len(pool)] for i in range(B // 2)]          # two whole sequences each: B sequences
    opts = {"default": _optimizer(None), "heads_2": _optimizer(2), "heads_10": _optimizer(10)}
    batches = {k: o.batch_from_rollouts(rollouts) for k, o in opts.items()}
    for k, b in batches.items():
        assert (b.seq_len, b.batch_size) == (S, B)
    for _ in range(3):                               # eager, capture, replay
        for k, o in opts.items():
            o.train(batches[k])
    times = _alternate([(k, (lambda o=o, b=batches[k]: o.train(b))) for k, o in opts.items()], args.steps)
    result["c2_step_ms"] = {k: _stats(v) for k, v in times.items()}
    for o in opts.values():
        o.close()

    rng = np.random.RandomState(3)
    ragged = [make_rollout(int(rng.randint(1000, 1401)), 60_000 + i) for i in range(88)]
    preps = {"default": _optimizer(None, 16, 256, "gru"), "heads_10": _optimizer(10, 16, 256, "gru")}
    for _ in range(2):
        for p in preps.values():
            p.batch_from_rollouts(ragged)
    times = _alternate([(k, (lambda p=p: p.batch_from_rollouts(ragged))) for k, p in preps.items()], args.preps)
    result["prep_88_rollouts_ms"] = {k: _stats(v) for k, v in times.items()}
    result["prep_88_rollouts_ms"]["tokens"] = int(sum((r["rewards"].shape[0] + 15) // 16 * 16 for r in ragged))
    result["prep_88_rollouts_ms"]["config"] = "GRU-256, seq_len 16"
    for p in preps.values():
        p.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
