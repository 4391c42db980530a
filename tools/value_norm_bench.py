"""Cost of ``value_norm=True`` (PopArt) on the device.

1. The fused loss kernel alone at C2's token count (256 sequences x 512 steps = 131,072 tokens): one
   ``dc_ppo_loss_fwd_bwd_dev`` call with hyper-parameter slot 7 = 0 (off) against one with (mu, sigma) set, on the same
   preallocated inputs with the clipped value loss, each call timed alone between two CUDA events, the two alternated call
   by call; median, min and max of ``--calls`` calls each.
2. The whole C2 training step (LSTM-128, S = 512, B = 256, replayed from its CUDA graph) on one batch, trained by two
   optimizers from the same seed, one with ``value_norm=True`` and one without; their steps alternate, each timed on the
   host around ``train()`` (which ends in the step's host sync).
3. ``batch_from_rollouts`` on 88 ragged rollouts of 1000-1400 steps (seq_len 16), with and without the feature,
   alternated: the value denormalisation, the statistics kernel, its host sync and the head rescale land here.

Prints one JSON line with the card and its power limit.

    python tools/value_norm_bench.py [--calls 200] [--steps 30] [--preps 10]
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
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

S, B, H = 512, 256, 128


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _optimizer(value_norm, seq_len=S, hidden_size=H, cell="lstm"):
    return DotaOptimizer(rmq_host="value_norm_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1,
                         min_seq_per_epoch=4, seq_len=seq_len, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=hidden_size, cell=cell, value_clip=0.2, value_norm=value_norm)


def _stats(xs):
    xs = sorted(xs)
    return {"median": float(np.median(xs)), "min": xs[0], "max": xs[-1], "n": len(xs)}


def _kernel_rows(calls):
    """The `_dev` entry point with slot 7 = 0 and with (mu, sigma) set, on the same random C2-sized inputs, alternated;
    microseconds per call."""
    d = torch.device("cuda")
    N = S * B
    g = torch.Generator(device=d).manual_seed(0)
    logits = [torch.randn(N, n, generator=g, device=d) for n in ops.HEAD_SIZES]
    masks = [torch.rand(N, n, generator=g, device=d) < 0.7 for n in ops.HEAD_SIZES]
    actions = []
    for n, m in zip(ops.HEAD_SIZES, masks):
        a = torch.zeros(N, n, dtype=torch.bool, device=d)
        a[torch.arange(N, device=d), torch.randint(0, n, (N,), generator=g, device=d)] = True
        actions.append(a & m)
    old = torch.randn(N, 5, generator=g, device=d) - 2.0
    adv, value = (torch.randn(N, generator=g, device=d) for _ in range(2))
    ret, old_value = (20.0 * torch.randn(N, generator=g, device=d) + 5.0 for _ in range(2))
    dlogits = [torch.empty_like(t) for t in logits]
    dvalue = torch.empty_like(value)
    out = torch.empty(_lib.LOSS_SLOTS, device=d)
    stats = torch.empty(_lib.PPO_STATS_SLOTS, device=d)
    n_act = torch.empty(5, dtype=torch.int32, device=d)
    ws = torch.empty(_lib.PPO_WORKSPACE_BYTES, dtype=torch.uint8, device=d)
    hps = {"off": ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5, value_clip=0.2),
           "value_norm": ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5, value_clip=0.2,
                                          value_norm=(5.0, 20.0))}
    u8 = [ops._u8(t) for t in masks], [ops._u8(t) for t in actions]
    lib, stream = _lib.load(), _lib.stream_ptr()
    ld = (_lib._c.c_int64 * 5)(*ops.HEAD_SIZES)
    head = (_lib.ptr5(logits), ld, _lib.ptr5(u8[0]), _lib.ptr5(u8[1]), old.data_ptr(), adv.data_ptr(), ret.data_ptr(),
            value.data_ptr(), 1, old_value.data_ptr(), N)

    def call(hp):
        return lib.dc_ppo_loss_fwd_bwd_dev(*head, hp.data_ptr(), _lib.ptr5(dlogits), ld, dvalue.data_ptr(), 1,
                                           out.data_ptr(), stats.data_ptr(), n_act.data_ptr(), ws.data_ptr(), stream)
    fns = {k: (lambda hp=hp: call(hp)) for k, hp in hps.items()}
    for _ in range(10):
        for f in fns.values():
            assert f() == 0
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
    res["value_norm_over_off_median"] = res["value_norm"]["median"] / res["off"]["median"]
    return res


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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed loss-kernel calls per setting (median; >= 200)")
    ap.add_argument("--steps", type=int, default=30, help="timed C2 steps per optimizer")
    ap.add_argument("--preps", type=int, default=10, help="timed batch_from_rollouts calls per optimizer")
    args = ap.parse_args()
    if args.calls < 200:
        ap.error("--calls must be >= 200")
    if not torch.cuda.is_available():
        raise SystemExit("value_norm_bench needs a CUDA device")
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls,
              "config": "C2: LSTM-128, seq_len 512, 256 sequences, value_clip 0.2"}
    result["loss_kernel_us"] = _kernel_rows(args.calls)

    pool = [make_rollout(2 * S, 50_000 + i) for i in range(8)]
    rollouts = [pool[i % len(pool)] for i in range(B // 2)]          # two whole sequences each: B sequences
    on, off = _optimizer(True), _optimizer(False)
    batch_on, batch_off = on.batch_from_rollouts(rollouts), off.batch_from_rollouts(rollouts)
    assert (batch_on.seq_len, batch_on.batch_size) == (S, B)
    for _ in range(3):                               # eager, capture, replay
        on.train(batch_on)
        off.train(batch_off)
    times = _alternate([("off", lambda: off.train(batch_off)), ("value_norm", lambda: on.train(batch_on))], args.steps)
    result["c2_step_ms"] = {k: _stats(v) for k, v in times.items()}
    result["c2_step_ms"]["value_norm_over_off_median"] = \
        result["c2_step_ms"]["value_norm"]["median"] / result["c2_step_ms"]["off"]["median"]
    on.close()
    off.close()

    rng = np.random.RandomState(3)
    ragged = [make_rollout(int(rng.randint(1000, 1401)), 60_000 + i) for i in range(88)]
    p_on, p_off = _optimizer(True, seq_len=16, hidden_size=256, cell="gru"), _optimizer(False, seq_len=16, hidden_size=256,
                                                                                        cell="gru")
    for _ in range(2):
        p_on.batch_from_rollouts(ragged)
        p_off.batch_from_rollouts(ragged)
    times = _alternate([("off", lambda: p_off.batch_from_rollouts(ragged)),
                        ("value_norm", lambda: p_on.batch_from_rollouts(ragged))], args.preps)
    result["prep_88_rollouts_ms"] = {k: _stats(v) for k, v in times.items()}
    result["prep_88_rollouts_ms"]["tokens"] = int(sum((r["rewards"].shape[0] + 15) // 16 * 16 for r in ragged))
    result["prep_88_rollouts_ms"]["config"] = "GRU-256, seq_len 16"
    p_on.close()
    p_off.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
