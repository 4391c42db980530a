"""Cost of the state refresh between PPO epochs (``DotaOptimizer(recompute_states=True)``) on the device, at two shapes:
C2 (LSTM-128, 256 rollouts of 512 steps in one chunk each, so no chunk start after the first: the refresh is its forward
alone) and the stream shape (GRU-256, 64 rollouts of 256 steps cut into 1024 sequences of 16).

1. The refresh alone (rollout-major no-grad forward over every rollout's padded length, the fill gathers and
   ``dc_refresh_states``) on the prepared batch, each call timed between two CUDA events; median, min and max of
   ``--calls`` calls.
2. ``train_epochs`` with ``epochs = 4`` and ``num_minibatches`` 1 and 4, by two optimizers from the same seed, one with the
   refresh and one without, their iterations alternated, each timed on the host around ``train_epochs`` (which ends in a
   step's host sync); median, min and max of ``--iters`` iterations each, after two untimed ones (graph capture).
3. Peak device memory of one ``train_epochs`` with and without the refresh, above what was allocated before it.

Prints one JSON line with the card and its power limit.

    python tools/state_refresh_bench.py [--calls 60] [--iters 10] [--shape c2|stream|both]
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
from dotaclient_b200.optimizer import DotaOptimizer  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

# name -> (cell, hidden, seq_len, rollout length, rollouts): C2 is 256 one-chunk rollouts of 512 steps, the stream shape
# 64 rollouts of 256 steps cut into 1024 sequences of 16
SHAPES = {"c2": ("lstm", 128, 512, 512, 256), "stream": ("gru", 256, 16, 256, 64)}
EPOCHS = 4


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _optimizer(cell, H, S, **kw):
    return DotaOptimizer(rmq_host="state_refresh_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=EPOCHS,
                         min_seq_per_epoch=4, seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=H, cell=cell, **kw)


def _stats(xs):
    xs = sorted(xs)
    return {"median": float(np.median(xs)), "min": xs[0], "max": xs[-1], "n": len(xs)}


def _timed_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def bench_shape(name, calls, iters):
    cell, H, S, L, R = SHAPES[name]
    rollouts = [make_rollout(L, 1000 + i) for i in range(R)]
    out = {"shape": {"cell": cell, "hidden": H, "seq_len": S, "sequences": R * L // S, "epochs": EPOCHS}}
    for M in (1, 4):
        on = _optimizer(cell, H, S, num_minibatches=M, recompute_states=True)
        off = _optimizer(cell, H, S, num_minibatches=M)
        b_on, b_off = on.batch_from_rollouts(rollouts), off.batch_from_rollouts(rollouts)
        assert b_on.batch_size == b_off.batch_size == R * L // S
        for _ in range(2):                                  # first sight of each shape, then the graph capture
            on.train_epochs(b_on)
            off.train_epochs(b_off)
        t_on, t_off = [], []
        for _ in range(iters):
            t_on.append(_timed_ms(lambda: on.train_epochs(b_on)))
            t_off.append(_timed_ms(lambda: off.train_epochs(b_off)))
        peak = {}
        for tag, opt, b in (("on", on, b_on), ("off", off, b_off)):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            opt.train_epochs(b)
            torch.cuda.synchronize()
            peak[tag] = (torch.cuda.max_memory_allocated() - base) / 2**20
        out["train_epochs_m%d_ms" % M] = {"on": _stats(t_on), "off": _stats(t_off)}
        out["peak_mb_m%d" % M] = peak
        if M == 1:
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(calls)]
            for _ in range(3):
                on._refresh_states(b_on)
            for a, z in ev:
                a.record()
                on._refresh_states(b_on)
                z.record()
            torch.cuda.synchronize()
            out["refresh_ms"] = _stats([a.elapsed_time(z) for a, z in ev])
            lay = b_on.state_refresh.layout
            out["rollouts"], out["padded_length"], out["states_replaced"] = lay.R, lay.L_max, int(lay.step.size)
            out["time_blocks"] = -(-lay.L_max // max(1, on.REFRESH_CHUNK_TOKENS // lay.R))
            # dc_refresh_states: 12 algorithmic bytes per state float (buffer read, batch read and write)
            out["refresh_states_bytes"] = 12 * int(lay.step.size) * H * (2 if cell == "lstm" else 1)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            on._refresh_states(b_on)
            torch.cuda.synchronize()
            out["refresh_peak_mb"] = (torch.cuda.max_memory_allocated() - base) / 2**20
        del on, off, b_on, b_off
        torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--calls", type=int, default=60)
    p.add_argument("--iters", type=int, default=10)
    p.add_argument("--shape", choices=("c2", "stream", "both"), default="both")
    args = p.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    res = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit()}
    for name in (("c2", "stream") if args.shape == "both" else (args.shape,)):
        res[name] = bench_shape(name, args.calls, args.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
