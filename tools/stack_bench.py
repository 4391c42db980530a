"""Cost of a stacked recurrent core (``num_layers``): ms per DotaOptimizer.train() step at C2's batch x seq (256 x 512).

    python tools/stack_bench.py [--steps 10] [--warmup 3]

Configurations: LSTM-128 at L = 1, 2, 3; GRU-256 at L = 1, 2; LSTM-192 at L = 1 (one layer with about the recurrent
parameter count of two 128-wide layers, on the generic recurrence kernel).  One JSON line each:
  ms_per_step          CUDA events around `steps` train() calls on a device-resident batch, replayed from the step's CUDA graph
  ms_launch_by_launch  the same steps launched kernel by kernel with ops.PROFILE events around every kernel call
  rnn_ms, rnn_share    recurrence kernels (rnn_fwd + rnn_bwd, all layers) per launch-by-launch step, and their share of it
  prep_ms              batch_from_rollouts for 12 rollouts of 1380 steps at seq_len 16 (the reference's defaults), wall time
                       ending in a device synchronise, median of 3 after one warm-up
The first line names the card, its power limit and its maximum SM clock; the last one gives ms per extra layer.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from dotaclient_b200 import ops  # noqa: E402
from dotaclient_b200.optimizer import DotaOptimizer  # noqa: E402
from dotaclient_b200.synthetic import make_rollout, rollout_seed  # noqa: E402

CONFIGS = [(128, "lstm", 1), (128, "lstm", 2), (128, "lstm", 3), (256, "gru", 1), (256, "gru", 2), (192, "lstm", 1)]
BATCH, SEQ = 256, 512                    # C2
PREP_ROLLOUTS, PREP_LEN, PREP_SEQ = 12, 1380, 16


def card():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:                 # the timings stand without it, but say it is missing
        info["power_limit"] = info["max_sm_clock"] = "unknown (%s)" % e
    return info


def optimizer(H, cell, L, seq_len, batch):
    return DotaOptimizer(rmq_host="stack_bench", rmq_port=0, epochs=1, min_seq_per_epoch=batch, seq_len=seq_len,
                         learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                         log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H,
                         cell=cell, num_layers=L)


def timed_ms(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def measure(H, cell, L, rollouts, prep_rollouts, steps, warmup):
    opt = optimizer(H, cell, L, SEQ, BATCH)
    with torch.no_grad():
        batch = opt.batch_from_rollouts(rollouts)
    for _ in range(max(3, warmup)):                # the second call of the shape captures the graph
        opt.train(batch)
    ms = timed_ms(lambda: opt.train(batch), steps)
    graphed = any(isinstance(v, tuple) for v in opt._graphs.values())
    ops.PROFILE.reset(enabled=True)
    opt.train(batch)                               # untimed: the launch-by-launch path re-grows its allocator pool
    ops.PROFILE.reset(enabled=True)
    ms_eager = timed_ms(lambda: opt.train(batch), steps)
    kern = ops.PROFILE.summary(steps)
    ops.PROFILE.reset(enabled=False)
    rnn_ms = kern.get("rnn_fwd", 0.0) + kern.get("rnn_bwd", 0.0)
    opt.close()
    del batch, opt
    torch.cuda.empty_cache()

    prep = optimizer(H, cell, L, PREP_SEQ, 1)
    walls = []
    for _ in range(4):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            b = prep.batch_from_rollouts(prep_rollouts)
        torch.cuda.synchronize()
        walls.append(1e3 * (time.perf_counter() - t0))
        del b
    prep.close()
    del prep
    torch.cuda.empty_cache()
    return {"hidden": H, "cell": cell, "num_layers": L, "batch": BATCH, "seq_len": SEQ, "cuda_graph": graphed,
            "ms_per_step": round(ms, 3), "ms_launch_by_launch": round(ms_eager, 3), "rnn_ms": round(rnn_ms, 3),
            "rnn_share": round(rnn_ms / ms_eager, 3), "prep_ms": round(statistics.median(walls[1:]), 2)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("stack_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    print(json.dumps(card()), flush=True)
    rollouts = [make_rollout(SEQ, rollout_seed(0, i)) for i in range(BATCH)]
    prep_rollouts = [make_rollout(PREP_LEN, 5000 + i) for i in range(PREP_ROLLOUTS)]
    results = {}
    for H, cell, L in CONFIGS:
        r = measure(H, cell, L, rollouts, prep_rollouts, a.steps, a.warmup)
        results[(H, cell, L)] = r
        print(json.dumps(r), flush=True)
    extra = {"%s-%d L%d-L%d" % (cell.upper(), H, L, L - 1): round(r["ms_per_step"] - results[(H, cell, L - 1)]["ms_per_step"], 3)
             for (H, cell, L), r in results.items() if (H, cell, L - 1) in results}
    print(json.dumps({"ms_per_extra_layer": extra}), flush=True)


if __name__ == "__main__":
    main()
