"""Cost of UPGO (``DotaOptimizer(upgo_coef=c)``) on one GPU:

1. Per-call time of ``dc_upgo_scan`` (GAE form and V-trace form) and ``dc_upgo_scan_indexed`` at C2's batch (256
   rollouts x 512 rows) and at ragged 1000-1400-step games padded to seq_len 512, each call timed alone between two CUDA
   events; median, min and max of ``--calls`` calls, against the algorithmic HBM bytes of the file header at 3.35 TB/s.
2. Experience prep of the C2 rollouts (``batch_from_rollouts``) with ``upgo_coef`` 0 and 0.5, alternated on one
   optimizer, each timed on the host up to a device synchronise; ``--preps`` runs each.

Prints one JSON line with the card and its power limit.

    python tools/upgo_bench.py [--calls 200] [--preps 3]
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
from dotaclient_b200 import ops  # noqa: E402
from dotaclient_b200.optimizer import DotaOptimizer  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

S, B, H = 512, 256, 128
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
BYTES_PER_ROW = {"gae": 40 + 4 + 4 + 4, "vtrace": 40 + 4 + 4 + 4 + 40, "indexed": 40 + 4 + 4 + 4 + 8}


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


def _median_us(fn, calls, warmup=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    pairs = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        pairs.append((e0, e1))
    torch.cuda.synchronize()
    return _stats([1000.0 * a.elapsed_time(b) for a, b in pairs])


def _kernels(lengths, calls):
    """The three entry points over rollout-major rows as prep lays them out ([real | padding] segments)."""
    g = torch.Generator().manual_seed(1)
    padded = [(L + S - 1) // S * S for L in lengths]
    off = [0]
    for L, Lp in zip(lengths, padded):
        off += [off[-1] + L, off[-1] + Lp]
    n = off[-1]
    d = torch.device("cuda")
    rewards = (0.01 * torch.randn(n, 10, generator=g)).to(d)
    values = torch.randn(n, generator=g).to(d)
    lt = (-torch.rand(n, 5, generator=g)).to(d)
    lb = (lt.cpu() + 0.1 * torch.randn(n, 5, generator=g)).to(d)
    seg = torch.tensor(off, dtype=torch.int64, device=d)
    valid = torch.tensor([v for L in lengths for v in (L, 0)], dtype=torch.int64, device=d)
    boot = torch.zeros(len(off) - 1, device=d)
    tok = torch.randperm(n, generator=g).to(d)
    adv = torch.zeros(n, device=d)
    res = {"segments": len(off) - 1, "rows": n}
    fns = {
        "gae": lambda: ops.upgo_scan(rewards, values, seg, adv, 0.98, 0.5, boot_value=boot, valid_len=valid, stats=True),
        "vtrace": lambda: ops.upgo_scan(rewards, values, seg, adv, 0.98, 0.5, boot_value=boot, logp_target=lt,
                                        logp_behaviour=lb, valid_len=valid, stats=True),
        "indexed": lambda: ops.upgo_scan_indexed(rewards, values, tok, seg, adv, 0.98, 0.5, boot_value=boot),
    }
    for k, f in fns.items():
        t = _median_us(f, calls)
        floor_us = 1e6 * n * BYTES_PER_ROW[k] / HBM_BYTES_PER_S
        res[k + "_us"] = t
        res[k + "_bytes"] = n * BYTES_PER_ROW[k]
        res[k + "_byte_floor_us"] = floor_us
        res[k + "_share_of_byte_floor"] = floor_us / t["median"]
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed calls per entry point and shape (median; >= 50)")
    ap.add_argument("--preps", type=int, default=3, help="timed experience preps per coefficient")
    args = ap.parse_args()
    if args.calls < 50:
        ap.error("--calls must be >= 50")
    if not torch.cuda.is_available():
        raise SystemExit("upgo_bench needs a CUDA device")
    rng = np.random.RandomState(0)
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls, "kernels": {}}
    shapes = {"c2_256x512": [512] * 256, "games_64x1000_1400": [int(v) for v in rng.randint(1000, 1401, size=64)]}
    for name, lengths in shapes.items():
        result["kernels"][name] = _kernels(lengths, args.calls)

    pool = [make_rollout(2 * S, 40_000 + i) for i in range(8)]
    rollouts = [pool[i % len(pool)] for i in range(B // 2)]          # two whole sequences each: B sequences
    opt = DotaOptimizer(rmq_host="upgo_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1, min_seq_per_epoch=4,
                        seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                        log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H,
                        cell="lstm")
    times = {"0.0": [], "0.5": []}
    for rep in range(args.preps + 1):               # the first round warms every shape up
        for c in (0.0, 0.5):
            opt.upgo_coef = c
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            batch = opt.batch_from_rollouts(rollouts)
            torch.cuda.synchronize()
            if rep:
                times[str(c)].append(1e3 * (time.perf_counter() - t0))
    assert (batch.seq_len, batch.batch_size) == (S, B) and opt.last_upgo_stats is not None
    result["c2_prep_ms"] = {"upgo_coef_" + k: _stats(v) for k, v in times.items()}
    result["c2_prep_ms"]["added_median"] = \
        result["c2_prep_ms"]["upgo_coef_0.5"]["median"] - result["c2_prep_ms"]["upgo_coef_0.0"]["median"]
    print(json.dumps(result))


if __name__ == "__main__":
    main()
