"""Per-call time of the two advantage scans of experience prep, ``dc_gae_scan`` and ``dc_vtrace_scan``, at the shapes prep
runs them: C2's batch (256 rollouts x 512 rows) and a stream iteration (~70 rollouts of up to 1380 steps, padded to a
multiple of seq_len 16).  Each call is timed alone between two CUDA events on the launching stream; the median of
``--calls`` calls is reported, with the card and its power limit.  Prints one JSON line.

    python tools/vtrace_bench.py [--calls 200]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dotaclient_b200 import ops  # noqa: E402


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _inputs(lengths, seq_len, seed):
    """Rollout-major inputs as prep lays them out: every rollout padded to a multiple of seq_len, 10 sub-rewards per row."""
    g = torch.Generator().manual_seed(seed)
    padded = [(L + seq_len - 1) // seq_len * seq_len for L in lengths]
    n = sum(padded)
    dev = torch.device("cuda")
    rewards = (0.01 * torch.randn(n, 10, generator=g)).to(dev)
    values = torch.randn(n, generator=g).to(dev)
    lp_target = (-torch.rand(n, 5, generator=g)).to(dev)
    lp_behaviour = (lp_target.cpu() + 0.1 * torch.randn(n, 5, generator=g)).to(dev)
    seg = torch.tensor(np.concatenate([[0], np.cumsum(padded)]), dtype=torch.int64, device=dev)
    valid = torch.tensor(lengths, dtype=torch.int64, device=dev)
    return rewards, values, lp_target, lp_behaviour, seg, valid


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
    times = sorted(1000.0 * e0.elapsed_time(e1) for e0, e1 in pairs)
    return float(np.median(times)), times[0], times[-1]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed calls per kernel and shape (median reported; >= 50)")
    args = ap.parse_args()
    if args.calls < 50:
        ap.error("--calls must be >= 50")
    if not torch.cuda.is_available():
        raise SystemExit("vtrace_bench needs a CUDA device")
    rng = np.random.RandomState(0)
    shapes = {
        "c2_256x512": [512] * 256,
        "stream_70x1380": [1380] + [int(v) for v in rng.randint(200, 1381, size=69)],
    }
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls, "shapes": {}}
    for name, lengths in shapes.items():
        r, v, lt, lb, seg, valid = _inputs(lengths, 16, 1)
        gae = _median_us(lambda: ops.gae_scan(r, v, seg, gamma=0.98, lam=0.97), args.calls)
        vtr = _median_us(lambda: ops.vtrace_scan(r, v, lt, lb, seg, 0.98, 0.97, 1.0, 1.0, valid_len=valid, stats=True),
                         args.calls)
        rows = int(seg[-1])
        result["shapes"][name] = {
            "segments": len(lengths), "rows": rows,
            "gae_scan_us": {"median": gae[0], "min": gae[1], "max": gae[2]},
            "vtrace_scan_us": {"median": vtr[0], "min": vtr[1], "max": vtr[2]},
            # algorithmic HBM bytes per call: rewards, values (+ two [rows, 5] log-probs) read, two outputs written
            "gae_bytes": rows * (40 + 4 + 8), "vtrace_bytes": rows * (40 + 4 + 40 + 8),
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
