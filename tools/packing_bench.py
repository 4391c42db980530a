"""Cost of the reset path of the recurrence and what sequence packing saves per PPO epoch.

1. The recurrence kernels alone at C2 (LSTM-128, 256 sequences x 512 steps) and C3 (GRU-256, 1024 x 512): forward and
   backward of ``dc_rnn_seq_fwd_reset`` / ``_bwd_reset`` with one reset per sequence (at a step that varies by sequence)
   against ``dc_rnn_seq_fwd`` / ``_bwd`` on the same inputs, alternated call by call, each call timed alone between two
   CUDA events (the gate buffer is restored before every call, outside the timed span); median, min and max.
2. ``train_epochs`` (one epoch, one minibatch) per iteration on ragged rollouts of 1000-1400 steps, LSTM-128 at
   ``seq_len`` 512 and 1024, packed (``pack_sequences=True``) against unpacked, both with ``mask_padding``: two optimizers
   from the same seed, steps alternated, replayed from their CUDA graphs, each timed on the host around ``train_epochs``
   (which ends in the step's host sync).  With the batch sizes and trained token counts.

Prints one JSON line with the card and its power limit.

    python tools/packing_bench.py [--calls 20] [--steps 10]
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


def _timed(fns, calls, before):
    """{name: stats of microseconds per call}, the calls of ``fns`` alternated, ``before()`` untimed ahead of each."""
    pairs = {k: [] for k in fns}
    for _ in range(calls):
        for k, f in fns.items():
            before()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            assert f() == 0, _lib.load().dc_last_error()
            e1.record()
            pairs[k].append((e0, e1))
    torch.cuda.synchronize()
    return {k: _stats([1000.0 * a.elapsed_time(b) for a, b in v]) for k, v in pairs.items()}


def _kernels(cell, H, B, S, calls):
    d = torch.device("cuda")
    G = ops.GATES[cell]
    g = torch.Generator(device=d).manual_seed(0)
    gi = torch.randn(S * B, G * H, generator=g, device=d)
    gates = torch.empty_like(gi)
    w_hh = torch.randn(G * H, H, generator=g, device=d) / H ** 0.5
    b_hh = torch.randn(G * H, generator=g, device=d) * 0.1
    ybuf = torch.randn(S + 1, B, H, generator=g, device=d) * 0.5
    cbuf = torch.randn(S + 1, B, H, generator=g, device=d) * 0.5
    dy = torch.randn(S, B, H, generator=g, device=d)
    dh0, dc0 = torch.empty(B, H, device=d), torch.empty(B, H, device=d)
    slot = torch.full((S, B), -1, dtype=torch.int32, device=d)
    slot[torch.arange(B, device=d) * 7 % S, torch.arange(B, device=d)] = 0       # one reset per sequence, K = 1
    prev = torch.randn(1, B, H, generator=g, device=d) * 0.5
    pre = torch.randn(1, B, G * H, generator=g, device=d)
    ws = ops._rnn_workspace(cell, B, H, d)
    lib, st, c = _lib.load(), _lib.stream_ptr(), ops.CELL_ID[cell]
    fwd = {"plain": lambda: lib.dc_rnn_seq_fwd(c, gates.data_ptr(), w_hh.data_ptr(), b_hh.data_ptr(), ybuf.data_ptr(),
                                               cbuf.data_ptr(), B, S, H, ws.data_ptr(), st),
           "reset": lambda: lib.dc_rnn_seq_fwd_reset(c, gates.data_ptr(), w_hh.data_ptr(), b_hh.data_ptr(), ybuf.data_ptr(),
                                                     cbuf.data_ptr(), slot.data_ptr(), prev.data_ptr(), pre.data_ptr(), 1,
                                                     B, S, H, ws.data_ptr(), st)}
    out = {"fwd_us": _timed(fwd, calls, lambda: gates.copy_(gi))}
    fwd["plain"]()
    acts = gates.clone()
    bwd = {"plain": lambda: lib.dc_rnn_seq_bwd(c, gates.data_ptr(), w_hh.data_ptr(), ybuf.data_ptr(), cbuf.data_ptr(),
                                               dy.data_ptr(), None, None, dh0.data_ptr(), dc0.data_ptr(), B, S, H,
                                               ws.data_ptr(), st),
           "reset": lambda: lib.dc_rnn_seq_bwd_reset(c, gates.data_ptr(), w_hh.data_ptr(), ybuf.data_ptr(), cbuf.data_ptr(),
                                                     dy.data_ptr(), None, None, dh0.data_ptr(), dc0.data_ptr(),
                                                     slot.data_ptr(), prev.data_ptr(), 1, B, S, H, ws.data_ptr(), st)}
    out["bwd_us"] = _timed(bwd, calls, lambda: gates.copy_(acts))
    for k in ("fwd_us", "bwd_us"):
        out[k]["reset_over_plain_median"] = out[k]["reset"]["median"] / out[k]["plain"]["median"]
    return out


def _optimizer(S, pack):
    return DotaOptimizer(rmq_host="packing_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1,
                         min_seq_per_epoch=4, seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=128, cell="lstm", mask_padding=True, pack_sequences=pack)


def _epochs(S, n_rollouts, steps, pool):
    rng = np.random.default_rng(S)
    lens = rng.integers(1000, 1401, size=n_rollouts).tolist()

    def cut(i, L):
        r = pool[i % len(pool)]
        return {k: ({kk: vv[:L] for kk, vv in v.items()} if isinstance(v, dict) else v[:L]) if k in
                ("observations", "masks", "actions", "rewards") else v for k, v in r.items()}
    rollouts = [cut(i, L) for i, L in enumerate(lens)]
    opts = {"unpacked": _optimizer(S, False), "packed": _optimizer(S, True)}
    batches = {k: o.batch_from_rollouts(rollouts) for k, o in opts.items()}
    res = {"seq_len": S, "rollouts": n_rollouts, "real_steps": int(sum(lens))}
    for k, b in batches.items():
        res[k + "_sequences"] = b.batch_size
        res[k + "_tokens"] = b.batch_size * S
    for _ in range(3):                               # eager, capture, replay
        for k, o in opts.items():
            o.train_epochs(batches[k])
    times = {k: [] for k in opts}
    for _ in range(steps):
        for k, o in opts.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            o.train_epochs(batches[k])
            times[k].append(1e3 * (time.perf_counter() - t0))
    res["ms_per_iteration"] = {k: _stats(v) for k, v in times.items()}
    res["packed_over_unpacked_median"] = res["ms_per_iteration"]["packed"]["median"] / \
        res["ms_per_iteration"]["unpacked"]["median"]
    res["token_ratio"] = res["packed_tokens"] / res["unpacked_tokens"]
    for o in opts.values():
        o.close()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=20, help="timed recurrence calls per entry point")
    ap.add_argument("--steps", type=int, default=10, help="timed iterations per optimizer")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("packing_bench needs a CUDA device")
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit()}
    result["kernels_c2_lstm128_B256_S512"] = _kernels("lstm", 128, 256, 512, args.calls)
    result["kernels_c3_gru256_B1024_S512"] = _kernels("gru", 256, 1024, 512, args.calls)
    pool = [make_rollout(1400, 40_000 + i) for i in range(8)]
    result["train_epochs_lstm128_S512"] = _epochs(512, 100, args.steps, pool)
    result["train_epochs_lstm128_S1024"] = _epochs(1024, 64, args.steps, pool)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
