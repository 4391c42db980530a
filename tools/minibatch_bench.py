"""Cost of minibatch PPO on the device: minibatch assembly and whole epochs.

1. ``ExperienceBatch.gather`` (one ``dc_gather_columns`` launch) against per-tensor ``index_select`` at two sizes: a quarter
   of C2's batch (64 of 256 sequences x 512 steps, LSTM-128) and a quarter of the reference's default iteration (256 of 1024
   sequences x 16 steps, GRU-256).  Each call is timed alone between two CUDA events; the median of ``--calls`` calls is
   reported, for the whole ``gather`` call (allocation, host index check and upload, launch) and for the kernel alone, with
   the algorithmic bytes (read + write) over the kernel time against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.
2. Wall time of ``train_epochs`` (``--epochs`` epochs, ending in a device synchronise) at C2's batch with 1, 2 and 4
   minibatches, per optimizer step, and the share of it spent in gathers (the gathers of one epoch timed alone).

Batches are real experience prep outputs of synthetic rollouts.  Prints one JSON line with the card and its power limit.

    python tools/minibatch_bench.py [--calls 200] [--epochs 4]
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
from dotaclient_b200 import _lib  # noqa: E402
from dotaclient_b200.optimizer import DotaOptimizer, minibatch_indices  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

HBM_DATASHEET_TBPS = 3.35


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _optimizer(hidden, cell, seq_len, num_minibatches=1, epochs=4):
    return DotaOptimizer(rmq_host="minibatch_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=epochs,
                         min_seq_per_epoch=4, seq_len=seq_len, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=hidden, cell=cell, num_minibatches=num_minibatches)


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


def _gather_row(batch, n_pick, calls):
    idx = np.random.default_rng(0).permutation(batch.batch_size)[:n_pick]
    idx_dev = torch.as_tensor(idx, device=batch.advantages.device)
    call = _median_us(lambda: batch.gather(idx), calls)
    torch_ = _median_us(lambda: batch.map(lambda v: v.index_select(1, idx_dev)), calls)
    # the kernel alone: one dc_gather_columns launch into preallocated outputs (no allocation, no index check or upload)
    out = batch.gather(idx)
    pairs = [(s, d) for (_, _, s), (_, _, d) in zip(batch.tensors(), out.tensors())]
    D = _lib.GatherDesc
    descs = (D * len(pairs))(*[D(s.data_ptr(), d.data_ptr(), s.shape[0], s.shape[1], s[0, 0].numel() * s.element_size())
                               for s, d in pairs])
    lib, stream = _lib.load(), _lib.stream_ptr()
    kernel = _median_us(lambda: lib.dc_gather_columns(descs, len(pairs), idx_dev.data_ptr(), n_pick, stream), calls)
    moved = batch.nbytes() * n_pick // batch.batch_size          # bytes written = bytes read
    return {"sequences": "%d of %d" % (n_pick, batch.batch_size), "seq_len": batch.seq_len,
            "tensors": len(pairs), "bytes_each_way": moved,
            "gather_call_us": {"median": call[0], "min": call[1], "max": call[2]},
            "gather_kernel_us": {"median": kernel[0], "min": kernel[1], "max": kernel[2]},
            "index_select_us": {"median": torch_[0], "min": torch_[1], "max": torch_[2]},
            "kernel_tbps_read_plus_write": 2 * moved / (kernel[0] * 1e-6) / 1e12,
            "kernel_share_of_datasheet_hbm": 2 * moved / (kernel[0] * 1e-6) / 1e12 / HBM_DATASHEET_TBPS,
            "index_select_tbps_read_plus_write": 2 * moved / (torch_[0] * 1e-6) / 1e12}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed gather calls per size and method (median; >= 200)")
    ap.add_argument("--epochs", type=int, default=4)
    args = ap.parse_args()
    if args.calls < 200:
        ap.error("--calls must be >= 200")
    if not torch.cuda.is_available():
        raise SystemExit("minibatch_bench needs a CUDA device")
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(),
              "hbm_datasheet_tbps": HBM_DATASHEET_TBPS, "calls": args.calls, "gather": {}, "train_epochs": {}}

    ref = _optimizer(256, "gru", 16)
    ref_batch = ref.batch_from_rollouts([make_rollout(16, 10_000 + i) for i in range(1024)])
    result["gather"]["reference_default_quarter"] = _gather_row(ref_batch, 256, args.calls)
    del ref, ref_batch

    c2 = _optimizer(128, "lstm", 512, epochs=args.epochs)
    c2_batch = c2.batch_from_rollouts([make_rollout(512, 20_000 + i) for i in range(256)])
    result["gather"]["c2_quarter"] = _gather_row(c2_batch, 64, args.calls)

    for M in (1, 2, 4):
        c2.num_minibatches = M
        c2.train_epochs(c2_batch)                      # warm-up: every minibatch shape runs, is captured and replayed
        c2.train_epochs(c2_batch)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c2.train_epochs(c2_batch)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        steps = args.epochs * M
        gather_ms = 0.0
        if M > 1:
            idxs = minibatch_indices(c2_batch.batch_size, M, np.random.default_rng(1))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for idx in idxs:
                c2_batch.gather(idx)
            e1.record()
            torch.cuda.synchronize()
            gather_ms = e0.elapsed_time(e1) * args.epochs      # one epoch's gathers, times the epochs
        result["train_epochs"]["M%d" % M] = {"steps": steps, "wall_ms": 1e3 * wall, "ms_per_step": 1e3 * wall / steps,
                                             "gather_ms": gather_ms, "gather_share": gather_ms / (1e3 * wall)}
    c2.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
