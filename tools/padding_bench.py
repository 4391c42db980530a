"""Cost of ``mask_padding`` on the device, and how much of a batch is padding.

1. The fused loss kernel alone at C2's token count (256 sequences x 512 steps = 131,072 tokens): one
   ``dc_ppo_loss_fwd_bwd_masked`` call (workspace clear + statistics pass + loss pass) against one
   ``dc_ppo_loss_fwd_bwd_dev`` call on the same preallocated inputs, each call timed alone between two CUDA events, the
   two entry points alternated call by call; median, min and max of ``--calls`` calls each.  The mask is that of the
   ragged rollouts of part 2.
2. The whole C2 training step (LSTM-128, S = 512, B = 256, replayed from its CUDA graph) on one batch prepared from
   ragged rollouts of 1000-1400 steps, trained by two optimizers from the same seed, one with ``mask_padding`` and one
   without; their steps alternate, each timed on the host around ``train()`` (which ends in the step's host sync).
3. The padding share of that batch, and the share expected from shapes alone for rollout lengths uniform in 1000-1400 at
   ``seq_len`` 16, 128 and 512.

Prints one JSON line with the card and its power limit.

    python tools/padding_bench.py [--calls 200] [--steps 30]
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


def _optimizer(mask_padding):
    return DotaOptimizer(rmq_host="padding_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1,
                         min_seq_per_epoch=4, seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=H, cell="lstm", mask_padding=mask_padding)


def _ragged_lengths(rng):
    """Rollout lengths in 1000-1400 whose chunks of S add up to exactly B sequences (the last one is shortened)."""
    lens, chunks = [], 0
    while chunks < B:
        L = int(rng.integers(1000, 1401))
        n = (L + S - 1) // S
        if chunks + n > B:
            L = (B - chunks) * S - int(rng.integers(0, S))
            n = B - chunks
        lens.append(L)
        chunks += n
    return lens


def _stats(xs):
    xs = sorted(xs)
    return {"median": float(np.median(xs)), "min": xs[0], "max": xs[-1], "n": len(xs)}


def _kernel_rows(valid, calls):
    """Both entry points on the same random C2-sized inputs, alternated; microseconds per call."""
    d = valid.device
    N = valid.numel()
    g = torch.Generator(device=d).manual_seed(0)
    logits = [torch.randn(N, n, generator=g, device=d) for n in ops.HEAD_SIZES]
    masks = [torch.rand(N, n, generator=g, device=d) < 0.7 for n in ops.HEAD_SIZES]
    actions = []
    for n, m in zip(ops.HEAD_SIZES, masks):
        a = torch.zeros(N, n, dtype=torch.bool, device=d)
        a[torch.arange(N, device=d), torch.randint(0, n, (N,), generator=g, device=d)] = True
        actions.append(a & m)
    old = torch.randn(N, 5, generator=g, device=d) - 2.0
    adv, ret, value, old_value = (torch.randn(N, generator=g, device=d) for _ in range(4))
    dlogits = [torch.empty_like(t) for t in logits]
    dvalue = torch.empty_like(value)
    out = torch.empty(_lib.LOSS_SLOTS, device=d)
    stats = torch.empty(_lib.PPO_STATS_SLOTS, device=d)
    n_act = torch.empty(5, dtype=torch.int32, device=d)
    ws = torch.empty(_lib.PPO_WORKSPACE_BYTES, dtype=torch.uint8, device=d)
    hp = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5)
    u8 = [ops._u8(t) for t in masks], [ops._u8(t) for t in actions]
    vmask = ops._u8(valid)
    lib, stream = _lib.load(), _lib.stream_ptr()
    ld = (_lib._c.c_int64 * 5)(*ops.HEAD_SIZES)
    head = (_lib.ptr5(logits), ld, _lib.ptr5(u8[0]), _lib.ptr5(u8[1]), old.data_ptr(), adv.data_ptr(), ret.data_ptr(),
            value.data_ptr(), 1, old_value.data_ptr())
    tail = (N, hp.data_ptr(), _lib.ptr5(dlogits), ld, dvalue.data_ptr(), 1, out.data_ptr(), stats.data_ptr(),
            n_act.data_ptr(), ws.data_ptr(), stream)
    fns = {"dev": lambda: lib.dc_ppo_loss_fwd_bwd_dev(*head, *tail),
           "masked": lambda: lib.dc_ppo_loss_fwd_bwd_masked(*head, vmask.data_ptr(), *tail)}
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
    res["valid_tokens"] = int(valid.sum())
    res["masked_over_dev_median"] = res["masked"]["median"] / res["dev"]["median"]
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed loss-kernel calls per entry point (median; >= 200)")
    ap.add_argument("--steps", type=int, default=30, help="timed C2 steps per optimizer")
    args = ap.parse_args()
    if args.calls < 200:
        ap.error("--calls must be >= 200")
    if not torch.cuda.is_available():
        raise SystemExit("padding_bench needs a CUDA device")
    rng = np.random.default_rng(0)
    lens = _ragged_lengths(rng)
    pool = [make_rollout(1400, 30_000 + i) for i in range(8)]

    def cut(i, L):
        r = pool[i % len(pool)]
        return {k: ({kk: vv[:L] for kk, vv in v.items()} if isinstance(v, dict) else v[:L]) if k in
                ("observations", "masks", "actions", "rewards") else v for k, v in r.items()}
    rollouts = [cut(i, L) for i, L in enumerate(lens)]

    masked = _optimizer(True)
    plain = _optimizer(False)
    batch = masked.batch_from_rollouts(rollouts)
    assert (batch.seq_len, batch.batch_size) == (S, B)
    plain_batch = plain.batch_from_rollouts(rollouts)
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls,
              "config": "C2: LSTM-128, seq_len 512, 256 sequences", "rollouts": len(lens)}
    result["loss_kernel_us"] = _kernel_rows(batch.valid.reshape(-1).contiguous(), args.calls)

    for _ in range(3):                               # eager, capture, replay
        masked.train(batch)
        plain.train(plain_batch)
    times = {"mask_padding": [], "default": []}
    for _ in range(args.steps):
        for key, opt, b in (("default", plain, plain_batch), ("mask_padding", masked, batch)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            opt.train(b)
            times[key].append(1e3 * (time.perf_counter() - t0))
    result["c2_step_ms"] = {k: _stats(v) for k, v in times.items()}
    result["c2_step_ms"]["masked_over_default_median"] = \
        result["c2_step_ms"]["mask_padding"]["median"] / result["c2_step_ms"]["default"]["median"]

    tokens = B * S
    result["padding_share"] = {"this_batch": (tokens - sum(lens)) / tokens}
    for s in (16, 128, 512):
        Ls = np.arange(1000, 1401)
        padded = (Ls + s - 1) // s * s
        result["padding_share"]["uniform_1000_1400_seq_len_%d" % s] = float((padded - Ls).sum() / padded.sum())
    masked.close()
    plain.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
