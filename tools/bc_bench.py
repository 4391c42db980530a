"""Cost of behaviour cloning (``objective='bc'``) on the device, at C2 (LSTM-128, seq_len 512, 256 sequences = 131,072
tokens).

1. The fused loss kernel alone at C2's token count with a valid mask: ``dc_ppo_loss_fwd_bwd_masked`` against
   ``dc_ppo_loss_fwd_bwd_bc``, on the same preallocated inputs, each call timed alone between two CUDA events, the two
   alternated call by call; median, min and max of ``--calls`` calls each.
2. The replayed C2 step of an optimizer with ``objective='ppo'`` against one with ``objective='bc'``, on the same batch
   (synthetic rollouts, whose rows follow the action hierarchy, so they are valid demonstrations), alternated step by step.

Prints one JSON line with the card and its power limit.

    python tools/bc_bench.py [--calls 200] [--steps 30]
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


def _optimizer(**kw):
    return DotaOptimizer(rmq_host="bc_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1, min_seq_per_epoch=4,
                         seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                         log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H,
                         cell="lstm", **kw)


def _stats(xs):
    xs = sorted(xs)
    return {"median": float(np.median(xs)), "min": xs[0], "max": xs[-1], "n": len(xs)}


def _kernel(calls):
    """The two loss calls on the same random C2-sized inputs (90 % valid tokens), alternated; microseconds per call."""
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
    adv, ret, value, old_value = (torch.randn(N, generator=g, device=d) for _ in range(4))
    valid = ops._u8(torch.rand(N, generator=g, device=d) < 0.9)
    dlogits = [torch.empty_like(t) for t in logits]
    dvalue = torch.empty_like(value)
    out = torch.empty(_lib.LOSS_SLOTS, device=d)
    stats = torch.empty(_lib.PPO_STATS_SLOTS, device=d)
    bc_stats = torch.empty(_lib.BC_STATS_SLOTS, device=d)
    n_act = torch.empty(5, dtype=torch.int32, device=d)
    ws = torch.empty(_lib.PPO_WORKSPACE_BYTES, dtype=torch.uint8, device=d)
    hp = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5)
    u8 = [ops._u8(t) for t in masks], [ops._u8(t) for t in actions]
    lib, stream = _lib.load(), _lib.stream_ptr()
    ld = (_lib._c.c_int64 * 5)(*ops.HEAD_SIZES)
    lp5, m5, a5, d5 = _lib.ptr5(logits), _lib.ptr5(u8[0]), _lib.ptr5(u8[1]), _lib.ptr5(dlogits)

    def masked():
        return lib.dc_ppo_loss_fwd_bwd_masked(lp5, ld, m5, a5, old.data_ptr(), adv.data_ptr(), ret.data_ptr(),
                                              value.data_ptr(), 1, old_value.data_ptr(), valid.data_ptr(), N, hp.data_ptr(),
                                              d5, ld, dvalue.data_ptr(), 1, out.data_ptr(), stats.data_ptr(),
                                              n_act.data_ptr(), ws.data_ptr(), stream)

    def bc():
        return lib.dc_ppo_loss_fwd_bwd_bc(lp5, ld, m5, a5, adv.data_ptr(), ret.data_ptr(), value.data_ptr(), 1,
                                          old_value.data_ptr(), valid.data_ptr(), N, hp.data_ptr(), d5, ld, dvalue.data_ptr(),
                                          1, out.data_ptr(), stats.data_ptr(), bc_stats.data_ptr(), n_act.data_ptr(),
                                          ws.data_ptr(), stream)
    fns = {"masked": masked, "bc": bc}
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
    res["bc_over_masked_median"] = res["bc"]["median"] / res["masked"]["median"]
    # algorithmic bytes of the loss pass: 686 per token + 1 for valid + 4 for the old value; bc reads no old_logp (20) and
    # no advantage (4)
    res["loss_pass_bytes_per_token"] = {"masked": 691, "bc": 691 - 24}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed loss-kernel calls per entry point (median; >= 200)")
    ap.add_argument("--steps", type=int, default=30, help="timed C2 steps per objective")
    args = ap.parse_args()
    if args.calls < 200:
        ap.error("--calls must be >= 200")
    if not torch.cuda.is_available():
        raise SystemExit("bc_bench needs a CUDA device")
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls,
              "config": "C2: LSTM-128, seq_len 512, 256 sequences"}
    result["loss_kernel_us"] = _kernel(args.calls)

    pool = [make_rollout(2 * S, 40_000 + i) for i in range(8)]
    rollouts = [pool[i % len(pool)] for i in range(B // 2)]          # two whole sequences each: B sequences
    opts = {"ppo": _optimizer(), "bc": _optimizer(objective="bc")}
    batches = {k: o.batch_from_rollouts(rollouts) for k, o in opts.items()}
    assert all((b.seq_len, b.batch_size) == (S, B) for b in batches.values())
    for _ in range(3):                               # eager, capture, replay
        for k, o in opts.items():
            o.train(batches[k])
    times = {k: [] for k in opts}
    for _ in range(args.steps):
        for k, o in opts.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            o.train(batches[k])
            times[k].append(1e3 * (time.perf_counter() - t0))
    assert all(any(isinstance(v, tuple) for v in o._graphs.values()) for o in opts.values())
    result["c2_step_ms"] = {k: _stats(v) for k, v in times.items()}
    result["c2_step_ms"]["bc_over_ppo_median"] = result["c2_step_ms"]["bc"]["median"] / result["c2_step_ms"]["ppo"]["median"]
    result["bc_stats_last_step"] = opts["bc"].last_bc_stats
    for o in opts.values():
        o.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
