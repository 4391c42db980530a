"""Cost of dual-clip PPO (``dual_clip``) on the device, at C2 (LSTM-128, seq_len 512, 256 sequences = 131,072 tokens).

1. The fused loss kernel alone at C2's token count with a valid mask: ``dc_ppo_loss_fwd_bwd_masked`` against
   ``_dual_clip`` (c = 3, per-head ratios), and ``_joint`` against ``_dual_clip`` with the joint ratio, on the same
   preallocated inputs, each call timed alone between two CUDA events, the four alternated call by call; median, min and
   max of ``--calls`` calls each.  The old log-probs are spread so that about a tenth of the rows bind.
2. The replayed C2 step of two optimizers, one without dual clip and one with ``dual_clip=3``, each on its own batch of
   the same rollouts, alternated step by step.

Prints one JSON line with the card and its power limit.

    python tools/dual_clip_bench.py [--calls 200] [--steps 30]
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

S, B, H, C = 512, 256, 128, 3.0


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _optimizer(**kw):
    return DotaOptimizer(rmq_host="dual_clip_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1,
                         min_seq_per_epoch=4, seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=H, cell="lstm", **kw)


def _stats(xs):
    xs = sorted(xs)
    return {"median": float(np.median(xs)), "min": xs[0], "max": xs[-1], "n": len(xs)}


def _kernel_rows(calls):
    """The four loss calls on the same random C2-sized inputs (90 % valid tokens), alternated; microseconds per call."""
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
    lp = ops.selected_logp(logits, masks, actions)
    old = lp + 6.0 * torch.rand(N, 5, generator=g, device=d) - 3.0     # per-head ratios in about [0.05, 20]
    old_joint = lp.clone()
    old_joint[:, 0] += 6.0 * torch.rand(N, generator=g, device=d) - 3.0
    adv, ret, value, old_value = (torch.randn(N, generator=g, device=d) for _ in range(4))
    valid = ops._u8(torch.rand(N, generator=g, device=d) < 0.9)
    dlogits = [torch.empty_like(t) for t in logits]
    dvalue = torch.empty_like(value)
    out = torch.empty(_lib.LOSS_SLOTS, device=d)
    stats = torch.empty(_lib.PPO_STATS_SLOTS, device=d)
    d_stats = torch.empty(_lib.DUAL_CLIP_STATS_SLOTS, device=d)
    n_act = torch.empty(5, dtype=torch.int32, device=d)
    ws = torch.empty(_lib.PPO_WORKSPACE_BYTES, dtype=torch.uint8, device=d)
    hp = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5)
    c = torch.tensor([C], dtype=torch.float64, device=d)
    u8 = [ops._u8(t) for t in masks], [ops._u8(t) for t in actions]
    lib, stream = _lib.load(), _lib.stream_ptr()
    ld = (_lib._c.c_int64 * 5)(*ops.HEAD_SIZES)
    lp5, m5, a5, d5 = _lib.ptr5(logits), _lib.ptr5(u8[0]), _lib.ptr5(u8[1]), _lib.ptr5(dlogits)

    def head(o):
        return (lp5, ld, m5, a5, o.data_ptr(), adv.data_ptr(), ret.data_ptr(), value.data_ptr(), 1, old_value.data_ptr(),
                valid.data_ptr())
    tail = (N, hp.data_ptr(), d5, ld, dvalue.data_ptr(), 1, out.data_ptr(), stats.data_ptr(), n_act.data_ptr(),
            ws.data_ptr(), stream)

    def dual(joint):
        o = old_joint if joint else old
        return lib.dc_ppo_loss_fwd_bwd_dual_clip(
            lp5, ld, m5, a5, o.data_ptr(), None, None, adv.data_ptr(), ret.data_ptr(), value.data_ptr(), 1,
            old_value.data_ptr(), valid.data_ptr(), N, hp.data_ptr(), None, c.data_ptr(), 1 if joint else 0, d5, ld,
            dvalue.data_ptr(), 1, out.data_ptr(), stats.data_ptr(), None, None, d_stats.data_ptr(), n_act.data_ptr(),
            ws.data_ptr(), stream)
    fns = {"masked": lambda: lib.dc_ppo_loss_fwd_bwd_masked(*head(old), *tail), "dual_clip": lambda: dual(False),
           "joint": lambda: lib.dc_ppo_loss_fwd_bwd_joint(*head(old_joint), *tail), "dual_clip_joint": lambda: dual(True)}
    bound = {}
    for _ in range(10):
        for k, f in fns.items():
            assert f() == 0
            if k.startswith("dual"):
                torch.cuda.synchronize()
                bound[k] = d_stats.tolist()
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
    res["dual_clip_over_masked_median"] = res["dual_clip"]["median"] / res["masked"]["median"]
    res["dual_clip_joint_over_joint_median"] = res["dual_clip_joint"]["median"] / res["joint"]["median"]
    res["bound_fraction"] = {"per_head_mean": bound["dual_clip"][0], "joint": bound["dual_clip_joint"][6]}
    # algorithmic bytes of the loss pass: 686 per token + 1 for valid + 4 for the old value; the cap adds none
    res["loss_pass_bytes_per_token"] = {k: 691 for k in fns}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed loss-kernel calls per entry point (median; >= 200)")
    ap.add_argument("--steps", type=int, default=30, help="timed C2 steps per optimizer")
    args = ap.parse_args()
    if args.calls < 200:
        ap.error("--calls must be >= 200")
    if not torch.cuda.is_available():
        raise SystemExit("dual_clip_bench needs a CUDA device")
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls,
              "config": "C2: LSTM-128, seq_len 512, 256 sequences; c = %g" % C}
    result["loss_kernel_us"] = _kernel_rows(args.calls)

    pool = [make_rollout(2 * S, 40_000 + i) for i in range(8)]
    rollouts = [pool[i % len(pool)] for i in range(B // 2)]          # two whole sequences each: B sequences
    opts = {"without": _optimizer(), "dual_clip_3": _optimizer(dual_clip=C)}
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
    result["c2_step_ms"]["dual_clip_3_over_without_median"] = \
        result["c2_step_ms"]["dual_clip_3"]["median"] / result["c2_step_ms"]["without"]["median"]
    result["c2_step_dual_clip_fraction"] = opts["dual_clip_3"].last_dual_clip_stats["fraction"]
    for o in opts.values():
        o.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
