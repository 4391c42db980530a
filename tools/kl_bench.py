"""Cost of KL control (``kl_coef`` / ``kl_stop``) on the device.

1. The fused loss kernel alone at C2's token count (256 sequences x 512 steps = 131,072 tokens): one
   ``dc_ppo_loss_fwd_bwd_kl`` call with beta > 0 in each ratio mode against ``dc_ppo_loss_fwd_bwd_masked`` and
   ``dc_ppo_loss_fwd_bwd_joint`` on the same preallocated inputs and valid mask, each call timed alone between two CUDA
   events, the four calls alternated call by call; median, min and max of ``--calls`` calls each.
2. The whole C2 training step (LSTM-128, S = 512, B = 256, replayed from its CUDA graph) on one batch, trained by two
   optimizers from the same seed, one with ``kl_coef=0.2, kl_stop=100`` and one without KL control; their steps alternate,
   each timed on the host around ``train()`` (which ends in the step's host sync).
3. The prep kernel: ``dc_selected_logp_rows`` against ``dc_selected_logp`` at the same token count, alternated.

Prints one JSON line with the card and its power limit.

    python tools/kl_bench.py [--calls 200] [--steps 30]
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
    return DotaOptimizer(rmq_host="kl_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1,
                         min_seq_per_epoch=4, seq_len=S, learning_rate=5e-5, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True,
                         hidden_size=H, cell="lstm", **kw)


def _stats(xs):
    xs = sorted(xs)
    return {"median": float(np.median(xs)), "min": xs[0], "max": xs[-1], "n": len(xs)}


def _kernel_rows(calls):
    """The four entry points on the same random C2-sized inputs (90 % valid tokens), alternated; microseconds per call.
    Also the two prep kernels, alternated."""
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
    n_act = torch.empty(5, dtype=torch.int32, device=d)
    ws = torch.empty(_lib.PPO_WORKSPACE_BYTES, dtype=torch.uint8, device=d)
    hp = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5, kl_coef=0.2)
    sel = torch.empty(N, 5, device=d)
    rows = torch.empty(N, _lib.KL_ROW_FLOATS, device=d)
    kl_out = torch.empty(2, device=d)
    u8 = [ops._u8(t) for t in masks], [ops._u8(t) for t in actions]
    lib, stream = _lib.load(), _lib.stream_ptr()
    ld = (_lib._c.c_int64 * 5)(*ops.HEAD_SIZES)
    head = (_lib.ptr5(logits), ld, _lib.ptr5(u8[0]), _lib.ptr5(u8[1]), old.data_ptr(), adv.data_ptr(), ret.data_ptr(),
            value.data_ptr(), 1, old_value.data_ptr(), valid.data_ptr())
    tail = (N, hp.data_ptr(), _lib.ptr5(dlogits), ld, dvalue.data_ptr(), 1, out.data_ptr(), stats.data_ptr(),
            n_act.data_ptr(), ws.data_ptr(), stream)
    lp = (_lib.ptr5(logits), _lib.ptr5(u8[0]), _lib.ptr5(u8[1]), N, sel.data_ptr())
    assert lib.dc_selected_logp_rows(*lp, rows.data_ptr(), stream) == 0

    def kl(joint):
        return lib.dc_ppo_loss_fwd_bwd_kl(head[0], ld, head[2], head[3], old.data_ptr(), rows.data_ptr(), adv.data_ptr(),
                                          ret.data_ptr(), value.data_ptr(), 1, old_value.data_ptr(), valid.data_ptr(), N,
                                          hp.data_ptr(), joint, _lib.ptr5(dlogits), ld, dvalue.data_ptr(), 1,
                                          out.data_ptr(), stats.data_ptr(), kl_out.data_ptr(), n_act.data_ptr(),
                                          ws.data_ptr(), stream)
    fns = {"masked": lambda: lib.dc_ppo_loss_fwd_bwd_masked(*head, *tail),
           "kl_per_head": lambda: kl(0),
           "joint": lambda: lib.dc_ppo_loss_fwd_bwd_joint(*head, *tail),
           "kl_joint": lambda: kl(1),
           "prep_selected_logp": lambda: lib.dc_selected_logp(*lp, stream),
           "prep_selected_logp_rows": lambda: lib.dc_selected_logp_rows(*lp, rows.data_ptr(), stream)}
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
    res["kl_over_masked_median"] = res["kl_per_head"]["median"] / res["masked"]["median"]
    res["kl_joint_over_joint_median"] = res["kl_joint"]["median"] / res["joint"]["median"]
    res["prep_added_us_median"] = res["prep_selected_logp_rows"]["median"] - res["prep_selected_logp"]["median"]
    # algorithmic bytes of the loss pass: 686 per token + 1 for valid + 4 for the old value, + 260 for the old rows
    res["loss_pass_bytes_per_token"] = {"masked": 691, "kl": 691 + 4 * _lib.KL_ROW_FLOATS}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed loss-kernel calls per entry point (median; >= 200)")
    ap.add_argument("--steps", type=int, default=30, help="timed C2 steps per optimizer")
    args = ap.parse_args()
    if args.calls < 200:
        ap.error("--calls must be >= 200")
    if not torch.cuda.is_available():
        raise SystemExit("kl_bench needs a CUDA device")
    pool = [make_rollout(2 * S, 40_000 + i) for i in range(8)]
    rollouts = [pool[i % len(pool)] for i in range(B // 2)]          # two whole sequences each: B sequences
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls,
              "config": "C2: LSTM-128, seq_len 512, 256 sequences"}
    result["loss_kernel_us"] = _kernel_rows(args.calls)

    kl, default = _optimizer(kl_coef=0.2, kl_stop=100.0), _optimizer()
    batch_k, batch_d = kl.batch_from_rollouts(rollouts), default.batch_from_rollouts(rollouts)
    assert (batch_k.seq_len, batch_k.batch_size) == (S, B) and batch_k.old_log_probs is not None
    for _ in range(3):                               # eager, capture, replay
        kl.train(batch_k)
        default.train(batch_d)
    times = {"kl": [], "default": []}
    for _ in range(args.steps):
        for key, opt, b in (("default", default, batch_d), ("kl", kl, batch_k)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            opt.train(b)
            times[key].append(1e3 * (time.perf_counter() - t0))
    result["c2_step_ms"] = {k: _stats(v) for k, v in times.items()}
    result["c2_step_ms"]["kl_over_default_median"] = \
        result["c2_step_ms"]["kl"]["median"] / result["c2_step_ms"]["default"]["median"]
    assert kl.last_ppo_stats["kl_skipped"] == 0.0
    kl.close()
    default.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
