"""The C2 training step (LSTM-128, 256 sequences x 512 steps = 131,072 tokens, replayed from its CUDA graph) at a forced
share of tokens that use the target-unit head.

The batch is bench.py's (synthetic rollouts, about 25 % of the steps choose to attack).  For each share f the target_unit
mask and action rows are rewritten on the device: a seeded share f of the tokens gets a mask row (units 1..39 valid) and
an action in it, the other tokens get empty rows.  The step's graph is captured once for the batch shape and replayed for
every share (the rows are copied into its static inputs), each share timed over --steps steps on the host around
``train()``, which ends in the step's host sync.  The shares are run in turn, --rounds times; the median, min and max step
time per share are reported.  Also prints the per-call CUDA-event times of the target-unit branch from one launch-by-launch
step per share, and the per-call times of the branch's GEMMs on all 131,072 tokens (the dense branch's calls: q, d_att,
attention forward / data gradient / weight gradient, the head's share att^T s of dW_g), each call timed alone between two
CUDA events, median of --calls.  Works on any tree that has ``DotaOptimizer``: run it from another checkout to compare.

Prints one JSON line with the card and its power limit.

    python tools/target_unit_bench.py [--steps 20] [--rounds 3] [--shares 0.25,0.5,1.0]
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
from dotaclient_b200.synthetic import make_rollout, rollout_seed  # noqa: E402

S, B, H = 512, 256, 128
BRANCH = ("target_rows", "rows_zero", "target_unit_fwd", "target_unit_bwd")


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _force_share(batch, share, seed=0):
    mask, action = batch.masks['target_unit'], batch.actions['target_unit']
    g = torch.Generator().manual_seed(seed)
    act = (torch.rand(mask.shape[:-1], generator=g) < share).to(mask.device)
    pick = torch.randint(1, 40, mask.shape[:-1], generator=g).to(mask.device)
    mask.zero_()
    action.zero_()
    mask[..., 1:] = act.unsqueeze(-1)
    action.scatter_(-1, pick.unsqueeze(-1), act.unsqueeze(-1))


def _gemm_calls(n_calls):
    """ms per call (median) of the dense target-unit branch's GEMMs at C2: [N, 128] x [896, 128]^T (q), [N, 896] x [128, 896]^T
    (d_att), [N, H] x [128, H]^T + b (attention), [N, 128] x [H, 128]^T (its data gradient), 128 x H and 128 x 896 weight
    gradients over N tokens (attention, the head's att^T s)."""
    d = torch.device("cuda")
    g = torch.Generator(device=d).manual_seed(0)
    N = S * B
    y, att = torch.randn(N, H, generator=g, device=d), torch.randn(N, 128, generator=g, device=d)
    s, d_att = torch.randn(N, 896, generator=g, device=d), torch.randn(N, 128, generator=g, device=d)
    bm, w, b = torch.randn(128, 896, generator=g, device=d), torch.randn(128, H, generator=g, device=d), torch.randn(128, device=d)
    bm_t, w_t = bm.t().contiguous(), w.t().contiguous()
    calls = {
        "q": lambda: ops.gemm_tf32x3(att, bm_t),
        "d_att": lambda: ops.gemm_tf32x3(s, bm),
        "attention_fwd": lambda: ops.gemm_tf32x3(y, w, b),
        "attention_dgrad": lambda: ops.gemm_tf32x3(d_att, w_t),
        "attention_wgrad": lambda: ops.gemm_wgrad_tf32x3(d_att, y),
        "head_wgrad": lambda: ops.gemm_wgrad_tf32x3(att, s, want_bias=False),
    }
    out = {}
    for name, fn in calls.items():
        for _ in range(3):
            fn()
        ts = []
        for _ in range(n_calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        out[name] = round(float(np.median(ts)), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shares", default="0.25,0.5,1.0")
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    shares = [float(s) for s in args.shares.split(",")]
    opt = DotaOptimizer(rmq_host="target_unit_bench", rmq_port=0, epochs=1, min_seq_per_epoch=B, seq_len=S,
                        learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                        log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H, cell="lstm")
    with torch.no_grad():
        base = opt.batch_from_rollouts([make_rollout(S, rollout_seed(0, i)) for i in range(B)])
    natural = float((base.masks['target_unit'] | base.actions['target_unit']).any(-1).float().mean())
    batches = {}
    for f in shares:
        b = base.map(lambda t: t.clone())
        _force_share(b, f)
        batches[f] = b
    for f in shares:                                  # warm-up: the first calls run launch by launch, then the graph is captured
        for _ in range(3):
            opt.train(batches[f])
    times = {f: [] for f in shares}
    for _ in range(args.rounds):
        for f in shares:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                opt.train(batches[f])
            times[f].append(1e3 * (time.perf_counter() - t0) / args.steps)
    branch = {}
    for f in shares:                                  # one launch-by-launch step with CUDA events around every call
        ops.PROFILE.reset(enabled=True)
        opt.train(batches[f])
        ops.PROFILE.reset(enabled=True)
        opt.train(batches[f])
        summ = ops.PROFILE.summary(1)
        branch[str(f)] = {k: round(v, 4) for k, v in summ.items() if k in BRANCH}
        ops.PROFILE.reset(enabled=False)
    line = {
        "tool": "target_unit_bench", "gpu": torch.cuda.get_device_name(), "power_limit": _power_limit(),
        "config": "c2 lstm-128 %dx%d" % (B, S), "natural_share": round(natural, 4), "steps": args.steps, "rounds": args.rounds,
        "ms_per_step": {str(f): {"median": float(np.median(v)), "min": min(v), "max": max(v)} for f, v in times.items()},
        "branch_ms_per_step": branch,
        "dense_branch_gemm_ms_per_call": _gemm_calls(args.calls),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
