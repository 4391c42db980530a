"""Per-kernel breakdown of one DotaOptimizer.train() step with torch.profiler (CUDA activities).

    python tools/profile_step.py [--config c2] [--steps 3]   ->  gpurun_out/step_profile_<config>.txt
Not a benchmark (profiler overhead); used to decide what to optimise next.
"""
import argparse
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from dotaclient_b200.optimizer import DotaOptimizer, ExperienceBatch  # noqa: E402
from dotaclient_b200.synthetic import make_rollout, rollout_seed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c2")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=None)
    a = ap.parse_args()
    cfg = dict(bench.CONFIGS[a.config])
    if a.batch:
        cfg["batch"] = a.batch
    B, S, H, cell = cfg["batch"], cfg["seq_len"], cfg["hidden"], cfg["cell"]
    torch.cuda.set_device(0)
    opt = DotaOptimizer(rmq_host="prof", rmq_port=0, epochs=1, min_seq_per_epoch=B, seq_len=S, learning_rate=5e-5,
                        checkpoint=False, pretrained_model=None, mq_prefetch_count=1, log_dir=tempfile.mkdtemp(),
                        entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H, cell=cell)
    seqs = []
    with torch.no_grad():
        for i in range(B):
            seqs.extend(opt.experiences_from_rollout(make_rollout(S, rollout_seed(0, i))))
    batch = ExperienceBatch.from_sequences(seqs, opt.device)
    del seqs
    for _ in range(3):
        opt.train(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            opt.train(batch)
        torch.cuda.synchronize()
    table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=45, max_name_column_width=70)
    out = os.path.join(ROOT, "gpurun_out", "step_profile_%s.txt" % a.config)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        f.write("config %s: B=%d S=%d H=%d %s, %d profiled steps\n" % (a.config, B, S, H, cell, a.steps))
        f.write(table)
    print(table)


if __name__ == "__main__":
    main()
