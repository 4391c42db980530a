"""Cost of kickstarting (``teacher_model``) on the device, at C2 (LSTM-128 student, seq_len 512, 256 sequences = 131,072
tokens) with the reference's GRU-256 as the teacher.

1. The fused loss kernel alone at C2's token count, per-head ratio with a valid mask: ``dc_ppo_loss_fwd_bwd_masked`` (no
   rows), ``_kl`` (the KL penalty's rows), ``_teacher`` without old rows (the teacher's rows) and ``_teacher`` with both,
   on the same preallocated inputs, each call timed alone between two CUDA events, the four alternated call by call;
   median, min and max of ``--calls`` calls each.
2. Experience prep of the C2 rollouts (``batch_from_rollouts``) by the same student with and without the teacher,
   alternated, each timed on the host up to a device synchronise.
3. The replayed C2 step of the optimizer with the teacher at lambda > 0 against lambda = 0 in the same run (the batch carries
   the teacher's rows both times, so the same graph replays), alternated step by step.

Prints one JSON line with the card and its power limit.

    python tools/teacher_bench.py [--calls 200] [--steps 30] [--preps 5]
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
from dotaclient_b200.policy import Policy  # noqa: E402
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
    return DotaOptimizer(rmq_host="teacher_bench", rmq_port=int(time.time() * 1e6) % 100000, epochs=1,
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
    old = torch.randn(N, 5, generator=g, device=d) - 2.0
    adv, ret, value, old_value = (torch.randn(N, generator=g, device=d) for _ in range(4))
    valid = ops._u8(torch.rand(N, generator=g, device=d) < 0.9)
    dlogits = [torch.empty_like(t) for t in logits]
    dvalue = torch.empty_like(value)
    out = torch.empty(_lib.LOSS_SLOTS, device=d)
    stats = torch.empty(_lib.PPO_STATS_SLOTS, device=d)
    t_stats = torch.empty(_lib.TEACHER_STATS_SLOTS, device=d)
    n_act = torch.empty(5, dtype=torch.int32, device=d)
    ws = torch.empty(_lib.PPO_WORKSPACE_BYTES, dtype=torch.uint8, device=d)
    hp = ops.hparam_block(d, e_clip=0.1, entropy_coef=5e-4, vf_coef=0.5, kl_coef=0.2)
    lam = torch.tensor([1.0], dtype=torch.float64, device=d)
    rows = ops.selected_logp_rows(logits, masks, actions)[1]
    t_rows = ops.selected_logp_rows([l + torch.randn_like(l) for l in logits], masks, actions)[1]
    kl_out = torch.empty(2, device=d)
    u8 = [ops._u8(t) for t in masks], [ops._u8(t) for t in actions]
    lib, stream = _lib.load(), _lib.stream_ptr()
    ld = (_lib._c.c_int64 * 5)(*ops.HEAD_SIZES)
    lp5, m5, a5, d5 = _lib.ptr5(logits), _lib.ptr5(u8[0]), _lib.ptr5(u8[1]), _lib.ptr5(dlogits)
    head = (lp5, ld, m5, a5, old.data_ptr(), adv.data_ptr(), ret.data_ptr(), value.data_ptr(), 1, old_value.data_ptr(),
            valid.data_ptr())
    tail = (N, hp.data_ptr(), d5, ld, dvalue.data_ptr(), 1, out.data_ptr(), stats.data_ptr(), n_act.data_ptr(),
            ws.data_ptr(), stream)

    def kl():
        return lib.dc_ppo_loss_fwd_bwd_kl(lp5, ld, m5, a5, old.data_ptr(), rows.data_ptr(), adv.data_ptr(), ret.data_ptr(),
                                          value.data_ptr(), 1, old_value.data_ptr(), valid.data_ptr(), N, hp.data_ptr(), 0,
                                          d5, ld, dvalue.data_ptr(), 1, out.data_ptr(), stats.data_ptr(),
                                          kl_out.data_ptr(), n_act.data_ptr(), ws.data_ptr(), stream)

    def teacher(with_kl):
        return lib.dc_ppo_loss_fwd_bwd_teacher(
            lp5, ld, m5, a5, old.data_ptr(), rows.data_ptr() if with_kl else None, t_rows.data_ptr(), adv.data_ptr(),
            ret.data_ptr(), value.data_ptr(), 1, old_value.data_ptr(), valid.data_ptr(), N, hp.data_ptr(), lam.data_ptr(), 0,
            d5, ld, dvalue.data_ptr(), 1, out.data_ptr(), stats.data_ptr(), kl_out.data_ptr() if with_kl else None,
            t_stats.data_ptr(), n_act.data_ptr(), ws.data_ptr(), stream)
    fns = {"masked": lambda: lib.dc_ppo_loss_fwd_bwd_masked(*head, *tail), "kl": kl,
           "teacher": lambda: teacher(False), "kl_teacher": lambda: teacher(True)}
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
    for k in ("kl", "teacher", "kl_teacher"):
        res[k + "_over_masked_median"] = res[k]["median"] / res["masked"]["median"]
    # algorithmic bytes of the loss pass: 686 per token + 1 for valid + 4 for the old value, + 260 per row set
    r = 4 * _lib.KL_ROW_FLOATS
    res["loss_pass_bytes_per_token"] = {"masked": 691, "kl": 691 + r, "teacher": 691 + r, "kl_teacher": 691 + 2 * r}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=200, help="timed loss-kernel calls per entry point (median; >= 200)")
    ap.add_argument("--steps", type=int, default=30, help="timed C2 steps per coefficient")
    ap.add_argument("--preps", type=int, default=5, help="timed experience preps per optimizer")
    args = ap.parse_args()
    if args.calls < 200:
        ap.error("--calls must be >= 200")
    if not torch.cuda.is_available():
        raise SystemExit("teacher_bench needs a CUDA device")
    pool = [make_rollout(2 * S, 40_000 + i) for i in range(8)]
    rollouts = [pool[i % len(pool)] for i in range(B // 2)]          # two whole sequences each: B sequences
    result = {"device": torch.cuda.get_device_name(), "power_limit": _power_limit(), "calls": args.calls,
              "config": "C2: LSTM-128 student, seq_len 512, 256 sequences; teacher GRU-256 (reference init)"}
    result["loss_kernel_us"] = _kernel_rows(args.calls)

    tdir = tempfile.mkdtemp()
    path = os.path.join(tdir, "teacher_gru256.pt")
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(7)
        torch.save(Policy().state_dict(), path)
    teach, plain = _optimizer(teacher_model=path), _optimizer()
    times = {"with_teacher": [], "without": []}
    for rep in range(args.preps + 1):               # the first round warms every shape up
        for key, opt in (("without", plain), ("with_teacher", teach)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            batch = opt.batch_from_rollouts(rollouts)
            torch.cuda.synchronize()
            if rep:
                times[key].append(1e3 * (time.perf_counter() - t0))
    assert batch.teacher_log_probs is not None and (batch.seq_len, batch.batch_size) == (S, B)
    result["c2_prep_ms"] = {k: _stats(v) for k, v in times.items()}
    result["c2_prep_ms"]["added_median"] = \
        result["c2_prep_ms"]["with_teacher"]["median"] - result["c2_prep_ms"]["without"]["median"]
    plain.close()
    del plain

    for _ in range(3):                               # eager, capture, replay
        teach.train(batch)
    times = {"lambda_1": [], "lambda_0": []}
    for _ in range(args.steps):
        for key, lam in (("lambda_0", 0.0), ("lambda_1", 1.0)):
            teach.teacher_coef = lam
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            teach.train(batch)
            times[key].append(1e3 * (time.perf_counter() - t0))
    assert any(isinstance(v, tuple) for v in teach._graphs.values())
    result["c2_step_ms"] = {k: _stats(v) for k, v in times.items()}
    result["c2_step_ms"]["lambda_1_over_lambda_0_median"] = \
        result["c2_step_ms"]["lambda_1"]["median"] / result["c2_step_ms"]["lambda_0"]["median"]
    teach.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
