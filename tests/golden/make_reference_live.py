"""Records tests/golden/reference_live.npz from the UNMODIFIED reference (TimZaman/dotaclient @ 8615b90).

Run where the reference tree is importable (``oracle/reference_shim.py``, ``DOTACLIENT_REFERENCE``):

    python tests/golden/make_reference_live.py

Two recordings, checked bit for bit by tests/test_oracle.py against the CPU oracle:
  * ``live_*``: one reference optimizer (seq_len 8), a ragged 29-step rollout (seed 5), its prepared sequences and
    two train() epochs;
  * ``gloo_*``: two gloo ranks running the reference's distributed.py wrapper on rollouts 300 and 301, two train() calls.
A state_dict is stored as float64 per-parameter sums plus a fixed sample of 64 values per parameter (the file stays small).
"""
import copy
import os
import socket
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import reference_shim  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_live.npz")
SAMPLE = 64


def sample_index(n):
    return np.sort(np.random.default_rng(0).choice(n, min(n, SAMPLE), replace=False))


def state_summary(sd, prefix, rec):
    rec[prefix + "param_sums"] = np.array([float(v.double().sum()) for v in sd.values()])
    for i, v in enumerate(sd.values()):
        a = v.detach().reshape(-1).numpy()
        rec["%sparam_sample_%02d" % (prefix, i)] = a[sample_index(a.size)]


def live(rec):
    torch.set_num_threads(1)
    ref = reference_shim.make_reference_optimizer(seq_len=8)
    with torch.no_grad():
        xr = ref.experiences_from_rollout(copy.deepcopy(make_rollout(29, 5)))
    rec["live_n_seq"] = np.array(len(xr))
    for i, x in enumerate(xr):
        rec["live_adv_%d" % i] = x.advantages.numpy()
        rec["live_ret_%d" % i] = x.returns.numpy()
        rec["live_hidden_%d" % i] = x.hidden.numpy()
    for ep in range(2):
        l, e, g = ref.train(xr)
        rec["live_loss_keys_%d" % ep] = np.array(list(l))
        rec["live_loss_%d" % ep] = np.array([l[k].detach().numpy() for k in l])
        rec["live_ent_keys_%d" % ep] = np.array(list(e))
        rec["live_ent_%d" % ep] = np.array([e[k].detach().numpy() for k in e])
        rec["live_gnorm_%d" % ep] = np.array([g["unclipped"].detach().numpy(), g["clipped"].detach().numpy()])
    state_summary(ref.policy_base.state_dict(), "live_", rec)


def gloo_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    O, P, D = reference_shim.load()
    opt = reference_shim.make_reference_optimizer(seq_len=8)
    with torch.no_grad():
        xs = opt.experiences_from_rollout(make_rollout(24, 300 + rank))
    opt.policy = D.DistributedDataParallelSparseParamCPU(opt.policy_base)
    opt.optimizer = torch.optim.Adam(opt.policy.parameters(), lr=5e-5)
    recs = []
    for _ in range(2):
        l, e, g = opt.train(xs)
        recs.append([float(l[k]) for k in ("loss", "policy_loss", "entropy_loss", "value_loss")] + [float(g["unclipped"]), float(g["clipped"])])
    torch.save({"recs": recs, "sd": opt.policy_base.state_dict()}, os.path.join(out_dir, "ref_rank%d.pt" % rank))
    dist.destroy_process_group()


def gloo(rec):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(gloo_worker, args=(2, port, d), nprocs=2, join=True)
        for r in range(2):
            got = torch.load(os.path.join(d, "ref_rank%d.pt" % r))
            rec["gloo_recs_%d" % r] = np.array(got["recs"], dtype=np.float64)
            state_summary(got["sd"], "gloo_%d_" % r, rec)


if __name__ == "__main__":
    assert reference_shim.available(), "reference tree not present"
    rec = {}
    live(rec)
    gloo(rec)
    np.savez_compressed(OUT, **rec)
    print(OUT, os.path.getsize(OUT))
