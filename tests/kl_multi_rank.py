"""Two-rank KL control (TEST INFRASTRUCTURE for ``tests/test_gpu_kl_multi.py``): every rank runs the product's
DotaOptimizer on its own batches with ``kl_coef``, ``kl_target`` and ``kl_stop`` through ``run_iteration``.  The loss writes
the rank's (sum_t KL_t, T_a) behind the has-grad flags, the step's one gradient all-reduce sums them, and the finish decides
the skip; the parent checks that both ranks reached the same decisions, the same coefficient and the same weights.

``backend='nccl'``: one GPU per rank, the step replayed from its captured graph with the all-reduce inside.  ``'gloo'``: both
ranks on one GPU (NCCL refuses two ranks on one device), the step launch by launch (a gloo collective cannot be captured)."""
import datetime
import os
import pickle
import tempfile

import torch

S, H, CELL, WORLD = 16, 128, "lstm", 2
EPOCHS, KL_COEF, KL_TARGET, KL_STOP, LR = 4, 0.3, 1e-6, 1e-4, 1e-2
# different rollouts on the two ranks: different batches, different rank-local KLs
LENGTHS = {0: (40, 23, 57, 31), 1: (50, 17, 33, 64)}


def kl_worker(rank, world, port, out_dir, backend):
    import torch.distributed as dist
    from dotaclient_b200.optimizer import DotaOptimizer, MessageQueue
    from dotaclient_b200.synthetic import make_rollout
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    host = "klmulti%d" % rank
    opt = DotaOptimizer(rmq_host=host, rmq_port=rank, epochs=EPOCHS, min_seq_per_epoch=4, seq_len=S, learning_rate=LR,
                        checkpoint=False, pretrained_model=None, mq_prefetch_count=1, log_dir=tempfile.mkdtemp(),
                        entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H, cell=CELL, mask_padding=True,
                        kl_coef=KL_COEF, kl_target=KL_TARGET, kl_stop=KL_STOP)
    if backend == "gloo":
        opt.use_cuda_graph = False
    actor = MessageQueue(host=host, port=rank, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for i, L in enumerate(LENGTHS[rank]):
        actor.publish_experience(pickle.dumps(make_rollout(L, 700 + 10 * rank + i, game_id=i, weight_version=1)))
    recs = []
    for it in (1, 2):
        m = opt.run_iteration(it)
        recs.append({k: float(m[k]) for k in ("kl/coef", "kl/all_ranks", "kl/updates_run", "kl/updates_skipped", "ppo/kl")})
        recs[-1]["coef_after"] = opt.kl_coef
        recs[-1]["batch_size"] = opt._last_iteration_shape[1]
    torch.save({"recs": recs, "param": opt.flat.param.cpu(), "steps": opt.adam_steps.cpu()},
               os.path.join(out_dir, "kl_rank%d.pt" % rank))
    opt.close()                                     # graphs with NCCL work die before the process group
    dist.barrier()
    dist.destroy_process_group()


def run(out_dir, backend):
    """Spawns the two ranks; returns their records."""
    import torch.multiprocessing as mp
    import multi_rank
    mp.spawn(kl_worker, args=(WORLD, multi_rank._free_port(), str(out_dir), backend), nprocs=WORLD, join=True)
    return [torch.load(os.path.join(str(out_dir), "kl_rank%d.pt" % r)) for r in range(WORLD)]
