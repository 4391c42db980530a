"""Two-rank behaviour cloning (TEST INFRASTRUCTURE for ``tests/test_gpu_bc.py``): both ranks run the product's
DotaOptimizer with ``objective='bc'`` on their own demonstrations through ``run_iteration``, over gloo with both ranks on
one GPU (the step launch by launch: a gloo collective cannot be captured).  The NLL's gradient goes through the same one
all-reduce as the PPO loss's, so the replicas stay identical; the parent checks the weights and the step counters."""
import datetime
import os
import pickle
import tempfile

import torch

S, H, CELL, WORLD = 16, 128, "lstm", 2
EPOCHS, LR = 2, 1e-3
LENGTHS = {0: (40, 23, 57, 31), 1: (50, 17, 33, 64)}


def bc_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from dotaclient_b200.optimizer import DotaOptimizer, MessageQueue
    from dotaclient_b200.synthetic import make_rollout
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    host = "bcmulti%d" % rank
    opt = DotaOptimizer(rmq_host=host, rmq_port=rank, epochs=EPOCHS, min_seq_per_epoch=4, seq_len=S, learning_rate=LR,
                        checkpoint=False, pretrained_model=None, mq_prefetch_count=1, log_dir=tempfile.mkdtemp(),
                        entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H, cell=CELL, mask_padding=True,
                        objective="bc")
    opt.use_cuda_graph = False
    actor = MessageQueue(host=host, port=rank, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for it in range(2):
        for i, L in enumerate(LENGTHS[rank]):
            actor.publish_experience(pickle.dumps(make_rollout(L, 700 + 100 * rank + 10 * it + i, game_id=i,
                                                               weight_version=1)))
    nll, acc = [], []
    for it in (1, 2):
        m = opt.run_iteration(it)
        assert "loss/policy" not in m and "ppo/approx_kl" not in m and "ppo/clip_fraction" not in m
        nll.append(float(m["loss/bc"]))
        acc.append(float(m["bc/accuracy"]))
    torch.save({"nll": nll, "acc": acc, "param": opt.flat.param.cpu(), "steps": opt.adam_steps.cpu()},
               os.path.join(out_dir, "bc_rank%d.pt" % rank))
    opt.close()
    dist.barrier()
    dist.destroy_process_group()


def run(out_dir):
    """Spawns the two ranks; returns their records."""
    import torch.multiprocessing as mp
    import multi_rank
    mp.spawn(bc_worker, args=(WORLD, multi_rank._free_port(), str(out_dir)), nprocs=WORLD, join=True)
    return [torch.load(os.path.join(str(out_dir), "bc_rank%d.pt" % r)) for r in range(WORLD)]
