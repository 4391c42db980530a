"""Two-rank dual-clip PPO (TEST INFRASTRUCTURE for ``tests/test_gpu_dual_clip.py``): both ranks run the product's
DotaOptimizer with the same c on their own batches through ``run_iteration``, over gloo with both ranks on one GPU (the
step launch by launch: a gloo collective cannot be captured).  The cap acts on each rank's loss before the one gradient
all-reduce, so the replicas stay identical; the parent checks the weights, the step counters and the reported values."""
import datetime
import os
import pickle
import tempfile

import torch

S, H, CELL, WORLD = 16, 128, "lstm", 2
EPOCHS, LR, C = 3, 3e-3, 1.2
LENGTHS = {0: (40, 23, 57, 31), 1: (50, 17, 33, 64)}


def dual_clip_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from dotaclient_b200.optimizer import DotaOptimizer, MessageQueue
    from dotaclient_b200.synthetic import make_rollout
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    host = "dualclipmulti%d" % rank
    opt = DotaOptimizer(rmq_host=host, rmq_port=rank, epochs=EPOCHS, min_seq_per_epoch=4, seq_len=S, learning_rate=LR,
                        checkpoint=False, pretrained_model=None, mq_prefetch_count=1, log_dir=tempfile.mkdtemp(),
                        entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H, cell=CELL, mask_padding=True,
                        dual_clip=C)
    opt.use_cuda_graph = False
    actor = MessageQueue(host=host, port=rank, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for i, L in enumerate(LENGTHS[rank]):
        actor.publish_experience(pickle.dumps(make_rollout(L, 700 + 10 * rank + i, game_id=i, weight_version=1)))
    fraction, coef = [], []
    for it in (1, 2):
        m = opt.run_iteration(it)
        fraction.append(float(m["ppo/dual_clip_fraction"]))
        coef.append(float(m["dual_clip/coef"]))
    torch.save({"fraction": fraction, "coef": coef, "param": opt.flat.param.cpu(), "steps": opt.adam_steps.cpu()},
               os.path.join(out_dir, "dual_clip_rank%d.pt" % rank))
    opt.close()
    dist.barrier()
    dist.destroy_process_group()


def run(out_dir):
    """Spawns the two ranks; returns their records."""
    import torch.multiprocessing as mp
    import multi_rank
    mp.spawn(dual_clip_worker, args=(WORLD, multi_rank._free_port(), str(out_dir)), nprocs=WORLD, join=True)
    return [torch.load(os.path.join(str(out_dir), "dual_clip_rank%d.pt" % r)) for r in range(WORLD)]
