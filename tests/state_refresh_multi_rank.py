"""Two-rank state refresh (TEST INFRASTRUCTURE for ``tests/test_gpu_state_refresh.py``): every rank runs the product's
DotaOptimizer with ``recompute_states=True`` and ``recompute_advantages=True`` and two minibatches through
``run_iteration`` on its own rollouts, so the ranks hold batches of different sizes and refresh them on their own; the
gradient all-reduce is the only collective of a step.  The parent checks that both ranks ran every refresh, reported the
drift, and keep bit-identical weights and Adam step counts.

``backend='nccl'``: one GPU per rank, the step replayed from its captured graph.  ``'gloo'``: both ranks on one GPU (NCCL
refuses two ranks on one device), the step launch by launch (a gloo collective cannot be captured)."""
import datetime
import os
import pickle
import tempfile

import torch

S, H, CELL, WORLD, EPOCHS, ITERATIONS = 8, 128, "lstm", 2, 3, 2
# the rollouts published per iteration; with min_seq_per_epoch = 2 an iteration pulls one of them: rank 0 trains on batches
# of 3 and then 2 sequences, rank 1 on batches of 4 and then 3.  No chunk holds a single real step: a minibatch of that
# one sequence would normalise its advantages over one token
LENGTHS = {0: (20, 13), 1: (30, 19)}


def state_refresh_worker(rank, world, port, out_dir, backend):
    import torch.distributed as dist
    from dotaclient_b200.optimizer import DotaOptimizer, MessageQueue
    from dotaclient_b200.synthetic import make_rollout
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    host = "staterefreshmulti%d" % rank
    opt = DotaOptimizer(rmq_host=host, rmq_port=rank, epochs=EPOCHS, min_seq_per_epoch=2, seq_len=S, learning_rate=5e-4,
                        checkpoint=False, pretrained_model=None, mq_prefetch_count=1, log_dir=tempfile.mkdtemp(),
                        entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H, cell=CELL, mask_padding=True,
                        num_minibatches=2, recompute_advantages=True, recompute_states=True)
    if backend == "gloo":
        opt.use_cuda_graph = False
    refreshes = []
    real = opt._refresh_states

    def counted(batch):
        refreshes.append(batch.batch_size)
        real(batch)
    opt._refresh_states = counted
    actor = MessageQueue(host=host, port=rank, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for it in range(ITERATIONS):
        for i, L in enumerate(LENGTHS[rank]):
            actor.publish_experience(pickle.dumps(make_rollout(L, 900 + 100 * it + 10 * rank + i, game_id=i,
                                                               weight_version=1)))
    sizes, drifts = [], []
    for it in range(1, ITERATIONS + 1):
        metrics = opt.run_iteration(it)
        sizes.append(opt._last_iteration_shape[1])
        drifts.append(metrics["refresh/state_drift"])
    torch.save({"param": opt.flat.param.cpu(), "exp_avg": opt.exp_avg.cpu(), "steps": opt.adam_steps.cpu(),
                "sizes": sizes, "refreshes": refreshes, "drifts": drifts},
               os.path.join(out_dir, "state_refresh_rank%d.pt" % rank))
    opt.close()
    dist.barrier()
    dist.destroy_process_group()


def run(out_dir, backend):
    """Spawns the two ranks; returns their records."""
    import torch.multiprocessing as mp
    import multi_rank
    mp.spawn(state_refresh_worker, args=(WORLD, multi_rank._free_port(), str(out_dir), backend), nprocs=WORLD, join=True)
    return [torch.load(os.path.join(str(out_dir), "state_refresh_rank%d.pt" % r)) for r in range(WORLD)]
