"""2-GPU tests of the data-parallel step: NCCL all-reduce of the flat gradient buffer + fused finish, against
the N-rank oracle (``oracle/ref_distributed.py``, itself pinned to the reference's ``distributed.py`` under gloo), and
data-parallel resume from a checkpoint (Adam state restored on the master must reach every rank)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import multi_rank  # noqa: E402

pytestmark = pytest.mark.gpu
needs2 = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")


@needs2
def test_two_rank_step_matches_nrank_oracle(tmp_path):
    multi_rank.run_two_rank_step_check(tmp_path)


@needs2
def test_two_rank_resume_broadcasts_adam_state(tmp_path):
    """ADVICE r1: only the master restores ``adam_*.state``; without a broadcast the other ranks would restart Adam from
    zero moments / step 0 and the replicas would diverge after the first resumed step."""
    import torch.multiprocessing as mp
    mp.spawn(multi_rank.resume_worker, args=(multi_rank.WORLD, multi_rank._free_port(), str(tmp_path)), nprocs=multi_rank.WORLD, join=True)
    a, b = (torch.load(tmp_path / ("resume%d.pt" % r)) for r in range(2))
    assert a["iteration_start"] == b["iteration_start"] == 6
    assert torch.equal(a["steps"], b["steps"]) and int(a["steps"].max()) == 3          # 2 steps restored + 1 resumed
    assert torch.equal(a["exp_avg"], b["exp_avg"]) and float(a["exp_avg"].abs().max()) > 0
    assert torch.equal(a["param"], b["param"])                                         # replicas still bit-identical
