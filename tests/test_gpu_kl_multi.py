"""Two ranks with different batches under KL control reach the same skip step and the same adaptive coefficient, and keep
bit-identical weights: the rank-local (sum_t KL_t, T_a) travels in the gradient all-reduce and every decision reads the
all-ranks KL.  With NCCL (one GPU per rank, graph replay; skipped on one GPU) and with gloo (both ranks on one GPU)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kl_multi_rank as KM  # noqa: E402
import kl_oracle as KO  # noqa: E402

pytestmark = pytest.mark.gpu


def _check(got):
    a, b = got
    assert torch.equal(a["param"], b["param"]) and torch.equal(a["steps"], b["steps"])     # replicas bit-identical
    coef = KM.KL_COEF
    skipped = 0
    for ra, rb in zip(a["recs"], b["recs"]):
        for k in ("kl/coef", "kl/all_ranks", "kl/updates_run", "kl/updates_skipped", "coef_after"):
            assert ra[k] == rb[k], (k, ra[k], rb[k])
        assert ra["kl/coef"] == coef
        coef = KO.kl_coef_update(coef, ra["kl/all_ranks"], KM.KL_TARGET)                   # the rule, on the shared KL
        assert ra["coef_after"] == coef
        assert ra["kl/updates_run"] + ra["kl/updates_skipped"] == KM.EPOCHS
        skipped += ra["kl/updates_skipped"]
        assert ra["ppo/kl"] != rb["ppo/kl"]                                                  # the rank-local KLs differ
    assert skipped > 0, "no step was skipped: the test does not reach the early stop"
    assert a["recs"][0]["batch_size"] != b["recs"][0]["batch_size"]                        # different batches
    assert coef == KM.KL_COEF * 4                                                           # doubled twice


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_nccl_same_skip_step_and_beta(tmp_path):
    _check(KM.run(tmp_path, "nccl"))


def test_two_ranks_gloo_one_gpu_same_skip_step_and_beta(tmp_path):
    _check(KM.run(tmp_path, "gloo"))
