"""GPU tests of minibatch PPO: ``dc_gather_columns`` bit-exact against ``index_select``, ``train_epochs`` with minibatches
against the same steps on ``index_select`` batches (launch by launch and from CUDA graphs), against the CPU oracle, through
``run_iteration``, and data-parallel across two ranks with different batch sizes."""
import copy
import os
import pickle
import sys
import tempfile
import uuid

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_parity as P  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu


def make_optimizer(tmp_path, hidden_size=128, cell="lstm", seq_len=16, epochs=2, min_seq=8, port=None, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="minibatch", rmq_port=port if port is not None else uuid.uuid4().int % 100000,
                         epochs=epochs, min_seq_per_epoch=min_seq, seq_len=seq_len, learning_rate=5e-5, checkpoint=False,
                         pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=5e-4, vf_coef=0.5,
                         run_local=True, hidden_size=hidden_size, cell=cell, **kw)


def _rollouts_b8(seed=0):
    """Three ragged rollouts giving 3 + 2 + 3 = 8 sequences of 16 steps."""
    return [make_rollout(L, 500 + 10 * seed + i, game_id=i) for i, L in enumerate((40, 23, 48))]


# ------------------------------------------------------------------------------------------------ the kernel
def _check_gather(pairs_src, idx):
    """gather_columns == index_select(1, idx), bitwise, and two runs agree bitwise."""
    from dotaclient_b200 import ops
    idx_dev = torch.as_tensor(np.asarray(idx), dtype=torch.int64, device=P.dev())
    outs = []
    for _ in range(2):
        dsts = [torch.empty((s.shape[0], len(idx)) + tuple(s.shape[2:]), dtype=s.dtype, device=s.device) for s in pairs_src]
        for d in dsts:
            d.view(torch.uint8).fill_(0xA5) if d.dtype != torch.bool else d.fill_(True)
        ops.gather_columns(list(zip(pairs_src, dsts)), idx)
        outs.append(dsts)
    torch.cuda.synchronize()
    for s, a, b in zip(pairs_src, outs[0], outs[1]):
        want = s.index_select(1, idx_dev)
        assert a.dtype == want.dtype and a.shape == want.shape
        assert torch.equal(a.view(torch.uint8), want.contiguous().view(torch.uint8)) if a.dtype != torch.bool else \
            torch.equal(a, want)
        assert torch.equal(a, b)


@pytest.mark.parametrize("H,cell,L", [(256, "gru", 1), (128, "lstm", 2)])
@pytest.mark.parametrize("old_values", [True, False])
def test_gather_real_batches_bit_exact(H, cell, L, old_values, tmp_path):
    opt = make_optimizer(tmp_path, hidden_size=H, cell=cell, num_layers=L)
    batch = opt.batch_from_rollouts(_rollouts_b8(1) + _rollouts_b8(2))
    if not old_values:
        batch.old_values = None
    B = batch.batch_size
    assert B == 16 and batch.h0.shape == (L, B, H) and (batch.c0 is not None) == (cell == "lstm")
    rng = np.random.default_rng(3)
    for idx in (rng.permutation(B)[:5], rng.permutation(B), np.array([3, 3, 0, 15, 3]), np.array([9])):
        got = batch.gather(idx)
        want = batch.map(lambda v: v.index_select(1, torch.as_tensor(idx, device=v.device)))
        names = [k for _, k, _ in got.tensors()]
        assert names == [k for _, k, _ in want.tensors()] == [k for _, k, _ in batch.tensors()]
        assert (got.old_values is None) == (not old_values) and (got.c0 is None) == (cell == "gru")
        for (_, k, a), (_, _, b) in zip(got.tensors(), want.tensors()):
            assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), k
    _check_gather([v for _, _, v in batch.tensors()], rng.permutation(B)[:7])


ROW_BYTES = [1, 3, 4, 9, 12, 20, 40, 48, 240, 768, 1024]


def _synthetic(outer, cols, row_bytes, offset, gen):
    """A [outer, cols, row_bytes] uint8 view starting `offset` bytes into a random buffer (misaligned for offset % 16)."""
    n = outer * cols * row_bytes
    buf = torch.randint(0, 256, (n + offset,), generator=gen, dtype=torch.uint8).to(P.dev())
    return buf[offset:].view(outer, cols, row_bytes)


@pytest.mark.parametrize("offset", [0, 4, 1])
def test_gather_synthetic_descriptors_bit_exact(offset):
    """Every row width through each copy unit (16-byte, 4-byte, byte: offset 0 / 4 / 1), with outer = 1, n_index = 1,
    repeated indices and a full permutation."""
    gen = torch.Generator().manual_seed(offset)
    rng = np.random.default_rng(offset)
    srcs = [_synthetic(outer, 37, rb, offset, gen) for rb in ROW_BYTES for outer in (1, 5)]
    for idx in (np.array([17]), np.array([2, 2, 2, 36, 0, 2]), rng.permutation(37), rng.integers(0, 37, 300)):
        _check_gather(srcs, idx)
    # fp32 / int64 / bool tensors of the batch's shapes, at misaligned destinations as well
    f = torch.randn(16, 37, 5, generator=gen).to(P.dev())
    i64 = torch.randint(-9, 9, (3, 37, 2), generator=gen).to(P.dev())
    bl = (torch.rand(16, 37, 9, generator=gen) < 0.5).to(P.dev())
    _check_gather([f, i64, bl], rng.permutation(37)[:11])


def test_gather_more_than_one_call_of_descriptors():
    from dotaclient_b200 import _lib
    gen = torch.Generator().manual_seed(9)
    n = 2 * _lib.GATHER_MAX_TENSORS + 5
    srcs = [_synthetic(1 + k % 3, 21, ROW_BYTES[k % len(ROW_BYTES)], k % 5, gen) for k in range(n)]
    _check_gather(srcs, np.random.default_rng(1).permutation(21)[:13])


def test_gather_c2_quarter_shape_bit_exact():
    """A large descriptor (the C2 observation shapes at 64 of 256 sequences) through the 16-byte path."""
    gen = torch.Generator().manual_seed(4)
    src = torch.randn(512, 256, 192, generator=gen).to(P.dev())
    _check_gather([src, src[:, :, :3].contiguous()], np.random.default_rng(4).permutation(256)[:64])


# ------------------------------------------------------------------------------------------------ the step
def _record(out, losses, entropies, norms, stats):
    out.append(([float(v) for v in losses.values()], [float(v) for v in entropies.values()],
                [float(v) for v in norms.values()], dict(stats)))


@pytest.mark.parametrize("graphs", [False, True])
def test_train_epochs_equals_steps_on_index_select_batches(graphs, tmp_path):
    """M = 3, B = 8, 2 epochs: train_epochs (gathered minibatches) against a second optimizer from the same seed that runs
    train() on index_select batches with the same indices.  Bit-identical after the 6 steps."""
    from dotaclient_b200.optimizer import minibatch_indices
    a = make_optimizer(tmp_path, num_minibatches=3)
    b = make_optimizer(tmp_path)
    a.use_cuda_graph = b.use_cuda_graph = graphs
    rollouts = _rollouts_b8()
    batch_a = a.batch_from_rollouts(copy.deepcopy(rollouts))
    batch_b = b.batch_from_rollouts(copy.deepcopy(rollouts))
    assert batch_a.batch_size == 8
    rng = copy.deepcopy(a.minibatch_rng)
    la, ea, ga, sa = a.train_epochs(batch_a)
    got = []
    for x in zip(la, ea, ga, sa):
        _record(got, *x)
    want = []
    for _ in range(2):
        for idx in minibatch_indices(8, 3, rng):
            mb = batch_b.map(lambda v: v.index_select(1, torch.as_tensor(idx, device=v.device)))
            _record(want, *b.train(mb), b.last_ppo_stats)
    assert len(got) == len(want) == 6
    for step, (g, w) in enumerate(zip(got, want)):
        assert g[:3] == w[:3], step
        assert g[3].keys() == w[3].keys() and all(g[3][k] == w[3][k] or (g[3][k] != g[3][k] and w[3][k] != w[3][k])
                                                  for k in g[3]), step
    assert torch.equal(a.flat.param, b.flat.param)
    assert torch.equal(a.exp_avg, b.exp_avg) and torch.equal(a.exp_avg_sq, b.exp_avg_sq)
    assert torch.equal(a.adam_steps, b.adam_steps) and int(a.adam_steps.max()) == 6
    captured = [k for k, v in a._graphs.items() if isinstance(v, tuple)]
    if graphs:
        assert sorted(k[1] for k in captured) == [2, 3], a._graphs     # both minibatch shapes captured and replayed
    else:
        assert not captured


def test_train_epochs_vs_oracle(tmp_path):
    """Ragged multi-chunk rollouts at H = 128 LSTM, M = 3, 2 epochs: the oracle trains on the same sequences per step."""
    from dotaclient_b200.optimizer import minibatch_indices
    torch.set_num_threads(4)
    S = 16
    mine = make_optimizer(tmp_path, min_seq=3, num_minibatches=3)
    oracle = P.make_oracle(128, "lstm", S)
    rollouts = P._rollouts(4, S, seed=21)
    batch = mine.batch_from_rollouts(copy.deepcopy(rollouts))
    xs_o = [s for r in rollouts for s in oracle.experiences_from_rollout(copy.deepcopy(r))]
    B = batch.batch_size
    assert B == len(xs_o) and B >= 6
    rng = copy.deepcopy(mine.minibatch_rng)
    lm, em, gm, _ = mine.train_epochs(batch)
    step = 0
    for _ in range(2):
        for idx in minibatch_indices(B, 3, rng):
            lo, eo, go = oracle.train([xs_o[i] for i in idx])
            for k in lo:
                np.testing.assert_allclose(float(lm[step][k]), float(lo[k]), rtol=2e-4, atol=2e-6, err_msg="%s %d" % (k, step))
            for k in eo:
                np.testing.assert_allclose(float(em[step][k]), float(eo[k]), rtol=2e-4, atol=1e-6, err_msg="%s %d" % (k, step))
            np.testing.assert_allclose(float(gm[step]["unclipped"]), float(go["unclipped"]), rtol=2e-3)
            np.testing.assert_allclose(float(gm[step]["clipped"]), float(go["clipped"]), rtol=2e-3)
            step += 1
    assert step == 6
    sd = mine.optimizer.state_dict()["state"]
    want = P._adam_state_by_name(oracle)
    names = [n for n, _ in oracle.policy_base.named_parameters()]
    assert sorted(names[i] for i in sd) == sorted(want)
    for i, st in sd.items():
        w = want[names[i]]
        assert float(st["step"]) == float(w["step"])
        m_scale = float(w["exp_avg"].abs().max())
        v_scale = float(w["exp_avg_sq"].abs().max())
        torch.testing.assert_close(st["exp_avg"], w["exp_avg"], rtol=2e-3, atol=2e-3 * m_scale + 1e-12)
        torch.testing.assert_close(st["exp_avg_sq"], w["exp_avg_sq"], rtol=4e-3, atol=4e-3 * v_scale + 1e-20)
        cos = torch.nn.functional.cosine_similarity(st["exp_avg"].flatten(), w["exp_avg"].flatten(), dim=0)
        assert cos > 0.9999, (names[i], float(cos))


def test_train_epochs_refuses_a_batch_smaller_than_the_minibatch_count(tmp_path):
    opt = make_optimizer(tmp_path, num_minibatches=3)
    batch = opt.batch_from_rollouts([make_rollout(20, 1)])
    assert batch.batch_size == 2
    with pytest.raises(ValueError, match="num_minibatches=3"):
        opt.train_epochs(batch)
    assert int(opt.adam_steps.max()) == 0


# ------------------------------------------------------------------------------------------------ run_iteration
def _run_iteration(tmp_path, port, rollouts, **kw):
    from dotaclient_b200.optimizer import MessageQueue
    opt = make_optimizer(tmp_path, min_seq=6, port=port, **kw)
    actor = MessageQueue(host="minibatch", port=port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for r in rollouts:
        actor.publish_experience(pickle.dumps(r))
    steps = []
    inner = opt.train_epochs

    def recording(batch):
        res = inner(batch)
        steps.append(res)
        return res
    opt.train_epochs = recording
    metrics = opt.run_iteration(1)
    return opt, metrics, steps[0], opt.mq.xp_queue_size


def test_run_iteration_with_minibatches(tmp_path):
    rollouts = [make_rollout(L, 800 + i, game_id=i, weight_version=1, with_canvas=True) for i, L in enumerate((40, 23, 57, 30))]
    base = uuid.uuid4().int % 100000
    m3, met3, (l3, _, _, _), left3 = _run_iteration(tmp_path, base, rollouts, num_minibatches=3)
    m1, met1, _, left1 = _run_iteration(tmp_path, base + 1, rollouts, num_minibatches=1)
    m0, met0, _, left0 = _run_iteration(tmp_path, base + 2, rollouts)
    assert left3 == left1 == left0 == 1                         # 3 + 2 + 4 >= 6 sequences: the same three rollouts pulled
    assert met3["avg_rollout_len"] == met1["avg_rollout_len"]
    assert int(m3.adam_steps.max()) == 2 * 3 and int(m1.adam_steps.max()) == 2
    assert set(met3) == set(met1) == set(met0)
    assert len(l3) == 6
    want = float(torch.stack([torch.as_tensor(s["loss"]) for s in l3]).mean())
    assert float(met3["loss/sum"]) == pytest.approx(want, rel=1e-6, abs=1e-9)
    # the default and an explicit num_minibatches=1 are the same computation
    assert torch.equal(m1.flat.param, m0.flat.param)
    assert torch.equal(m1.exp_avg, m0.exp_avg) and torch.equal(m1.exp_avg_sq, m0.exp_avg_sq)


# ------------------------------------------------------------------------------------------------ two ranks
WORLD, S_DP, H_DP = 2, 8, 128
DP_LENGTHS = {0: (20, 13), 1: (30, 17, 9)}      # rank 0: 3 + 2 = 5 sequences, rank 1: 4 + 3 + 2 = 9


def _dp_rollouts(rank):
    return [make_rollout(L, 600 + 10 * rank + i) for i, L in enumerate(DP_LENGTHS[rank])]


def dp_worker(rank, world, port, out_dir):
    import multi_rank
    dist = multi_rank._init(rank, world, port)
    from dotaclient_b200.optimizer import DotaOptimizer
    opt = DotaOptimizer(rmq_host="mbdp%s" % out_dir, rmq_port=rank, epochs=2, min_seq_per_epoch=2, seq_len=S_DP,
                        learning_rate=5e-5, checkpoint=False, pretrained_model=None, mq_prefetch_count=1,
                        log_dir=tempfile.mkdtemp(), entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=H_DP,
                        cell="lstm", num_minibatches=2)
    batch = opt.batch_from_rollouts(_dp_rollouts(rank))
    losses, entropies, norms, _ = opt.train_epochs(batch)
    recs = [([float(l[k]) for k in ("loss", "policy_loss", "entropy_loss", "value_loss")], float(g["unclipped"]),
             float(g["clipped"])) for l, g in zip(losses, norms)]
    torch.save({"recs": recs, "B": batch.batch_size, "param": opt.flat.param.cpu(),
                "sd": {k: v.cpu() for k, v in opt.policy_base.state_dict().items()}},
               os.path.join(out_dir, "rank%d.pt" % rank))
    opt.close()
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_different_batch_sizes(tmp_path):
    import multi_rank
    import torch.multiprocessing as mp
    from oracle import ref_distributed, ref_optimizer as RO
    from oracle.ref_policy import RefPolicy
    from dotaclient_b200.optimizer import minibatch_indices
    mp.spawn(dp_worker, args=(WORLD, multi_rank._free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    got = [torch.load(os.path.join(str(tmp_path), "rank%d.pt" % r)) for r in range(WORLD)]
    assert got[0]["B"] != got[1]["B"]
    assert len(got[0]["recs"]) == len(got[1]["recs"]) == 4
    assert torch.equal(got[0]["param"], got[1]["param"])
    opts = []
    for _ in range(WORLD):
        torch.manual_seed(7)
        opts.append(RO.RefOptimizer(RefPolicy(H_DP, "lstm"), seq_len=S_DP))
    xs = [[s for r in _dp_rollouts(rank) for s in opts[rank].experiences_from_rollout(r)] for rank in range(WORLD)]
    rngs = [np.random.default_rng(7 + r) for r in range(WORLD)]
    step = 0
    for _ in range(2):
        idxs = [minibatch_indices(len(xs[r]), 2, rngs[r]) for r in range(WORLD)]
        for m in range(2):
            res = ref_distributed.train_ranks(opts, [[xs[r][i] for i in idxs[r][m]] for r in range(WORLD)])
            for r in range(WORLD):
                l, _, g = res[r]
                want = [float(l[k]) for k in ("loss", "policy_loss", "entropy_loss", "value_loss")]
                np.testing.assert_allclose(got[r]["recs"][step][0], want, rtol=2e-4, atol=2e-6)
                np.testing.assert_allclose(got[r]["recs"][step][1], float(g["unclipped"]), rtol=2e-3)
                np.testing.assert_allclose(got[r]["recs"][step][2], float(g["clipped"]), rtol=2e-3)
            step += 1
