"""GPU tests of the iteration driver: in-process broker -> prep -> epochs x train -> checkpoint/publish
(``optimizer.py:436-579,697-723``), checkpoint format compatibility and resume."""
import io
import os
import pickle
import uuid

import numpy as np
import pytest
import torch

from dotaclient_b200.synthetic import make_rollout

pytestmark = pytest.mark.gpu


def _optimizer(tmp_path, port, checkpoint=True, **kw):
    from dotaclient_b200.optimizer import DotaOptimizer
    args = dict(rmq_host="loop", rmq_port=port, epochs=2, min_seq_per_epoch=6, seq_len=8, learning_rate=5e-5,
                checkpoint=checkpoint, pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path),
                entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=128, cell="lstm")
    args.update(kw)
    return DotaOptimizer(**args)


def test_run_iteration_consumes_queue_and_publishes_model(tmp_path):
    from dotaclient_b200.optimizer import MessageQueue
    from oracle.ref_policy import RefPolicy
    port = uuid.uuid4().int % 100000
    opt = _optimizer(tmp_path, port)
    actor = MessageQueue(host="loop", port=port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    body0, hdr0 = actor.latest_model()                 # initial model published before any step (optimizer.py:284)
    assert hdr0 == {"version": 1}
    for i in range(4):
        actor.publish_experience(pickle.dumps(make_rollout(20 + i, 50 + i, weight_version=1, with_canvas=True)))
    before = opt.flat.param.clone()
    metrics = opt.run_iteration(1)
    assert actor.xp_queue_size == 2                    # 2 rollouts x 3 chunks >= min_seq_per_epoch = 6
    for key in (opt.SPEED_KEY, "loss/sum", "loss/policy", "loss/entropy", "loss/value", "entropy", "avg_rollout_len",
                "avg_weight_age", "timing/it", "timing/xp_total", "timing/xp_mq_wait", "timing/optimizer",
                "entropy/enum", "grad_norm/unclipped", "grad_norm/clipped", "reward_per_sec/win", "reward_per_sec/sum"):
        assert key in metrics, key
    assert np.isfinite(float(metrics["loss/sum"])) and float(metrics["avg_rollout_len"]) == 20.5
    assert not torch.equal(before, opt.flat.param)     # two Adam steps happened
    assert int(opt.adam_steps.max()) == 2
    # published model == checkpoint file == torch.save(state_dict) bytes the reference's agents load (agent.py:207-213)
    body, hdr = actor.latest_model()
    assert hdr == {"version": 1}
    with open(tmp_path / "model_000000001.pt", "rb") as f:
        assert f.read() == body
    sd = torch.load(io.BytesIO(body), map_location="cpu")
    ref = RefPolicy(128, "lstm")
    ref.load_state_dict(sd, strict=True)               # same 34 keys / shapes
    for k, v in opt.policy_base.state_dict().items():
        assert torch.equal(v.cpu(), sd[k])


def test_resume_from_latest_checkpoint(tmp_path):
    from dotaclient_b200.optimizer import DotaOptimizer, MessageQueue
    port = uuid.uuid4().int % 100000
    opt = _optimizer(tmp_path, port)
    actor = MessageQueue(host="loop", port=port, prefetch_count=1, use_model_exchange=False)
    actor.connect()
    for i in range(4):
        actor.publish_experience(pickle.dumps(make_rollout(24, 70 + i, with_canvas=True)))
    opt.run_iteration(1)
    opt.run_iteration(2)
    assert DotaOptimizer.iteration_from_model_filename("x/model_000000123.pt") == 123
    assert opt.get_latest_model(str(tmp_path)) == "model_000000002.pt"
    resumed = _optimizer(tmp_path, port + 1)
    assert resumed.iteration_start == 3                # optimizer.py:253
    for (k, a), (_, b) in zip(opt.policy_base.state_dict().items(), resumed.policy_base.state_dict().items()):
        assert torch.equal(a, b), k
    # extension: the Adam moments are checkpointed next to the weights (torch.optim.Adam layout) and restored on resume
    assert os.path.isfile(os.path.join(str(tmp_path), "adam_000000002.state"))
    assert torch.equal(opt.exp_avg, resumed.exp_avg) and torch.equal(opt.exp_avg_sq, resumed.exp_avg_sq)
    assert torch.equal(opt.adam_steps, resumed.adam_steps) and int(resumed.adam_steps.max()) == 4      # 2 iterations x 2 epochs
    stock = torch.optim.Adam([torch.nn.Parameter(p.detach().cpu().clone()) for p in opt.flat.params], lr=opt.learning_rate)
    stock.load_state_dict(resumed.optimizer.state_dict())             # a stock torch optimizer accepts it
    i0 = opt.flat.names.index("affine_pre_rnn.weight")
    lo, hi = opt.flat.starts[i0], opt.flat.ends[i0]
    torch.testing.assert_close(stock.state[stock.param_groups[0]['params'][i0]]['exp_avg'].reshape(-1), opt.exp_avg[lo:hi].cpu(),
                               rtol=0, atol=0)


def test_train_accepts_host_pinned_batch(tmp_path):
    """The e2e path bench.py times: inputs in pinned host memory, H2D inside train()."""
    from dotaclient_b200.optimizer import ExperienceBatch
    opt = _optimizer(tmp_path, uuid.uuid4().int % 100000, checkpoint=False)
    twin = _optimizer(tmp_path, uuid.uuid4().int % 100000, checkpoint=False)
    seqs = opt.experiences_from_rollout(make_rollout(32, 5))
    dev_batch = ExperienceBatch.from_sequences(seqs, opt.device)
    host_batch = dev_batch.pin_memory()
    assert not host_batch.advantages.is_cuda and host_batch.advantages.is_pinned()
    assert host_batch.nbytes() == dev_batch.nbytes() and (host_batch.seq_len, host_batch.batch_size) == (8, 4)
    l1, e1, g1 = opt.train(host_batch)
    l2, e2, g2 = twin.train(dev_batch)
    # same arithmetic; only the order of float64 atomics in the loss / norm reductions may differ
    np.testing.assert_allclose(float(l1["loss"]), float(l2["loss"]), rtol=1e-6)
    np.testing.assert_allclose(float(g1["unclipped"]), float(g2["unclipped"]), rtol=1e-6)
    torch.testing.assert_close(opt.flat.param, twin.flat.param, rtol=0, atol=1e-7)


def test_prefetch_double_buffers_the_upload(tmp_path):
    """DotaOptimizer.prefetch(): the next batch's H2D copy is issued before the current step is launched; two pipelined
    steps give the same parameters as two plain train() calls on device-resident batches."""
    from dotaclient_b200.optimizer import ExperienceBatch
    opt = _optimizer(tmp_path, uuid.uuid4().int % 100000, checkpoint=False)
    twin = _optimizer(tmp_path, uuid.uuid4().int % 100000, checkpoint=False)
    dev = [ExperienceBatch.from_sequences(opt.experiences_from_rollout(make_rollout(32, s)), opt.device) for s in (5, 6)]
    host = [b.pin_memory() for b in dev]
    cur = opt.prefetch(host[0])
    assert cur.advantages.is_cuda and opt.prefetch(cur) is cur          # a device batch passes through
    nxt = opt.prefetch(host[1])                                         # upload of step 2 in flight while step 1 runs
    opt.train(cur)
    l1, _, g1 = opt.train(nxt)
    twin.train(dev[0])
    l2, _, g2 = twin.train(dev[1])
    np.testing.assert_allclose(float(l1["loss"]), float(l2["loss"]), rtol=1e-6)
    np.testing.assert_allclose(float(g1["unclipped"]), float(g2["unclipped"]), rtol=1e-6)
    torch.testing.assert_close(opt.flat.param, twin.flat.param, rtol=0, atol=1e-7)


def test_pending_upload_leaves_other_batches_on_the_graph_path(tmp_path):
    """A batch uploaded from pinned memory and not trained on yet keeps its ready-events to itself: a different
    device-resident batch trained meanwhile is captured and replayed from a CUDA graph, and the uploaded batch, trained
    afterwards, gives the same step as the same batch trained from device memory."""
    from dotaclient_b200.optimizer import ExperienceBatch
    opt = _optimizer(tmp_path, uuid.uuid4().int % 100000, checkpoint=False)
    twin = _optimizer(tmp_path, uuid.uuid4().int % 100000, checkpoint=False)
    a, p_dev = [ExperienceBatch.from_sequences(opt.experiences_from_rollout(make_rollout(32, s)), opt.device) for s in (5, 6)]
    p = p_dev.pin_memory().to(opt.device)                                # copies in flight on the side stream, not prefetch()
    for _ in range(3):
        opt.train(a)
        twin.train(a)
    assert isinstance(opt._graphs.get((8, 4, True)), tuple), "the step was never captured"
    l1, _, g1 = opt.train(p)
    l2, _, g2 = twin.train(p_dev)
    np.testing.assert_allclose(float(l1["loss"]), float(l2["loss"]), rtol=1e-6)
    np.testing.assert_allclose(float(g1["unclipped"]), float(g2["unclipped"]), rtol=1e-6)
    torch.testing.assert_close(opt.flat.param, twin.flat.param, rtol=0, atol=1e-7)


@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_batched_experience_prep_equals_per_rollout_prep(tmp_path, cell):
    """experiences_from_rollouts (one batched pass over ragged rollouts) == experiences_from_rollout per rollout
    (optimizer.py:328-430): same chunk count, carried hidden states, old log-probs, values, GAE advantages/returns."""
    from dotaclient_b200.optimizer import DotaOptimizer
    opt = DotaOptimizer(rmq_host="loop", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=4, seq_len=8,
                        learning_rate=1e-4, checkpoint=False, pretrained_model=None, mq_prefetch_count=1, log_dir=str(tmp_path),
                        entropy_coef=5e-4, vf_coef=0.5, run_local=True, hidden_size=128, cell=cell)
    datas = [make_rollout(L, 300 + i) for i, L in enumerate((19, 8, 33, 5))]
    with torch.no_grad():
        single = [opt.experiences_from_rollout(d) for d in datas]
        batched = opt.experiences_from_rollouts(datas)
    assert [len(b) for b in batched] == [len(s) for s in single] == [3, 1, 5, 1]
    for ss, bs in zip(single, batched):
        for a, b in zip(ss, bs):
            for k in a.observations:
                assert torch.equal(a.observations[k], b.observations[k])
            for k in a.actions:
                assert torch.equal(a.actions[k], b.actions[k]) and torch.equal(a.masks[k], b.masks[k])
            ha = a.hidden if isinstance(a.hidden, tuple) else (a.hidden,)
            hb = b.hidden if isinstance(b.hidden, tuple) else (b.hidden,)
            for x, y in zip(ha, hb):
                torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(a.values, b.values, rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(a.dense_old_logp(), b.dense_old_logp(), rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(torch.as_tensor(a.advantages), torch.as_tensor(b.advantages), rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(torch.as_tensor(a.returns), torch.as_tensor(b.returns), rtol=1e-5, atol=1e-6)
            assert np.array_equal(a.rewards, b.rewards)
