"""GPU parity of the whole optimizer at recurrent widths that are multiples of 32 but not of 128 (64, 96, 160, 192).
Their dense layers run on the ragged-N GEMM tiles and their recurrence on the generic kernels (csrc/rnn_generic.cuh).
The checks and tolerances are those of test_gpu_parity.py; the H = 128 / 256 tests there are the templates."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_parity as P  # noqa: E402
from dotaclient_b200.synthetic import make_rollout  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cell", ["gru", "lstm"])
@pytest.mark.parametrize("B,S,H", [(3, 7, 64), (5, 16, 96), (2, 5, 160), (33, 9, 192)])
def test_rnn_sequence_unaligned_width_vs_torch(cell, B, S, H):
    """ops.rnn_sequence (i2h GEMM with a ragged N, generic recurrence, weight gradients) against torch.nn.GRU / nn.LSTM on the
    CPU, as test_rnn_forward_backward_vs_torch checks it at the multiples of 128."""
    P.test_rnn_forward_backward_vs_torch(cell, B, S, H)


@pytest.mark.parametrize("cell", ["gru", "lstm"])
@pytest.mark.parametrize("H", [32, 64, 96, 192])
def test_rnn_sequence_unaligned_width_is_deterministic(cell, H):
    """Two runs of ops.rnn_sequence forward + backward on the same inputs are bitwise equal.  Below H = 128 the generic
    backward splits its dh mat-vec into slices, whose partial sums are added in a fixed order."""
    from dotaclient_b200 import ops
    B, S = 9, 12
    torch.manual_seed(H)
    G = 3 if cell == "gru" else 4
    d = P.dev()
    x = torch.randn(S, B, H, device=d)
    w = [torch.randn(G * H, H, device=d) * 0.3, torch.randn(G * H, H, device=d) * 0.3, torch.randn(G * H, device=d),
         torch.randn(G * H, device=d)]
    h0 = torch.randn(B, H, device=d) * 0.5
    c0 = torch.randn(B, H, device=d) * 0.5 if cell == "lstm" else None
    wy = torch.randn(S, B, H, device=d)

    def run():
        xg = x.clone().requires_grad_(True)
        ps = [t.clone().requires_grad_(True) for t in w]
        h0g = h0.clone().requires_grad_(True)
        y, hn, _ = ops.rnn_sequence(xg, *ps, h0g, c0, cell)
        ((y * wy).sum() + hn.sum()).backward()
        return [y.detach(), xg.grad, h0g.grad] + [p.grad for p in ps]

    for a, b in zip(run(), run()):
        assert torch.equal(a, b)


@pytest.mark.parametrize("H,cell,S", [(64, "gru", 16), (96, "lstm", 16), (160, "lstm", 8), (192, "gru", 8)])
def test_optimizer_step_unaligned_width_vs_oracle(H, cell, S, tmp_path):
    """experiences_from_rollout + three train() epochs against the oracle: losses, entropies, gradient norms, per-tensor
    gradients and the Adam update, exactly as test_optimizer_step_vs_oracle checks them at H = 128 / 256 / 512."""
    P.test_optimizer_step_vs_oracle(H, cell, S, tmp_path)


@pytest.mark.parametrize("H,cell,S,B", [(96, "lstm", 256, 8)])
def test_optimizer_step_long_bptt_unaligned_width_vs_oracle(H, cell, S, B, tmp_path):
    """Two train() steps with S = 256 BPTT at an unaligned width, including torch.optim.Adam's state after two steps, as
    test_optimizer_step_long_bptt_vs_oracle checks them."""
    P.test_optimizer_step_long_bptt_vs_oracle(H, cell, S, B, tmp_path)


def test_graph_replay_equals_launch_by_launch_h96(tmp_path):
    """train() replayed from the CUDA graph of the step == the same step launched kernel by kernel, at H = 96."""
    S, B, H = 16, 6, 96
    a = P.make_optimizer(H, "gru", S, tmp_path)
    b = P.make_optimizer(H, "gru", S, tmp_path)
    b.use_cuda_graph = False
    rollouts = [make_rollout(S, 40 + i) for i in range(B)]
    batch_a = a.batch_from_rollouts(copy.deepcopy(rollouts))
    batch_b = b.batch_from_rollouts(copy.deepcopy(rollouts))
    for step in range(5):
        la, ea, ga = a.train(batch_a)
        lb, eb, gb = b.train(batch_b)
        for k in la:
            np.testing.assert_allclose(float(la[k]), float(lb[k]), rtol=1e-6, atol=1e-9, err_msg="%s step %d" % (k, step))
        np.testing.assert_allclose(float(ga["unclipped"]), float(gb["unclipped"]), rtol=1e-6)
    assert any(isinstance(v, tuple) for v in a._graphs.values()), "the step was never captured"
    assert not any(isinstance(v, tuple) for v in b._graphs.values())
    torch.testing.assert_close(a.flat.param, b.flat.param, rtol=1e-6, atol=1e-9)
    torch.testing.assert_close(a.exp_avg, b.exp_avg, rtol=1e-5, atol=1e-12)
    assert torch.equal(a.adam_steps, b.adam_steps)


def test_batch_from_rollouts_equals_stacked_sequences_h96(tmp_path):
    """The one-chunk fast path of batch_from_rollouts == ExperienceBatch.from_sequences over experiences_from_rollout, at H = 96."""
    from dotaclient_b200.optimizer import ExperienceBatch
    S = 16
    mine = P.make_optimizer(96, "lstm", S, tmp_path)
    rollouts = [make_rollout(S, 70 + i) for i in range(5)]
    fast = mine.batch_from_rollouts(copy.deepcopy(rollouts))
    slow = ExperienceBatch.from_sequences([s for r in rollouts for s in mine.experiences_from_rollout(copy.deepcopy(r))], P.dev())
    for (_, ka, a), (_, kb, b) in zip(fast.tensors(), slow.tensors()):
        assert ka == kb and a.shape == b.shape, (ka, a.shape, b.shape)
        if a.dtype == torch.bool or ka in ("h0", "c0"):
            assert torch.equal(a, b), ka
        else:
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6, msg=ka)


def test_act_batched_pool_matches_per_agent_single_h96(tmp_path):
    """Actor pool step at H = 96: A agents through one batched forward + one selection launch == each agent's own
    Policy.single() on the oracle followed by the pinned index function, over two steps of carried hidden state."""
    from oracle.ref_policy import sample_index
    H, cell, A = 96, "gru", 37
    mine = P.make_optimizer(H, cell, 8, tmp_path).policy_base
    oracle = P.make_oracle(H, cell, 8).policy_base
    d = P.dev()
    g = torch.Generator().manual_seed(5)
    rolls = [make_rollout(2, 600 + a) for a in range(A)]
    hid_m = torch.zeros(1, A, H, device=d)
    hid_o = [oracle.init_hidden() for _ in range(A)]
    for t in range(2):
        obs = {k: torch.stack([r["observations"][k][t] for r in rolls]) for k in mine.INPUT_KEYS}
        masks = {k: torch.rand(A, n, generator=g) < 0.7 for k, n in zip(P.HEADS, P.SIZES)}
        for k in masks:
            masks[k][:, 1 if k == "target_unit" else 0] = True
        u = torch.rand(A, 5, generator=g)
        chosen, logp, logits, value, hid_m = mine.act_batched(hid_m, {k: v.to(d) for k, v in obs.items()},
                                                              {k: v.to(d) for k, v in masks.items()}, u.to(d))
        follow = {0: (), 1: ("x", "y"), 2: ("target_unit",), 3: ("ability",)}
        for a in range(A):
            with torch.no_grad():
                lo, vo, hid_o[a] = oracle.sequence(hidden=hid_o[a], **{k: v[a:a + 1] for k, v in obs.items()})
            for k in P.HEADS:
                torch.testing.assert_close(logits[k][a].cpu(), lo[k][0, 0], rtol=1e-4, atol=3e-5)
            torch.testing.assert_close(value[a].cpu(), vo[0, 0, 0], rtol=1e-4, atol=3e-5)
            e = sample_index(logits["enum"][a].cpu(), masks["enum"][a], float(u[a, 0]))
            assert int(chosen["enum"][a]) == e
            for h, k in enumerate(P.HEADS):
                if k == "enum":
                    continue
                want = sample_index(logits[k][a].cpu(), masks[k][a], float(u[a, h])) if k in follow[e] else -1
                assert int(chosen[k][a]) == want, (t, a, k)
        torch.testing.assert_close(hid_m[0].cpu(), torch.cat([h[0] for h in hid_o]), rtol=1e-4, atol=3e-5)


def test_policy_width_not_multiple_of_32_fails_at_first_forward(tmp_path):
    """Policy(hidden_size=100) constructs (it can hold a state_dict); its first CUDA forward raises the GEMM's width rule."""
    from dotaclient_b200.policy import Policy
    pol = Policy(hidden_size=100, cell="gru").to(P.dev())
    r = make_rollout(4, 3)
    obs = {k: v.to(P.dev()) for k, v in r["observations"].items()}
    with torch.no_grad(), pytest.raises(RuntimeError, match=r"N % 32 == 0 and K % 32 == 0"):
        pol.sequence(hidden=pol.init_hidden().to(P.dev()), **obs)
