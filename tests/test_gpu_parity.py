"""GPU parity tests: every CUDA kernel and the whole optimizer step against the CPU oracle.

All calls go through the C-ABI library (``dotaclient_b200._lib`` -> ``libdotaclient_b200.so``).
Tolerances (fp32 SIMT kernels vs torch-CPU fp32 oracle; stated per test):
  GAE                    bit-exact expected, <= 1 fp32 ulp allowed (float64 scan, different association)
  recurrence forward     atol 2e-5 on h after S steps
  recurrence backward    rtol 2e-4 / atol 2e-6 on dgi-derived gradients
  loss terms, entropies  rtol 1e-4, atol 1e-6
  parameter gradients    rtol 2e-3 on per-tensor norms, cosine >= 0.9999 on sampled tensors
  integer work           bit-exact (n_actions); action-index selection equal to sample_index on the random u used here
                         (a u within fp32 rounding of a cumulative boundary may take the adjacent index:
                         test_gpu_actor_fp64.py)
"""
import copy
import os
import uuid

import numpy as np
import pytest
import torch

from oracle import ref_optimizer as RO
from oracle.ref_policy import RefPolicy, masked_softmax
from dotaclient_b200.synthetic import make_rollout, ragged_lengths

pytestmark = pytest.mark.gpu
HEADS = ("enum", "x", "y", "target_unit", "ability")
SIZES = (4, 9, 9, 40, 3)


def dev():
    return torch.device("cuda", 0)


def make_optimizer(hidden_size, cell, seq_len, tmp_path, lr=5e-5, entropy_coef=5e-4, vf_coef=0.5):
    from dotaclient_b200.optimizer import DotaOptimizer
    return DotaOptimizer(rmq_host="test", rmq_port=uuid.uuid4().int % 100000, epochs=1, min_seq_per_epoch=1,
                         seq_len=seq_len, learning_rate=lr, checkpoint=False, pretrained_model=None,
                         mq_prefetch_count=1, log_dir=str(tmp_path), entropy_coef=entropy_coef, vf_coef=vf_coef,
                         run_local=True, hidden_size=hidden_size, cell=cell)


def make_oracle(hidden_size, cell, seq_len, **kw):
    torch.manual_seed(7)
    return RO.RefOptimizer(RefPolicy(hidden_size, cell), seq_len=seq_len, **kw)


def ulp_diff(a, b):
    a = np.ascontiguousarray(a, dtype=np.float32).view(np.int32).astype(np.int64)
    b = np.ascontiguousarray(b, dtype=np.float32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


# ------------------------------------------------------------------------------------------------ library
def test_native_library_loaded_and_device_is_hopper():
    from dotaclient_b200 import _lib
    lib = _lib.load()
    assert lib.dc_version() >= 100
    import ctypes
    sm, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(lib.dc_device_info(ctypes.byref(sm), ctypes.byref(major), ctypes.byref(minor)), "dc_device_info")
    assert major.value == 9 and sm.value >= 100


# ------------------------------------------------------------------------------------------------ GAE
def test_gae_kernel_known_answer_and_golden(gae_golden):
    from dotaclient_b200.optimizer import advantage_returns, discount
    a, q = advantage_returns(gae_golden["r"], gae_golden["v"], 0.98, 0.97)
    np.testing.assert_array_equal(a, gae_golden["adv"])
    np.testing.assert_array_equal(q, gae_golden["ret"])
    a2, q2 = advantage_returns(gae_golden["r2"], gae_golden["v2"], 0.98, 0.97)
    assert ulp_diff(a2, gae_golden["adv2"]).max() <= 1 and ulp_diff(q2, gae_golden["ret2"]).max() <= 1
    assert (a2 == gae_golden["adv2"]).mean() > 0.99
    d = discount(gae_golden["r2"], 0.98)
    assert ulp_diff(d, RO.discount(gae_golden["r2"], 0.98)).max() <= 1


@pytest.mark.parametrize("n_sub", [1, 10])
def test_gae_kernel_ragged_segments(n_sub):
    from dotaclient_b200 import ops
    rng = np.random.RandomState(5)
    lens = [1, 2, 31, 32, 33, 64, 100, 512, 1380, 7]
    off = np.concatenate([[0], np.cumsum(lens)])
    n = int(off[-1])
    rewards = (rng.randn(n, n_sub) * 0.1).astype(np.float32)
    values = rng.randn(n).astype(np.float32)
    adv, ret = ops.gae_scan(torch.from_numpy(rewards if n_sub > 1 else rewards[:, 0]).to(dev()),
                            torch.from_numpy(values).to(dev()), torch.from_numpy(off).to(dev()))
    adv, ret = adv.cpu().numpy(), ret.cpu().numpy()
    for lo, hi in zip(off[:-1], off[1:]):
        r = np.append(np.sum(rewards[lo:hi], axis=1), np.float32(0)).astype(np.float32)
        v = np.append(values[lo:hi], np.float32(0))
        a, q = RO.advantage_returns(r, v)
        assert ulp_diff(adv[lo:hi], a).max() <= 1, (lo, hi)
        assert ulp_diff(ret[lo:hi], q).max() <= 1, (lo, hi)
    # empty segment list is a no-op
    e1, e2 = ops.gae_scan(torch.zeros(0, device=dev()), torch.zeros(0, device=dev()),
                          torch.zeros(1, dtype=torch.int64, device=dev()))
    assert e1.numel() == 0 and e2.numel() == 0


def test_gae_full_size_segment_independence():
    """C2-sized input (256 x 512): scanning all rollouts at once == scanning each one alone (sampled), and the
    scan is linear in the rewards."""
    from dotaclient_b200 import ops
    g = torch.Generator().manual_seed(3)
    B, S = 256, 512
    r = (torch.randn(B * S, generator=g) * 0.1).to(dev())
    v = torch.randn(B * S, generator=g).to(dev())
    off = (torch.arange(B + 1) * S).to(dev())
    adv, ret = ops.gae_scan(r, v, off)
    for b in (0, 17, 255):
        a1, q1 = ops.gae_scan(r[b * S:(b + 1) * S], v[b * S:(b + 1) * S], torch.tensor([0, S], device=dev()))
        assert torch.equal(a1, adv[b * S:(b + 1) * S]) and torch.equal(q1, ret[b * S:(b + 1) * S])
        a, q = RO.advantage_returns(np.append(r[b * S:(b + 1) * S].cpu().numpy(), np.float32(0)),
                                    np.append(v[b * S:(b + 1) * S].cpu().numpy(), np.float32(0)))
        assert ulp_diff(a1.cpu().numpy(), a).max() <= 1 and ulp_diff(q1.cpu().numpy(), q).max() <= 1
    _, ret2 = ops.gae_scan(2 * r, v, off)
    torch.testing.assert_close(ret2, 2 * ret, rtol=1e-6, atol=1e-7)


# ------------------------------------------------------------------------------------------------ recurrence
def _torch_rnn(cell, H):
    cls = torch.nn.GRU if cell == "gru" else torch.nn.LSTM
    return cls(input_size=H, hidden_size=H, num_layers=1, batch_first=False)


@pytest.mark.parametrize("cell", ["gru", "lstm"])
@pytest.mark.parametrize("B,S,H", [(3, 7, 128), (2, 40, 128), (5, 16, 256), (2, 5, 512), (9, 33, 128),
                                   (301, 6, 128), (1, 3, 128), (1, 1, 256), (33, 9, 256), (64, 128, 256), (70, 40, 512), (3, 5, 384)])
def test_rnn_forward_backward_vs_torch(cell, B, S, H):
    """Recurrence kernels (+ the wgmma i2h GEMM and wgrads) against torch.nn.GRU / nn.LSTM on CPU: outputs, final state,
    all gradients.  H = 128 one-SM kernels, H = 256 cluster kernels (1 / 2 / 3 clusters, partly filled), H = 384 / 512 step-wise."""
    from dotaclient_b200 import ops
    torch.manual_seed(B * 1000 + S * 10 + H)
    ref = _torch_rnn(cell, H)
    x = torch.randn(S, B, H)
    h0 = torch.randn(1, B, H) * 0.5
    c0 = torch.randn(1, B, H) * 0.5
    wy, wh, wc = torch.randn(S, B, H), torch.randn(B, H), torch.randn(B, H)

    xr = x.clone().requires_grad_(True)
    h0r, c0r = h0.clone().requires_grad_(True), c0.clone().requires_grad_(True)
    if cell == "lstm":
        yr, (hn, cn) = ref(xr, (h0r, c0r))
        loss = (yr * wy).sum() + (hn[0] * wh).sum() + (cn[0] * wc).sum()
    else:
        yr, hn = ref(xr, h0r)
        loss = (yr * wy).sum() + (hn[0] * wh).sum()
    loss.backward()

    d = dev()
    p = {k: v.detach().clone().to(d).requires_grad_(True) for k, v in ref.named_parameters()}
    xg = x.to(d).requires_grad_(True)
    h0g = h0[0].to(d).requires_grad_(True)
    c0g = c0[0].to(d).requires_grad_(True) if cell == "lstm" else None
    y, hng, cng = ops.rnn_sequence(xg, p["weight_ih_l0"], p["weight_hh_l0"], p["bias_ih_l0"], p["bias_hh_l0"], h0g, c0g, cell)
    lg = (y * wy.to(d)).sum() + (hng * wh.to(d)).sum()
    if cell == "lstm":
        lg = lg + (cng * wc.to(d)).sum()
    lg.backward()
    torch.testing.assert_close(y.detach().cpu(), yr.detach(), rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(hng.detach().cpu(), hn[0].detach(), rtol=1e-4, atol=2e-5)
    if cell == "lstm":
        torch.testing.assert_close(cng.detach().cpu(), cn[0].detach(), rtol=1e-4, atol=2e-5)
    scale = max(1.0, float(S))
    torch.testing.assert_close(xg.grad.cpu(), xr.grad, rtol=2e-4, atol=2e-6 * scale)
    torch.testing.assert_close(h0g.grad.cpu(), h0r.grad[0], rtol=2e-4, atol=2e-6 * scale)
    if cell == "lstm":
        torch.testing.assert_close(c0g.grad.cpu(), c0r.grad[0], rtol=2e-4, atol=2e-6 * scale)
    for k, v in ref.named_parameters():
        torch.testing.assert_close(p[k].grad.cpu(), v.grad, rtol=5e-4, atol=5e-6 * scale * B)


@pytest.mark.parametrize("cell", ["gru", "lstm"])
@pytest.mark.parametrize("H", [64, 96])
def test_rnn_generic_kernels_vs_torch(cell, H):
    """The shape-generic recurrence kernels (H % 4 == 0 but not a multiple of 128), called through the C-ABI directly:
    ops.rnn_sequence needs H % 128 == 0 for its i2h GEMM.  B = 5 leaves the last CTA's 4-sequence tile partly filled.
    The i2h pre-activations and the weight gradients are computed on the CPU from what the kernels leave behind."""
    from dotaclient_b200 import _lib, ops
    B, S = 5, 6
    torch.manual_seed(B * 1000 + S * 10 + H)
    ref = _torch_rnn(cell, H)
    x = torch.randn(S, B, H)
    h0 = torch.randn(1, B, H) * 0.5
    c0 = torch.randn(1, B, H) * 0.5
    wy, wh, wc = torch.randn(S, B, H), torch.randn(B, H), torch.randn(B, H)
    xr = x.clone().requires_grad_(True)
    h0r, c0r = h0.clone().requires_grad_(True), c0.clone().requires_grad_(True)
    if cell == "lstm":
        yr, (hn, cn) = ref(xr, (h0r, c0r))
        loss = (yr * wy).sum() + (hn[0] * wh).sum() + (cn[0] * wc).sum()
    else:
        yr, hn = ref(xr, h0r)
        loss = (yr * wy).sum() + (hn[0] * wh).sum()
    loss.backward()

    d = dev()
    lib = _lib.load()
    w_ih, w_hh, b_ih, b_hh = (getattr(ref, k).detach() for k in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"))
    x2 = x.view(S * B, H)
    gates = (x2 @ w_ih.t() + b_ih).to(d).contiguous()
    ybuf = torch.zeros(S + 1, B, H, device=d)
    cbuf = torch.zeros(S + 1, B, H, device=d)
    ybuf[0] = h0[0].to(d)
    if cell == "lstm":
        cbuf[0] = c0[0].to(d)
    ws = torch.empty(max(int(lib.dc_rnn_workspace_bytes(ops.CELL_ID[cell], B, H)), 16), dtype=torch.uint8, device=d)
    w_hh_d, b_hh_d = w_hh.to(d).contiguous(), b_hh.to(d).contiguous()
    _lib.check(lib.dc_rnn_seq_fwd(ops.CELL_ID[cell], gates.data_ptr(), w_hh_d.data_ptr(), b_hh_d.data_ptr(), ybuf.data_ptr(),
                                  cbuf.data_ptr(), B, S, H, ws.data_ptr(), _lib.stream_ptr()), "dc_rnn_seq_fwd")
    torch.testing.assert_close(ybuf[1:].cpu(), yr.detach(), rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(ybuf[S].cpu(), hn[0].detach(), rtol=1e-4, atol=2e-5)
    if cell == "lstm":
        torch.testing.assert_close(cbuf[S].cpu(), cn[0].detach(), rtol=1e-4, atol=2e-5)

    dy, dhn = wy.to(d).contiguous(), wh.to(d).contiguous()
    dcn = wc.to(d).contiguous() if cell == "lstm" else None
    dh0 = torch.empty(B, H, device=d)
    dc0 = torch.empty(B, H, device=d) if cell == "lstm" else None
    _lib.check(lib.dc_rnn_seq_bwd(ops.CELL_ID[cell], gates.data_ptr(), w_hh_d.data_ptr(), ybuf.data_ptr(), cbuf.data_ptr(),
                                  dy.data_ptr(), dhn.data_ptr(), _lib.ptr(dcn), dh0.data_ptr(), _lib.ptr(dc0), B, S, H,
                                  ws.data_ptr(), _lib.stream_ptr()), "dc_rnn_seq_bwd")
    torch.cuda.synchronize()
    dgi = gates.cpu().double()                                    # [S*B, G*H], written in place of the saved gates
    hprev = ybuf[:S].cpu().double().view(S * B, H)                # h_{t-1} of every token
    if cell == "lstm":
        dgh = dgi                                                 # LSTM: the h2h gate gradients equal dgi
    else:
        dgh = torch.cat([dgi[:, :2 * H], cbuf[1:].cpu().double().view(S * B, H)], dim=1)   # GRU: n gate from cbuf
    scale = max(1.0, float(S))
    torch.testing.assert_close(dh0.cpu(), h0r.grad[0], rtol=2e-4, atol=2e-6 * scale)
    if cell == "lstm":
        torch.testing.assert_close(dc0.cpu(), c0r.grad[0], rtol=2e-4, atol=2e-6 * scale)
    torch.testing.assert_close((dgi @ w_ih.double()).float().view(S, B, H), xr.grad, rtol=2e-4, atol=2e-6 * scale)
    grads = {"weight_ih_l0": dgi.t() @ x2.double(), "bias_ih_l0": dgi.sum(0),
             "weight_hh_l0": dgh.t() @ hprev, "bias_hh_l0": dgh.sum(0)}
    for k, v in ref.named_parameters():
        torch.testing.assert_close(grads[k].float(), v.grad, rtol=5e-4, atol=5e-6 * scale * B)


@pytest.mark.parametrize("cell,H,B", [("lstm", 128, 256), ("gru", 128, 256), ("lstm", 256, 512), ("gru", 256, 512)])
def test_rnn_full_size_sampled_sequences(cell, H, B):
    """C2 shape (B=256, S=512, H=128) and C3's per-GPU shape (B=512, S=512, H=256): sequences are independent, so sampled
    rows must match the CPU oracle run on just those rows; state must carry across a split at S/2 (truncated-BPTT
    chunking, optimizer.py:343-385)."""
    from dotaclient_b200 import ops
    S = 512
    torch.manual_seed(11)
    ref = _torch_rnn(cell, H)
    x = torch.randn(S, B, H) * 0.7
    d = dev()
    p = {k: v.detach().to(d) for k, v in ref.named_parameters()}
    h0 = torch.zeros(B, H, device=d)
    c0 = torch.zeros(B, H, device=d) if cell == "lstm" else None
    with torch.no_grad():
        y, hn, cn = ops.rnn_sequence(x.to(d), p["weight_ih_l0"], p["weight_hh_l0"], p["bias_ih_l0"], p["bias_hh_l0"], h0, c0, cell)
        rows = [0, 1, 100, B - 1]
        xs = x[:, rows]
        z = torch.zeros(1, len(rows), H)
        yr = ref(xs, (z, z) if cell == "lstm" else z)[0]
        torch.testing.assert_close(y[:, rows].cpu(), yr, rtol=1e-4, atol=5e-5)
        # split at S/2 with carried state == one pass
        ya, ha, ca = ops.rnn_sequence(x[:S // 2].to(d), p["weight_ih_l0"], p["weight_hh_l0"], p["bias_ih_l0"], p["bias_hh_l0"], h0, c0, cell)
        yb, hb, cb = ops.rnn_sequence(x[S // 2:].to(d), p["weight_ih_l0"], p["weight_hh_l0"], p["bias_ih_l0"], p["bias_hh_l0"], ha,
                                      ca if cell == "lstm" else None, cell)
        assert torch.equal(torch.cat([ya, yb]), y) and torch.equal(hb, hn)


# ------------------------------------------------------------------------------------------------ PPO loss
def _random_loss_inputs(n_tokens, seed, drop_head=None, pad_from=None):
    g = torch.Generator().manual_seed(seed)
    roll = make_rollout(n_tokens, seed)
    masks = {k: v.clone() for k, v in roll["masks"].items()}
    actions = {k: v.clone() for k, v in roll["actions"].items()}
    if drop_head is not None:           # nobody used this head in the batch (optimizer.py:627-630)
        masks[drop_head][:] = False
        actions[drop_head][:] = False
    if pad_from is not None:            # zero-padded tail (optimizer.py:367-380)
        for k in HEADS:
            masks[k][pad_from:] = False
            actions[k][pad_from:] = False
    logits = {k: torch.randn(n_tokens, n, generator=g) for k, n in zip(HEADS, SIZES)}
    values = torch.randn(n_tokens, generator=g)
    adv = torch.randn(n_tokens, generator=g)
    ret = torch.randn(n_tokens, generator=g)
    with torch.no_grad():
        old = {}
        for k in HEADS:
            lp = masked_softmax(logits[k] + 0.3 * torch.randn(logits[k].shape, generator=g), masks[k], dim=1)
            old[k] = lp[actions[k]]
    return logits, masks, actions, old, values, adv, ret


@pytest.mark.parametrize("n_tokens,drop,pad", [(300, None, None), (129, "ability", 100), (64, "target_unit", None),
                                               (1000, None, 900), (5, "x", None)])
@pytest.mark.parametrize("coefs", [(5e-4, 0.5), (0.0, 0.5), (0.01, 0.0)])
def test_ppo_loss_kernel_vs_oracle(n_tokens, drop, pad, coefs):
    """Fused loss+grad kernel vs the oracle's autograd: losses, entropies, n_actions (bit-exact), dlogits, dvalue."""
    from dotaclient_b200 import ops
    entropy_coef, vf_coef = coefs
    logits, masks, actions, old, values, adv, ret = _random_loss_inputs(n_tokens, 7 + n_tokens, drop, pad)
    lg = {k: v.clone().unsqueeze(0).requires_grad_(True) for k, v in logits.items()}
    vg = values.clone().view(1, -1, 1).requires_grad_(True)
    loss, p_loss, e_loss, v_loss, ents = RO.ppo_loss(lg, vg, {k: v.unsqueeze(0) for k, v in actions.items()},
                                                     {k: v.unsqueeze(0) for k, v in masks.items()}, old,
                                                     adv.view(1, -1), ret.view(1, -1), entropy_coef, vf_coef)
    loss.backward()
    d = dev()
    dense_old = torch.zeros(n_tokens, 5)
    for h, k in enumerate(HEADS):
        dense_old[actions[k].any(dim=1), h] = old[k]
    out, n_act, dlogits, dvalue = ops.ppo_loss_fwd_bwd(
        [logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS], [actions[k].to(d) for k in HEADS],
        dense_old.to(d), adv.to(d), ret.to(d), values.to(d), 0.1, entropy_coef, vf_coef)
    out = out.cpu().numpy()
    expect_counts = [int(actions[k].any(dim=1).sum()) for k in HEADS]
    assert n_act.cpu().tolist() == expect_counts                       # integer work: bit-exact
    np.testing.assert_allclose(out[0], float(loss), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out[1], float(p_loss), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out[2], float(e_loss), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out[3], float(v_loss), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out[4:9], [float(ents[k]) for k in HEADS], rtol=1e-4, atol=1e-6)
    for h, k in enumerate(HEADS):
        g_ref = lg[k].grad[0] if lg[k].grad is not None else torch.zeros_like(logits[k])
        torch.testing.assert_close(dlogits[h].cpu(), g_ref, rtol=2e-4, atol=1e-8)
    gv = vg.grad.view(-1) if vg.grad is not None else torch.zeros(n_tokens)
    torch.testing.assert_close(dvalue.cpu(), gv, rtol=1e-4, atol=1e-9)


def test_selected_logp_kernel_and_index_selection():
    from dotaclient_b200 import ops
    logits, masks, actions, _, _, _, _ = _random_loss_inputs(777, 21, None, 700)
    d = dev()
    got = ops.selected_logp([logits[k].to(d) for k in HEADS], [masks[k].to(d) for k in HEADS],
                            [actions[k].to(d) for k in HEADS]).cpu()
    for h, k in enumerate(HEADS):
        step = actions[k].any(dim=1)
        lp = masked_softmax(logits[k], masks[k], dim=1)
        torch.testing.assert_close(got[step, h], lp[actions[k]], rtol=1e-5, atol=1e-6)
        assert (got[~step, h] == 0).all()


# ------------------------------------------------------------------------------------------------ optimizer
def _rollouts(n, seq_len, seed):
    return [make_rollout(L, 100 * seed + i) for i, L in enumerate(ragged_lengths(n, seq_len, seed))]


def _compare_sequences(mine, theirs, cell):
    assert len(mine) == len(theirs)
    for a, b in zip(mine, theirs):
        torch.testing.assert_close(a.advantages.cpu(), b.advantages, rtol=1e-4, atol=2e-5)
        torch.testing.assert_close(a.returns.cpu(), b.returns, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(a.values.cpu(), b.values, rtol=1e-4, atol=2e-5)
        ha = a.hidden if isinstance(a.hidden, tuple) else (a.hidden,)
        hb = b.hidden if isinstance(b.hidden, tuple) else (b.hidden,)
        for x, y in zip(ha, hb):
            torch.testing.assert_close(x.cpu(), y, rtol=1e-4, atol=2e-5)
        for k in HEADS:
            assert torch.equal(a.actions[k].cpu(), b.actions[k])        # selected indices: bit-exact
            torch.testing.assert_close(a.log_probs_sel[k].cpu(), b.log_probs_sel[k], rtol=1e-4, atol=2e-5)


@pytest.mark.parametrize("H,cell,S", [(256, "gru", 16), (128, "lstm", 16), (128, "gru", 8), (512, "lstm", 8)])
def test_optimizer_step_vs_oracle(H, cell, S, tmp_path):
    """experiences_from_rollout + three train() epochs against the oracle on identical ragged rollouts."""
    torch.set_num_threads(4)
    mine = make_optimizer(H, cell, S, tmp_path)
    oracle = make_oracle(H, cell, S)
    for (k, a), (k2, b) in zip(mine.policy_base.state_dict().items(), oracle.policy_base.state_dict().items()):
        assert k == k2 and torch.equal(a.cpu(), b), k                    # identical seeded init, identical layout
    rollouts = _rollouts(3, S, seed=H + S)
    xs_m, xs_o = [], []
    for r in rollouts:
        xs_m.extend(mine.experiences_from_rollout(copy.deepcopy(r)))
        xs_o.extend(oracle.experiences_from_rollout(copy.deepcopy(r)))
    _compare_sequences(xs_m, xs_o, cell)
    for ep in range(3):
        lm, em, gm = mine.train(xs_m)
        lo, eo, go = oracle.train(xs_o)
        for k in lo:
            np.testing.assert_allclose(float(lm[k]), float(lo[k]), rtol=2e-4, atol=2e-6, err_msg="%s ep%d" % (k, ep))
        for k in eo:
            np.testing.assert_allclose(float(em[k]), float(eo[k]), rtol=2e-4, atol=1e-6, err_msg="entropy %s" % k)
        np.testing.assert_allclose(float(gm["unclipped"]), float(go["unclipped"]), rtol=2e-3)
        np.testing.assert_allclose(float(gm["clipped"]), float(go["clipped"]), rtol=2e-3)
        if ep == 0:       # gradients (clipped, as left in .grad by both implementations)
            for name, p in oracle.policy_base.named_parameters():
                g = mine.flat.grad_of(name).cpu()
                assert p.grad is not None
                cos = torch.nn.functional.cosine_similarity(g.flatten(), p.grad.flatten(), dim=0)
                assert cos > 0.9999, (name, float(cos))
                np.testing.assert_allclose(float(g.norm()), float(p.grad.norm()), rtol=2e-3, err_msg=name)
    # after 3 Adam steps: the UPDATE (param - init) must agree with the oracle's.  Early Adam steps are ~ lr*sign(g),
    # unstable for g ~ 0, so compare direction over the whole vector and bound the element-wise gap by 2*lr per step.
    init = make_oracle(H, cell, S).policy_base.state_dict()
    dm = torch.cat([(a.cpu() - init[k]).flatten() for k, a in mine.policy_base.state_dict().items()])
    do = torch.cat([(b - init[k]).flatten() for k, b in oracle.policy_base.state_dict().items()])
    assert float(do.abs().max()) > 5e-5
    cos = torch.nn.functional.cosine_similarity(dm, do, dim=0)
    assert cos > 0.995, float(cos)
    assert float((dm - do).abs().max()) <= 3 * 2 * 5e-5 + 1e-6


def _adam_state_by_name(oracle):
    names = [n for n, _ in oracle.policy_base.named_parameters()]
    out = {}
    for n, p in zip(names, oracle.policy_base.parameters()):
        st = oracle.optimizer.state.get(p)
        if st:
            out[n] = st
    return out


@pytest.mark.parametrize("H,cell,S,B", [(128, "lstm", 512, 8), (128, "lstm", 64, 1), (256, "gru", 64, 1), (256, "lstm", 128, 40)])
def test_optimizer_step_long_bptt_vs_oracle(H, cell, S, B, tmp_path):
    """Whole train() steps at BASELINE sequence lengths: C2's S = 512 (B = 8 keeps the CPU oracle at ~1 s/step), C1 (B = 1,
    S = 64, at the widths of both the named LSTM-128 and the reference's GRU-256), and an H = 256 batch wide enough for the
    cluster kernels (two clusters, one partly filled).  Error growth through S-step BPTT INSIDE the step is what is
    tested: losses, entropies, gradient norms, per-tensor gradient direction, and after two steps torch.optim.Adam's own
    state (step, exp_avg, exp_avg_sq) -- SURVEY.md 8(c) asks for moments, not only post-step weights."""
    torch.set_num_threads(8)
    mine = make_optimizer(H, cell, S, tmp_path)
    oracle = make_oracle(H, cell, S)
    rollouts = [make_rollout(S, 900 + 10 * H + i) for i in range(B)]
    xs_m = [s for grp in mine.experiences_from_rollouts(copy.deepcopy(rollouts)) for s in grp]
    xs_o = [s for r in rollouts for s in oracle.experiences_from_rollout(copy.deepcopy(r))]
    _compare_sequences(xs_m, xs_o, cell)
    for ep in range(2):
        lm, em, gm = mine.train(xs_m)
        lo, eo, go = oracle.train(xs_o)
        for k in lo:
            np.testing.assert_allclose(float(lm[k]), float(lo[k]), rtol=2e-4, atol=2e-6, err_msg="%s ep%d" % (k, ep))
        for k in eo:
            np.testing.assert_allclose(float(em[k]), float(eo[k]), rtol=2e-4, atol=1e-6, err_msg="entropy %s" % k)
        np.testing.assert_allclose(float(gm["unclipped"]), float(go["unclipped"]), rtol=2e-3)
        np.testing.assert_allclose(float(gm["clipped"]), float(go["clipped"]), rtol=2e-3)
        if ep == 0:
            for name, p in oracle.policy_base.named_parameters():
                g = mine.flat.grad_of(name).cpu()
                cos = torch.nn.functional.cosine_similarity(g.flatten(), p.grad.flatten(), dim=0)
                assert cos > 0.9999, (name, float(cos))
                np.testing.assert_allclose(float(g.norm()), float(p.grad.norm()), rtol=2e-3, err_msg=name)
    # Adam state after two steps, tensor by tensor, in torch.optim.Adam's own layout
    sd = mine.optimizer.state_dict()["state"]
    want = _adam_state_by_name(oracle)
    names = [n for n, _ in oracle.policy_base.named_parameters()]
    assert sorted(names[i] for i in sd) == sorted(want)
    for i, st in sd.items():
        w = want[names[i]]
        assert float(st["step"]) == float(w["step"]) == 2.0
        m_scale = float(w["exp_avg"].abs().max())
        v_scale = float(w["exp_avg_sq"].abs().max())
        torch.testing.assert_close(st["exp_avg"], w["exp_avg"], rtol=2e-3, atol=2e-3 * m_scale + 1e-12)
        torch.testing.assert_close(st["exp_avg_sq"], w["exp_avg_sq"], rtol=4e-3, atol=4e-3 * v_scale + 1e-20)
        cos = torch.nn.functional.cosine_similarity(st["exp_avg"].flatten(), w["exp_avg"].flatten(), dim=0)
        assert cos > 0.9999, (names[i], float(cos))


def test_graph_replay_equals_launch_by_launch(tmp_path):
    """train() replayed from the CUDA graph of the step == the same step launched kernel by kernel: same losses, same
    gradient norms, same parameters and Adam state after five steps (the graph is captured on the second call of a shape;
    both optimizers start from the same seeded init and see the same batch)."""
    S, B = 16, 6
    a = make_optimizer(256, "gru", S, tmp_path)
    b = make_optimizer(256, "gru", S, tmp_path)
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


def test_prefetch_into_graph_slots_equals_plain_train(tmp_path):
    """The end-to-end path of the bench: pinned host batches uploaded by prefetch() into the two sets of static graph inputs,
    one upload ahead of the step being trained -- same results as training the same batches from device memory."""
    S, B = 16, 5
    a = make_optimizer(128, "lstm", S, tmp_path)
    b = make_optimizer(128, "lstm", S, tmp_path)
    b.use_cuda_graph = False
    batches = [a.batch_from_rollouts([make_rollout(S, 300 + 10 * j + i) for i in range(B)]) for j in range(3)]
    hosts = [bt.pin_memory() for bt in batches]
    order = [0, 1, 2, 0, 1, 2, 2, 0]
    staged = a.prefetch(hosts[order[0]])
    for n, j in enumerate(order):
        nxt = a.prefetch(hosts[order[n + 1]]) if n + 1 < len(order) else None       # one upload ahead
        la, _, ga = a.train(staged)
        lb, _, gb = b.train(batches[j])
        for k in la:
            np.testing.assert_allclose(float(la[k]), float(lb[k]), rtol=1e-6, atol=1e-9, err_msg="%s step %d" % (k, n))
        np.testing.assert_allclose(float(ga["unclipped"]), float(gb["unclipped"]), rtol=1e-6)
        staged = nxt
    assert sum(isinstance(v, tuple) for v in a._graphs.values()) == 2, "both input slots should be captured"
    torch.testing.assert_close(a.flat.param, b.flat.param, rtol=1e-6, atol=1e-9)


def test_batch_from_rollouts_equals_stacked_sequences(tmp_path):
    """The one-chunk fast path of batch_from_rollouts == ExperienceBatch.from_sequences over experiences_from_rollout."""
    from dotaclient_b200.optimizer import ExperienceBatch
    S = 16
    mine = make_optimizer(128, "lstm", S, tmp_path)
    rollouts = [make_rollout(S, 70 + i) for i in range(5)]
    fast = mine.batch_from_rollouts(copy.deepcopy(rollouts))
    slow = ExperienceBatch.from_sequences([s for r in rollouts for s in mine.experiences_from_rollout(copy.deepcopy(r))], dev())
    for (_, ka, a), (_, kb, b) in zip(fast.tensors(), slow.tensors()):
        assert ka == kb and a.shape == b.shape, (ka, a.shape, b.shape)
        if a.dtype == torch.bool or ka in ("h0", "c0"):
            assert torch.equal(a, b), ka
        else:
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6, msg=ka)
    ragged = [make_rollout(L, 80 + i) for i, L in enumerate((S, 2 * S + 3, S - 5, 4 * S))]
    general = mine.batch_from_rollouts(copy.deepcopy(ragged))
    assert general.batch_size == 1 + 3 + 1 + 4 and general.seq_len == S
    slow2 = ExperienceBatch.from_sequences([s for grp in mine.experiences_from_rollouts(copy.deepcopy(ragged)) for s in grp], dev())
    for (_, ka, a), (_, kb, b) in zip(general.tensors(), slow2.tensors()):
        assert ka == kb and a.shape == b.shape, (ka, a.shape, b.shape)
        if a.dtype == torch.bool:
            assert torch.equal(a, b), ka
        else:
            torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7, msg=ka)       # same kernels on the same data: (near-)identical


@pytest.mark.parametrize("H,cell", [(256, "gru"), (128, "lstm")])
def test_policy_single_and_sequence_on_cuda(H, cell, tmp_path):
    """Policy.init_hidden / sequence / single (policy.py:77-90) with CUDA tensors: an actor stepping one observation at a
    time through .single() reproduces the hidden-state chain and the logits of one .sequence() call, and both match the
    oracle (this is the actor-side use of the same kernels, batch 1)."""
    mine = make_optimizer(H, cell, 8, tmp_path).policy_base
    oracle = make_oracle(H, cell, 8).policy_base
    d = dev()
    r = make_rollout(6, 31)
    obs = r["observations"]

    def to_d(h):
        return tuple(x.to(d) for x in h) if isinstance(h, tuple) else h.to(d)
    with torch.no_grad():
        lo, vo, ho = oracle.sequence(hidden=oracle.init_hidden(), **{k: v.clone() for k, v in obs.items()})
        lm, vm, hm = mine.sequence(hidden=to_d(mine.init_hidden()), **{k: v.to(d) for k, v in obs.items()})
        for k in HEADS:
            assert lm[k].shape == lo[k].shape == (1, 6, dict(zip(HEADS, SIZES))[k])
            torch.testing.assert_close(lm[k].cpu(), lo[k], rtol=1e-4, atol=2e-5)
        torch.testing.assert_close(vm.cpu(), vo, rtol=1e-4, atol=2e-5)
        h = to_d(mine.init_hidden())
        for t in range(6):
            lt, vt, h = mine.single(hidden=h, **{k: v[t].to(d) for k, v in obs.items()})
            for k in HEADS:
                assert lt[k].shape[:2] == (1, 1)
                torch.testing.assert_close(lt[k][0, 0].cpu(), lo[k][0, t], rtol=1e-4, atol=3e-5)
            torch.testing.assert_close(vt[0, 0].cpu(), vo[0, t], rtol=1e-4, atol=3e-5)
        for a, b in zip(h if isinstance(h, tuple) else (h,), ho if isinstance(ho, tuple) else (ho,)):
            assert a.shape == b.shape
            torch.testing.assert_close(a.cpu(), b, rtol=1e-4, atol=3e-5)


def test_unused_head_leaves_sparse_params_untouched(tmp_path):
    """No attack action in the batch -> affine_unit_attention / affine_unit_eth get no gradient: Adam must skip them
    and the grad-norm mean must exclude them (optimizer.py:627-630,693; SURVEY.md 3.4)."""
    S = 8
    mine = make_optimizer(128, "lstm", S, tmp_path)
    oracle = make_oracle(128, "lstm", S)
    r = make_rollout(24, 9)
    attack = r["actions"]["target_unit"].any(dim=1)
    r["actions"]["enum"][attack] = False
    r["actions"]["enum"][attack, 0] = True                               # turn attacks into no-ops
    r["actions"]["target_unit"][:] = False
    r["masks"]["target_unit"][:] = False
    xm = mine.experiences_from_rollout(copy.deepcopy(r))
    xo = oracle.experiences_from_rollout(copy.deepcopy(r))
    before = {k: v.detach().cpu().clone() for k, v in mine.policy_base.state_dict().items()}
    lm, em, gm = mine.train(xm)
    lo, eo, go = oracle.train(xo)
    np.testing.assert_allclose(float(lm["loss"]), float(lo["loss"]), rtol=2e-4, atol=2e-6)
    np.testing.assert_allclose(float(gm["unclipped"]), float(go["unclipped"]), rtol=2e-3)
    assert float(em["target_unit"]) == 0.0
    after = mine.policy_base.state_dict()
    for k in before:
        sparse = k.startswith("affine_unit_attention") or k.startswith("affine_unit_eth")
        assert torch.equal(before[k], after[k].cpu()) == sparse, k
        assert (dict(oracle.policy_base.named_parameters())[k].grad is None) == sparse


def test_nan_loss_raises_value_error_and_keeps_params(tmp_path):
    mine = make_optimizer(128, "gru", 8, tmp_path)
    xs = mine.experiences_from_rollout(make_rollout(16, 2))
    xs[0].advantages = xs[0].advantages.clone()
    xs[0].advantages[3] = float("nan")
    before = mine.flat.param.clone()
    with pytest.raises(ValueError):
        mine.train(xs)
    assert torch.equal(before, mine.flat.param)


def test_gpu_path_vs_reference_golden(golden, tmp_path):
    """The CUDA path against outputs recorded from the unmodified reference (H=256 GRU, tests/golden)."""
    S = int(golden["seq_len"])
    mine = make_optimizer(256, "gru", S, tmp_path)
    sums = np.array([float(v.double().sum()) for v in mine.policy_base.state_dict().values()])
    np.testing.assert_allclose(sums, golden["init_param_sums"], rtol=0, atol=1e-9)
    xs = mine.experiences_from_rollout(make_rollout(int(golden["rollout_len"]), int(golden["rollout_seed"])))
    np.testing.assert_allclose(torch.stack([s.advantages for s in xs]).cpu().numpy(), golden["advantages"], rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(torch.stack([s.returns for s in xs]).cpu().numpy(), golden["returns"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(torch.stack([s.values.reshape(-1) for s in xs]).cpu().numpy(), golden["values"], rtol=1e-4, atol=2e-5)
    for k in HEADS:
        got = torch.cat([s.log_probs_sel[k] for s in xs]).cpu().numpy()
        np.testing.assert_allclose(got, golden["old_logp_" + k], rtol=1e-4, atol=2e-5)
    for ep in range(int(golden["epochs"])):
        l, e, g = mine.train(xs)
        got = [float(l[k]) for k in ("loss", "policy_loss", "entropy_loss", "value_loss")]
        np.testing.assert_allclose(got, golden["losses"][ep], rtol=2e-4, atol=2e-6)
        np.testing.assert_allclose([float(e[k]) for k in HEADS], golden["entropies"][ep], rtol=2e-4, atol=1e-6)
        np.testing.assert_allclose([float(g["unclipped"]), float(g["clipped"])], golden["grad_norms"][ep], rtol=2e-3)
    np.testing.assert_allclose(mine.policy_base.state_dict()["rnn.bias_hh_l0"].cpu().numpy(), golden["final_rnn_bias_hh"],
                               rtol=0, atol=6e-5)


def test_policy_forward_batch_first_api_matches_time_major(tmp_path):
    """Policy.forward (reference signature, batch-first) == the time-major fast path, and == the oracle forward."""
    mine = make_optimizer(128, "lstm", 8, tmp_path)
    oracle = make_oracle(128, "lstm", 8)
    B, S = 3, 8
    rolls = [make_rollout(S, 40 + i) for i in range(B)]
    obs_bf = {k: torch.stack([r["observations"][k] for r in rolls]) for k in mine.policy_base.INPUT_KEYS}
    h = torch.randn(1, B, 128) * 0.3
    c = torch.randn(1, B, 128) * 0.3
    with torch.no_grad():
        lo, vo, (hn, cn) = oracle.policy_base(**obs_bf, hidden=(h, c))
        d = dev()
        lm, vm, (hm, cm) = mine.policy_base(**{k: v.to(d) for k, v in obs_bf.items()}, hidden=(h.to(d), c.to(d)))
        lt, vt, _ = mine.policy_base.forward_time_major({k: v.transpose(0, 1).contiguous().to(d) for k, v in obs_bf.items()},
                                                        (h.to(d), c.to(d)))
    for k in HEADS:
        assert lm[k].shape == lo[k].shape
        torch.testing.assert_close(lm[k].cpu(), lo[k], rtol=1e-4, atol=2e-5)
        torch.testing.assert_close(lt[k].transpose(0, 1).cpu(), lo[k], rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(vm.cpu(), vo, rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(hm.cpu(), hn, rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(cm.cpu(), cn, rtol=1e-4, atol=2e-5)


def test_act_batched_pool_matches_per_agent_single(tmp_path):
    """Actor pool step (SURVEY.md 8(f)4): A agents through ONE batched forward + ONE selection launch == each agent's own
    Policy.single() on the oracle followed by the pinned index function; two consecutive steps so the carried hidden state
    is exercised."""
    from oracle.ref_policy import sample_index
    H, cell, A = 256, "gru", 37
    mine = make_optimizer(H, cell, 8, tmp_path).policy_base
    oracle = make_oracle(H, cell, 8).policy_base
    d = dev()
    g = torch.Generator().manual_seed(5)
    rolls = [make_rollout(2, 600 + a) for a in range(A)]
    hid_m = torch.zeros(1, A, H, device=d)
    hid_o = [oracle.init_hidden() for _ in range(A)]
    for t in range(2):
        obs = {k: torch.stack([r["observations"][k][t] for r in rolls]) for k in mine.INPUT_KEYS}
        masks = {k: torch.rand(A, n, generator=g) < 0.7 for k, n in zip(HEADS, SIZES)}
        for k in masks:
            masks[k][:, 1 if k == "target_unit" else 0] = True
        u = torch.rand(A, 5, generator=g)
        chosen, logp, logits, value, hid_m = mine.act_batched(hid_m, {k: v.to(d) for k, v in obs.items()},
                                                              {k: v.to(d) for k, v in masks.items()}, u.to(d))
        follow = {0: (), 1: ("x", "y"), 2: ("target_unit",), 3: ("ability",)}
        for a in range(A):
            with torch.no_grad():
                lo, vo, hid_o[a] = oracle.sequence(hidden=hid_o[a], **{k: v[a:a + 1] for k, v in obs.items()})
            for k in HEADS:
                torch.testing.assert_close(logits[k][a].cpu(), lo[k][0, 0], rtol=1e-4, atol=3e-5)
            torch.testing.assert_close(value[a].cpu(), vo[0, 0, 0], rtol=1e-4, atol=3e-5)
            e = sample_index(logits["enum"][a].cpu(), masks["enum"][a], float(u[a, 0]))      # the index function on OUR logits
            assert int(chosen["enum"][a]) == e
            for h, k in enumerate(HEADS):
                if k == "enum":
                    continue
                want = sample_index(logits[k][a].cpu(), masks[k][a], float(u[a, h])) if k in follow[e] else -1
                assert int(chosen[k][a]) == want, (t, a, k)
        torch.testing.assert_close(hid_m[0].cpu(), torch.cat([h[0] for h in hid_o]), rtol=1e-4, atol=3e-5)


def test_cpu_tensors_are_rejected_loudly():
    from dotaclient_b200 import ops
    with pytest.raises(RuntimeError):
        ops.gae_scan(torch.zeros(4), torch.zeros(4), torch.tensor([0, 4]))


def test_select_actions_batched_matches_oracle_index_function():
    """Actor-side hierarchical sampling in one launch (csrc/actor.cu) vs oracle.ref_policy.sample_index (policy.py:190-216):
    integer parity of the chosen indices for given uniforms, the enum -> sub-head rule, and the chosen log-probabilities."""
    from oracle.ref_policy import sample_index, masked_softmax
    from dotaclient_b200.policy import Policy
    g = torch.Generator().manual_seed(123)
    A = 300
    sizes = dict(enum=4, x=9, y=9, target_unit=40, ability=3)
    logits = {k: torch.randn(A, n, generator=g) * 2.0 for k, n in sizes.items()}
    masks = {k: torch.rand(A, n, generator=g) < 0.6 for k, n in sizes.items()}
    for k in masks:
        masks[k][:, 1 if k == 'target_unit' else 0] = True       # at least one valid entry per row
    masks['target_unit'][:, 0] = False                            # policy.py:255: unit 0 (self) is never a target
    masks['enum'][::7] = torch.tensor([True, False, False, False])   # some agents can only no-op
    u = torch.rand(A, 5, generator=g)
    d = torch.device("cuda", 0)
    chosen, logp = Policy.select_actions_batched({k: v.to(d) for k, v in logits.items()}, {k: v.to(d) for k, v in masks.items()},
                                                 u.to(d))
    chosen = {k: v.cpu() for k, v in chosen.items()}
    logp = logp.cpu()
    follow = {0: (), 1: ('x', 'y'), 2: ('target_unit',), 3: ('ability',)}
    keys = list(sizes)
    n_checked = 0
    for a in range(A):
        e = sample_index(logits['enum'][a], masks['enum'][a], float(u[a, 0]))
        assert int(chosen['enum'][a]) == e
        for h, k in enumerate(keys):
            if k == 'enum':
                continue
            if k in follow[e]:
                want = sample_index(logits[k][a], masks[k][a], float(u[a, h]))
                assert int(chosen[k][a]) == want, (a, k)
                lp = masked_softmax(logits[k][a].view(1, 1, -1), masks[k][a].view(1, 1, -1)).view(-1)[want]
                np.testing.assert_allclose(float(logp[a, h]), float(lp), rtol=1e-5, atol=1e-6)
                n_checked += 1
            else:
                assert int(chosen[k][a]) == -1
    assert n_checked > A // 2
    assert bool((chosen['enum'][::7] == 0).all())
