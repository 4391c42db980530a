"""Host-side checks of the stacked recurrent core (``Policy(num_layers=L)``): parameter layout and seeded init against the
CPU oracle and stock torch, the flat parameter space, argument validation, the CLI flag, and the oracle's own wiring."""
import os
import re
import sys

import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from stacked_oracle import StackedRefPolicy  # noqa: E402
from dotaclient_b200.flat import FlatParameterSpace, head_dependency  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [(L, H, cell) for L in (1, 2, 3) for H, cell in ((256, "gru"), (128, "lstm"), (96, "gru"))]


def _rnn_cls(cell):
    return nn.GRU if cell == "gru" else nn.LSTM


@pytest.mark.parametrize("L,H,cell", CASES)
def test_state_dict_matches_stacked_oracle_and_torch_names(L, H, cell):
    from dotaclient_b200.policy import Policy
    torch.manual_seed(7)
    mine = Policy(hidden_size=H, cell=cell, num_layers=L)
    torch.manual_seed(7)
    ref = StackedRefPolicy(H, cell, L)
    a, b = mine.state_dict(), ref.state_dict()
    assert list(a) == list(b) and len(a) == 34 + 4 * (L - 1)
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k
    stock = _rnn_cls(cell)(input_size=H, hidden_size=H, num_layers=L, batch_first=True)
    assert [k for k in a if k.startswith("rnn.")] == ["rnn." + n for n in stock.state_dict()]
    # the rnn.* entries load into a stock multi-layer torch module and back
    stock.load_state_dict({k[4:]: v for k, v in a.items() if k.startswith("rnn.")}, strict=True)
    mine.rnn.load_state_dict(stock.state_dict(), strict=True)
    h = mine.init_hidden()
    for t in (h if cell == "lstm" else (h,)):
        assert t.shape == (L, 1, H) and not t.any()


@pytest.mark.parametrize("H,cell", [(256, "gru"), (128, "lstm")])
def test_single_layer_is_the_default_policy(H, cell):
    """num_layers=1 is the existing network: same keys, same seeded values; the stacked oracle at L = 1 is RefPolicy."""
    from dotaclient_b200.policy import Policy
    from oracle.ref_policy import RefPolicy
    torch.manual_seed(7)
    default = Policy(hidden_size=H, cell=cell).state_dict()
    torch.manual_seed(7)
    one = Policy(hidden_size=H, cell=cell, num_layers=1).state_dict()
    torch.manual_seed(7)
    ref = RefPolicy(H, cell).state_dict()
    torch.manual_seed(7)
    stacked_ref = StackedRefPolicy(H, cell, 1).state_dict()
    assert list(default) == list(one) == list(ref) == list(stacked_ref)
    for k in default:
        assert torch.equal(default[k], one[k]) and torch.equal(default[k], ref[k]) and torch.equal(ref[k], stacked_ref[k]), k
    assert Policy().num_layers == 1


@pytest.mark.parametrize("H,cell", [(256, "gru"), (128, "lstm")])
def test_stacked_oracle_at_one_layer_is_ref_policy(H, cell):
    """The stacked oracle at L = 1 is RefPolicy module for module (same children, same order, same types) and computes the
    same outputs, bit for bit, on a rollout."""
    from oracle.ref_policy import RefPolicy
    from dotaclient_b200.synthetic import make_rollout
    torch.manual_seed(7)
    ref = RefPolicy(H, cell)
    torch.manual_seed(7)
    stacked = StackedRefPolicy(H, cell, 1)
    assert [(n, type(m), repr(m)) for n, m in ref.named_children()] == \
        [(n, type(m), repr(m)) for n, m in stacked.named_children()]
    obs = make_rollout(12, 3)["observations"]
    with torch.no_grad():
        lr, vr, hr = ref.sequence(hidden=ref.init_hidden(), **obs)
        ls, vs, hs = stacked.sequence(hidden=stacked.init_hidden(), **obs)
    assert all(torch.equal(lr[k], ls[k]) for k in lr) and torch.equal(vr, vs)
    for a, b in zip(hr if cell == "lstm" else (hr,), hs if cell == "lstm" else (hs,)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("L", [1, 2, 3])
def test_flat_space_segments_of_a_stacked_policy(L):
    from dotaclient_b200.policy import Policy
    pol = Policy(hidden_size=128, cell="lstm", num_layers=L)
    flat = FlatParameterSpace(pol)
    assert flat.n_seg == 34 + 4 * (L - 1) and flat.names == list(pol.state_dict())
    rnn = [n for n in flat.names if n.startswith("rnn.")]
    assert len(rnn) == 4 * L
    assert all(head_dependency(n) == -1 for n in rnn)
    dep = dict(zip(flat.names, flat.seg_head.tolist()))
    assert all(dep[n] == -1 for n in rnn)


def test_layer_count_limit_matches_the_finish_kernel():
    """DotaOptimizer's 16-layer limit follows from the fused gradient-finish kernel's per-tensor slot count (kMaxSeg = 96):
    16 layers are 94 parameter tensors, 17 would be 98.  More than 16 are refused up front (before any device work) with a
    message naming the limit."""
    from dotaclient_b200 import _lib
    from dotaclient_b200.optimizer import DotaOptimizer
    from dotaclient_b200.policy import Policy
    with open(os.path.join(ROOT, "dotaclient_b200", "csrc", "grad_finish.cu")) as f:
        k_max_seg = int(re.search(r"constexpr int kMaxSeg = (\d+);", f.read()).group(1))
    assert _lib.MAX_PARAM_TENSORS == k_max_seg
    assert DotaOptimizer.MAX_LAYERS == 16
    n_tensors = [len(list(Policy(hidden_size=32, num_layers=L).parameters())) for L in (16, 17)]
    assert n_tensors[0] <= k_max_seg < n_tensors[1]
    for bad in (0, 17):
        with pytest.raises(ValueError, match="1 to 16 recurrent layers"):
            DotaOptimizer("x", 0, 1, 1, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, num_layers=bad)


def _adam_handle(H, L):
    """The optimizer's Adam handle over a CPU flat space of Policy(hidden_size=H, cell='lstm', num_layers=L)."""
    from types import SimpleNamespace
    from dotaclient_b200.optimizer import DotaOptimizer, _FusedAdamHandle
    from dotaclient_b200.policy import Policy
    flat = FlatParameterSpace(Policy(hidden_size=H, cell="lstm", num_layers=L))
    owner = SimpleNamespace(flat=flat, exp_avg=torch.zeros_like(flat.param), exp_avg_sq=torch.zeros_like(flat.param),
                            adam_steps=torch.zeros(flat.n_seg, dtype=torch.int32), learning_rate=5e-5,
                            ADAM_BETAS=DotaOptimizer.ADAM_BETAS, ADAM_EPS=DotaOptimizer.ADAM_EPS)
    return owner, _FusedAdamHandle(owner)


def test_adam_state_of_another_parameter_layout_is_refused_untouched():
    """Adam state is keyed by parameter index: a state saved for another layer count (or width) is refused with ValueError
    before any moment is changed; a state of the same layout round-trips."""
    g = torch.Generator().manual_seed(0)
    src, h_src = _adam_handle(128, 1)
    src.exp_avg.copy_(torch.randn(src.exp_avg.shape, generator=g))
    src.exp_avg_sq.copy_(torch.rand(src.exp_avg_sq.shape, generator=g))
    src.adam_steps.fill_(3)
    sd = h_src.state_dict()
    for H, L in ((128, 2), (96, 1)):                   # more tensors; same count, other shapes
        dst, h_dst = _adam_handle(H, L)
        dst.exp_avg.fill_(7.0)
        dst.adam_steps.fill_(5)
        with pytest.raises(ValueError, match="Adam state"):
            h_dst.load_state_dict(sd)
        assert bool((dst.exp_avg == 7.0).all()) and bool((dst.adam_steps == 5).all())
    with pytest.raises(ValueError, match="another parameter layout"):
        _adam_handle(128, 2)[1].load_state_dict({"exp_avg": src.exp_avg, "exp_avg_sq": src.exp_avg_sq, "step": src.adam_steps})
    same, h_same = _adam_handle(128, 1)
    h_same.load_state_dict(sd)
    assert torch.equal(same.adam_steps, src.adam_steps)
    for lo, hi in zip(same.flat.starts, same.flat.ends):
        assert torch.equal(same.exp_avg[lo:hi], src.exp_avg[lo:hi]) and torch.equal(same.exp_avg_sq[lo:hi], src.exp_avg_sq[lo:hi])


@pytest.mark.parametrize("bad", [0, -1, 1.5])
def test_policy_rejects_bad_layer_counts(bad):
    from dotaclient_b200.policy import Policy
    with pytest.raises(ValueError, match="num_layers"):
        Policy(hidden_size=128, num_layers=bad)


def test_cli_flag_num_layers():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    assert p.parse_args([]).num_layers == 1
    assert p.parse_args(["--num-layers", "2"]).num_layers == 2
    assert "recurrent layers (reference: 1)" in p.format_help()


@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_stacked_oracle_is_a_chain_of_single_layer_cells(cell):
    """The oracle's 2-layer torch module == two single-layer cells stepped by hand, layer 1 reading layer 0's outputs, with
    the same weights: output sequence and the [L, B, H] final states (h, and c for the LSTM)."""
    torch.manual_seed(3)
    H, B, S, L = 32, 3, 5, 2
    ref = StackedRefPolicy(H, cell, L)
    cell_cls = nn.GRUCell if cell == "gru" else nn.LSTMCell
    cells = []
    for k in range(L):
        c = cell_cls(H, H)
        for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
            getattr(c, n).data.copy_(getattr(ref.rnn, "%s_l%d" % (n, k)).data)
        cells.append(c)
    x = torch.randn(B, S, H)
    h0 = torch.randn(L, B, H) * 0.5
    c0 = torch.randn(L, B, H) * 0.5

    def by_hand(seq):
        hs, cs = [], []
        for k in range(L):
            h, c, out = h0[k], c0[k], []
            for t in range(S):
                if cell == "gru":
                    h = cells[k](seq[:, t], h)
                else:
                    h, c = cells[k](seq[:, t], (h, c))
                out.append(h)
            seq = torch.stack(out, dim=1)
            hs.append(h)
            cs.append(c)
        return seq, torch.stack(hs), torch.stack(cs)

    with torch.no_grad():
        y, hn, cn = by_hand(x)
        if cell == "gru":
            yr, hr = ref.rnn(x, h0)
        else:
            yr, (hr, cr) = ref.rnn(x, (h0, c0))
            torch.testing.assert_close(cr, cn, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(yr, y, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(hr, hn, rtol=1e-5, atol=1e-6)
