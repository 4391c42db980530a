"""CPU tests of KL control (``kl_coef``, ``kl_target``, ``kl_stop``): settings and CLI, the header against ``_lib``, the
adaptive coefficient and the skip decision against ``kl_oracle``, the batch field's plumbing, the coefficient's resume
round-trip, the flat gradient's tail, and the host half of two ranks over gloo (the same coefficient and the same stop
step from the all-reduced tail)."""
import os
import re
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kl_oracle as KO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
NEW_SYMBOLS = ("dc_selected_logp_rows", "dc_ppo_loss_fwd_bwd_kl", "dc_grad_finish_kl")


# ------------------------------------------------------------------------------------------------ settings and CLI
def test_settings_validation():
    from dotaclient_b200.optimizer import check_ppo_settings
    base = (0.98, 0.97, 0.1, 0.5)
    check_ppo_settings(*base)
    check_ppo_settings(*base, kl_coef=0.2, kl_target=0.01, kl_stop=0.05)
    check_ppo_settings(*base, kl_stop=0.02)                     # the early stop alone
    check_ppo_settings(*base, kl_coef=0.0)
    for kw, what in (({"kl_coef": -0.1}, "kl_coef"), ({"kl_coef": float("nan")}, "kl_coef"),
                     ({"kl_coef": float("inf")}, "kl_coef"), ({"kl_coef": True}, "kl_coef"),
                     ({"kl_coef": 0.1, "kl_target": 0.0}, "kl_target"), ({"kl_coef": 0.1, "kl_target": -1}, "kl_target"),
                     ({"kl_coef": 0.1, "kl_target": float("inf")}, "kl_target"),
                     ({"kl_coef": 0.1, "kl_target": float("nan")}, "kl_target"),
                     ({"kl_target": 0.01}, "kl_target"), ({"kl_coef": 0.0, "kl_target": 0.01}, "kl_target"),
                     ({"kl_stop": 0.0}, "kl_stop"), ({"kl_stop": -0.1}, "kl_stop"), ({"kl_stop": float("nan")}, "kl_stop"),
                     ({"kl_stop": float("inf")}, "kl_stop"), ({"kl_stop": "0.1"}, "kl_stop")):
        with pytest.raises(ValueError, match=what):
            check_ppo_settings(*base, **kw)


def test_constructor_and_main_refuse_bad_settings_up_front():
    from dotaclient_b200.optimizer import DotaOptimizer, main
    with pytest.raises(ValueError, match="kl_target"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, kl_target=0.01)
    with pytest.raises(ValueError, match="kl_stop"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, kl_stop=-1.0)


def test_cli_flags():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    a = p.parse_args([])
    assert a.kl_coef == 0.0 and a.kl_target is None and a.kl_stop is None
    a = p.parse_args(["--kl-coef", "0.2", "--kl-target", "0.01", "--kl-stop", "0.05"])
    assert (a.kl_coef, a.kl_target, a.kl_stop) == (0.2, 0.01, 0.05)
    for flag in ("--kl-coef", "--kl-target", "--kl-stop"):
        assert flag in p.format_help()


@pytest.mark.parametrize("kw", [{}, {"kl_coef": 0.2}, {"kl_coef": 0.2, "kl_target": 0.01, "kl_stop": 0.05}])
def test_main_passes_the_flags_to_the_optimizer(kw, monkeypatch):
    from dotaclient_b200 import optimizer as O
    seen = {}

    class Fake:
        mq = None

        def __init__(self, **k):
            seen.update(k)

        def run(self):
            seen["ran"] = True

    monkeypatch.setattr(O, "DotaOptimizer", Fake)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    O.main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, **kw)
    assert seen["kl_coef"] == kw.get("kl_coef", 0.0) and seen["kl_target"] == kw.get("kl_target")
    assert seen["kl_stop"] == kw.get("kl_stop") and seen["ran"]


# ------------------------------------------------------------------------------------------------ C ABI
def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(dc_\w+)\s*\(([^;{]*?)\)\s*;", text):
        args = m.group(2).strip()
        protos[m.group(1)] = 0 if args in ("", "void") else args.count(",") + 1
    return protos


def _defines():
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DC_[A-Z0-9_]+)\s+(-?\d+)", open(HEADER).read())}


def test_header_and_lib_table_agree():
    from dotaclient_b200 import _lib
    protos = _declared()
    for name in NEW_SYMBOLS:
        assert name in protos and name in _lib.SIGNATURES, name
        assert len(_lib.SIGNATURES[name][1]) == protos[name], name
    d = _defines()
    assert d["DC_HPARAM_SLOTS"] == _lib.HPARAM_SLOTS == 10
    assert (d["DC_HP_KL_COEF"], d["DC_HP_KL_STOP"]) == (_lib.HP_KL_COEF, _lib.HP_KL_STOP) == (8, 9)
    assert d["DC_PPO_STATS_SLOTS"] == _lib.PPO_STATS_SLOTS
    assert (d["DC_STAT_KL"], d["DC_STAT_KL_PENALTY"]) == (_lib.STAT_KL, _lib.STAT_KL_PENALTY)
    assert _lib.STAT_KL + 5 < _lib.STAT_KL_PENALTY < _lib.PPO_STATS_SLOTS
    assert _lib.STAT_JOINT_CLIP_FRACTION < _lib.STAT_KL        # the new slots come after every existing one
    assert d["DC_KL_ROW_FLOATS"] == _lib.KL_ROW_FLOATS == KO.ROW == 65
    assert d["DC_FINISH_KL_METRICS"] == _lib.FINISH_KL_METRICS == 6


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_new_symbols_are_exported_and_check_their_arguments(lib):
    from dotaclient_b200 import _lib
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name), name
    assert lib.dc_version() >= 110
    one = 4096
    p5 = _lib._ptr5(*[one] * 5)
    ld = (_lib._c.c_int64 * 5)(4, 9, 9, 40, 3)
    # null old_log_probs / hyper-parameter block / output pointers are refused before any CUDA call
    rc = lib.dc_ppo_loss_fwd_bwd_kl(p5, ld, p5, p5, one, None, one, one, one, 1, None, None, 8, one, 0, p5, ld, one, 1,
                                    one, one, None, one, one, None)
    assert rc == -1 and b"old_log_probs" in lib.dc_last_error()
    rc = lib.dc_ppo_loss_fwd_bwd_kl(p5, ld, p5, p5, one, one, one, one, one, 1, None, None, 8, None, 0, p5, ld, one, 1,
                                    one, one, None, one, one, None)
    assert rc == -1 and b"hyper-parameter" in lib.dc_last_error()
    assert lib.dc_selected_logp_rows(p5, p5, p5, 8, one, None, None) == -1
    assert lib.dc_selected_logp_rows(p5, p5, p5, 0, one, one, None) == -1
    rc = lib.dc_grad_finish_kl(one, one, one, one, one, one, one, one, 4, 64, None, 0.9, 0.999, 1e-8, one, one, one, None)
    assert rc == -1 and b"hyper-parameter" in lib.dc_last_error()


def test_hparam_block_slots():
    from dotaclient_b200 import _lib, ops
    import inspect
    sig = inspect.signature(ops.hparam_block)
    assert sig.parameters["kl_coef"].default == 0.0 and sig.parameters["kl_stop"].default is None
    assert _lib.HP_KL_COEF not in (_lib.HP_LR, _lib.HP_E_CLIP, _lib.HP_ENTROPY_COEF, _lib.HP_VF_COEF,
                                   _lib.HP_MAX_GRAD_NORM, _lib.HP_VALUE_CLIP, _lib.HP_VALUE_NORM_MEAN,
                                   _lib.HP_VALUE_NORM_STD)


# ------------------------------------------------------------------------------------------------ beta rule and skip
@pytest.mark.parametrize("kl,want", [(0.0151, 2.0), (0.015, 1.0), (0.0149, 1.0), (0.01, 1.0), (0.01 / 1.5, 1.0),
                                     (0.0066, 0.5), (0.0, 0.5), (10.0, 2.0)])
def test_beta_rule_and_its_boundaries(kl, want):
    from dotaclient_b200.optimizer import kl_coef_update
    got = kl_coef_update(0.4, kl, 0.01)
    assert got == KO.kl_coef_update(0.4, kl, 0.01) == 0.4 * want


def test_skip_decision():
    assert not KO.kl_skip(0.2, 10.0, None) and not KO.kl_skip(0.2, 10.0, 0.0)
    assert KO.kl_skip(0.21, 10.0, 0.02) and not KO.kl_skip(0.2, 10.0, 0.02)      # strictly above the limit
    assert not KO.kl_skip(5.0, 0.0, 0.02)                                       # T_a = 0: KL 0


def test_oracle_kl_is_zero_for_the_same_policy_and_positive_otherwise():
    from oracle.ref_policy import masked_softmax  # noqa: F401
    from dotaclient_b200.synthetic import make_rollout
    roll = make_rollout(50, 3)
    g = torch.Generator().manual_seed(1)
    logits = {k: torch.randn(50, n, generator=g, dtype=torch.float64) for k, n in zip(KO.HEADS, KO.SIZES)}
    rows = KO.masked_log_rows(logits, roll["masks"])
    kl, s, t_a, per = KO.exact_kl(logits, roll["actions"], roll["masks"], rows)
    assert abs(float(kl)) < 1e-12 and t_a > 0
    moved = {k: v + 0.3 * torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in logits.items()}
    kl2, _, _, per2 = KO.exact_kl(moved, roll["actions"], roll["masks"], rows)
    assert float(kl2) > 0 and all(v >= 0 for v in per2.values())


# ------------------------------------------------------------------------------------------------ batch plumbing
def _batch(with_rows, S=4, B=3):
    from dotaclient_b200.optimizer import ExperienceBatch
    from dotaclient_b200.policy import Policy
    obs = {k: torch.zeros(S, B, 2) for k in Policy.INPUT_KEYS}
    heads = {k: torch.zeros(S, B, n, dtype=torch.bool) for k, n in zip(KO.HEADS, KO.SIZES)}
    rows = torch.randn(S, B, 65) if with_rows else None
    return ExperienceBatch(obs, heads, dict(heads), torch.zeros(S, B, 5), torch.zeros(S, B), torch.zeros(S, B),
                           torch.zeros(1, B, 8), old_log_probs=rows)


def test_experience_batch_field():
    plain, kl = _batch(False), _batch(True)
    assert plain.old_log_probs is None and kl.old_log_probs.shape == (4, 3, 65)
    assert plain.graph_key() != kl.graph_key() and kl.graph_key()[:len(plain.graph_key())] == plain.graph_key()
    assert not any(f == "old_log_probs" for _, f, _ in plain.tensors())
    assert sum(f == "old_log_probs" for _, f, _ in kl.tensors()) == 1
    assert len(list(kl.tensors())) == len(list(plain.tensors())) + 1
    m = kl.map(lambda v: v.clone())
    assert torch.equal(m.old_log_probs, kl.old_log_probs) and m.old_log_probs is not kl.old_log_probs
    assert plain.map(lambda v: v.clone()).old_log_probs is None


def test_descriptor_budget():
    """The largest batch (LSTM, packed, valid, old values and the old rows) still fits one gather launch."""
    from dotaclient_b200 import _lib
    from dotaclient_b200.optimizer import ExperienceBatch
    from dotaclient_b200.policy import Policy
    n = len(Policy.INPUT_KEYS) + 2 * len(KO.HEADS) + len(ExperienceBatch.FIELDS)
    assert n <= _lib.GATHER_MAX_TENSORS, n


def test_from_sequences_carries_the_rows():
    from dotaclient_b200.optimizer import ExperienceBatch, Sequence
    from dotaclient_b200.policy import Policy
    S = 4
    seqs = []
    for i in range(2):
        obs = {k: torch.zeros(S, 2) for k in Policy.INPUT_KEYS}
        heads = {k: torch.zeros(S, n, dtype=torch.bool) for k, n in zip(KO.HEADS, KO.SIZES)}
        s = Sequence(None, 0, 0, obs, heads, dict(heads), torch.zeros(1, S, 1), torch.zeros(S), torch.zeros(1, 1, 8),
                     old_logp=torch.zeros(S, 5), old_log_probs=torch.full((S, 65), float(i)))
        s.advantages, s.returns = torch.zeros(S), torch.zeros(S)
        seqs.append(s)
    b = ExperienceBatch.from_sequences(seqs, torch.device("cpu"))
    assert b.old_log_probs.shape == (S, 2, 65) and float(b.old_log_probs[0, 1, 0]) == 1.0
    seqs[0].old_log_probs = None
    assert ExperienceBatch.from_sequences(seqs, torch.device("cpu")).old_log_probs is None


# ------------------------------------------------------------------------------------------------ flat tail
def test_grad_buffer_keeps_its_size_with_the_feature_off():
    from dotaclient_b200.flat import FlatParameterSpace
    net = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 2))
    off = FlatParameterSpace(net)
    assert off.grad_full.numel() == off.total + off.n_seg and off.kl_tail is None
    assert off.flags.numel() == off.n_seg
    net2 = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 2))
    on = FlatParameterSpace(net2, kl_tail=True)
    assert on.grad_full.numel() == on.total + on.n_seg + 2 and on.flags.numel() == on.n_seg
    assert on.kl_tail.numel() == 2 and on.kl_tail.data_ptr() == on.grad_full[on.total + on.n_seg:].data_ptr()


# ------------------------------------------------------------------------------------------------ resume
def _stub(tmp_path, kl_target):
    from dotaclient_b200.optimizer import DotaOptimizer
    o = DotaOptimizer.__new__(DotaOptimizer)
    o.kl_coef, o.kl_target, o.log_dir = 0.2, kl_target, str(tmp_path)
    return o


def test_beta_resume_round_trip(tmp_path):
    from dotaclient_b200.optimizer import DotaOptimizer
    path = os.path.join(str(tmp_path), DotaOptimizer.KL_COEF_FILENAME_FMT % 7)
    torch.save({"kl_coef": 0.8125}, path)
    o = _stub(tmp_path, 0.01)
    o._restore_kl_coef(path)
    assert o.kl_coef == 0.8125
    fresh = _stub(tmp_path, 0.01)
    fresh._restore_kl_coef(os.path.join(str(tmp_path), DotaOptimizer.KL_COEF_FILENAME_FMT % 8))   # absent: unchanged
    assert fresh.kl_coef == 0.2
    fixed = _stub(tmp_path, None)
    fixed._restore_kl_coef(path)                                  # without kl_target the file is ignored
    assert fixed.kl_coef == 0.2


# ------------------------------------------------------------------------------------------------ two ranks over gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _kl_worker(rank, world, port, out_dir):
    """Each rank holds its own (sum_t KL_t, T_a) per step in the flat gradient's tail; the one all-reduce of grad_full
    sums them, and the host decisions read only the reduced numbers."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dotaclient_b200.distributed import DistributedDataParallelSparseParamCPU
    from dotaclient_b200.flat import FlatParameterSpace
    from dotaclient_b200.optimizer import kl_coef_update
    torch.manual_seed(3)
    net = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 2))
    space = FlatParameterSpace(net, kl_tail=True)
    ddp = DistributedDataParallelSparseParamCPU(net, flat_space=space)
    # rank-local numbers that differ between the ranks: rank 1's KL grows faster
    local = [(0.004 * (s + 1) * (1 + 3 * rank) * (50 + rank), 50.0 + rank) for s in range(6)]
    all_ranks, stop = [], None
    for s, (ks, ta) in enumerate(local):
        space.grad_full.zero_()
        space.kl_tail.copy_(torch.tensor([ks, ta]))
        ddp.allreduce_gradients(divide=False)
        tot, cnt = space.kl_tail.tolist()
        all_ranks.append(tot / cnt)
        if stop is None and KO.kl_skip(tot, cnt, 0.03):
            stop = s
    beta = kl_coef_update(0.2, sum(all_ranks[:stop + 1]) / (stop + 1), 0.01)
    torch.save({"all_ranks": all_ranks, "stop": stop, "beta": beta, "local": local}, os.path.join(out_dir, "r%d.pt" % rank))
    dist.destroy_process_group()


def test_two_ranks_reach_the_same_stop_step_and_beta(tmp_path):
    mp.spawn(_kl_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    assert r0["all_ranks"] == r1["all_ranks"] and r0["stop"] == r1["stop"] and r0["beta"] == r1["beta"]
    # the reduced KL is the ratio of the summed numerators and counts, not a mean of the rank-local KLs
    for s, k in enumerate(r0["all_ranks"]):
        (a0, c0), (a1, c1) = r0["local"][s], r1["local"][s]
        assert abs(k - (a0 + a1) / (c0 + c1)) <= 1e-6 * k
    # rank 0 alone would not stop at all: the shared decision follows the all-ranks KL
    alone = next((s for s, (a, c) in enumerate(r0["local"]) if KO.kl_skip(a, c, 0.03)), None)
    assert r0["stop"] == 2 and alone is None
    assert r0["beta"] == 0.4                                       # d > 1.5 * 0.01: doubled on both ranks
