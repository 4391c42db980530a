"""CPU tests of kickstarting (``teacher_model``, ``teacher_coef``, ``teacher_anneal_iterations``): every refusal, the CLI
flags and their way through ``main``, the anneal schedule against ``teacher_oracle``, ``Policy.from_state_dict`` on the
architectures the project trains (and on the reference's network), the teacher loader's refusals, the header against
``_lib``, and the batch field's plumbing."""
import os
import re
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kl_oracle as KO  # noqa: E402
import teacher_oracle as TO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dotaclient_b200.h")
BASE = (0.98, 0.97, 0.1, 0.5)


# ------------------------------------------------------------------------------------------------ settings and CLI
def test_settings_validation():
    from dotaclient_b200.optimizer import check_ppo_settings
    check_ppo_settings(*BASE)
    check_ppo_settings(*BASE, teacher_model="t.pt")
    check_ppo_settings(*BASE, teacher_model="t.pt", teacher_coef=0.0, teacher_anneal_iterations=1)
    check_ppo_settings(*BASE, teacher_model="t.pt", teacher_coef=25.0, teacher_anneal_iterations=1000)
    for kw, what in (({"teacher_coef": -0.1}, "teacher_coef"), ({"teacher_coef": float("nan")}, "teacher_coef"),
                     ({"teacher_coef": float("inf")}, "teacher_coef"), ({"teacher_coef": True}, "teacher_coef"),
                     ({"teacher_coef": "1"}, "teacher_coef"), ({"teacher_anneal_iterations": 0}, "teacher_anneal"),
                     ({"teacher_anneal_iterations": -3}, "teacher_anneal"),
                     ({"teacher_anneal_iterations": 2.5}, "teacher_anneal"),
                     ({"teacher_anneal_iterations": True}, "teacher_anneal")):
        with pytest.raises(ValueError, match=what):
            check_ppo_settings(*BASE, teacher_model="t.pt", **kw)
    # a non-default coefficient or an anneal without a teacher
    with pytest.raises(ValueError, match="teacher_coef=0.5 needs teacher_model"):
        check_ppo_settings(*BASE, teacher_coef=0.5)
    with pytest.raises(ValueError, match="teacher_anneal_iterations=10 needs teacher_model"):
        check_ppo_settings(*BASE, teacher_anneal_iterations=10)


def test_constructor_and_main_refuse_bad_settings_up_front():
    from dotaclient_b200.optimizer import DotaOptimizer, main
    with pytest.raises(ValueError, match="needs teacher_model"):
        DotaOptimizer("x", 0, 1, 8, 16, 5e-5, False, None, 1, "/nonexistent", 5e-4, 0.5, True, teacher_coef=2.0)
    with pytest.raises(ValueError, match="teacher_coef"):
        main("x", 0, 1, 8, 16, 5e-5, None, 1, "/nonexistent", 5e-4, 0.5, True, teacher_model="t.pt",
             teacher_coef=-1.0)


def test_cli_flags():
    from dotaclient_b200.optimizer import build_arg_parser
    p = build_arg_parser()
    a = p.parse_args([])
    assert a.teacher_model is None and a.teacher_coef == 1.0 and a.teacher_anneal_iterations is None
    a = p.parse_args(["--teacher-model", "model_000000100.pt", "--teacher-coef", "2.5",
                      "--teacher-anneal-iterations", "300"])
    assert (a.teacher_model, a.teacher_coef, a.teacher_anneal_iterations) == ("model_000000100.pt", 2.5, 300)
    for flag in ("--teacher-model", "--teacher-coef", "--teacher-anneal-iterations"):
        assert flag in p.format_help()


@pytest.mark.parametrize("kw", [{}, {"teacher_model": "t.pt"},
                                {"teacher_model": "t.pt", "teacher_coef": 3.0, "teacher_anneal_iterations": 7}])
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
    assert seen["teacher_model"] == kw.get("teacher_model") and seen["teacher_coef"] == kw.get("teacher_coef", 1.0)
    assert seen["teacher_anneal_iterations"] == kw.get("teacher_anneal_iterations") and seen["ran"]


# ------------------------------------------------------------------------------------------------ the anneal
class _Teacherless:
    """The attributes ``DotaOptimizer.teacher_anneal`` reads and writes, without a device."""

    def __init__(self, coef, n_anneal):
        self.teacher_model, self.teacher = "t.pt", object()
        self._teacher_coef0 = self.teacher_coef = coef
        self.teacher_anneal_iterations, self.teacher_iterations = n_anneal, 0
        self.retired = 0

    def _retire_teacher(self):
        self.retired += 1
        self.teacher = None


@pytest.mark.parametrize("coef,n_anneal", [(1.0, 4), (2.5, 1), (0.3, 7), (5.0, None)])
def test_anneal_schedule(coef, n_anneal):
    from dotaclient_b200.optimizer import DotaOptimizer
    o = _Teacherless(coef, n_anneal)
    for n in range(10):
        o.teacher_coef = 123.0                      # any value assigned since is overridden by the schedule
        o.teacher_iterations = n
        DotaOptimizer.teacher_anneal(o)
        want = TO.anneal(coef, n, n_anneal)
        if n_anneal is None:
            assert o.teacher_coef == 123.0 and o.retired == 0
            continue
        assert o.teacher_coef == pytest.approx(want, rel=1e-15, abs=0.0), n
        assert (o.teacher is None) == (n >= n_anneal), n
    if n_anneal is not None:
        assert TO.anneal(coef, 0, n_anneal) == coef and TO.anneal(coef, n_anneal, n_anneal) == 0.0


# ------------------------------------------------------------------------------------------------ from_state_dict
@pytest.mark.parametrize("cell", ["gru", "lstm"])
@pytest.mark.parametrize("layers", [1, 3])
@pytest.mark.parametrize("H", [64, 128, 256])
@pytest.mark.parametrize("K", [1, 3])
def test_from_state_dict_architectures(cell, layers, H, K):
    from dotaclient_b200.policy import Policy
    torch.manual_seed(H + layers)
    src = Policy(hidden_size=H, cell=cell, num_layers=layers, value_heads=K)
    pol = Policy.from_state_dict(src.state_dict())
    assert (pol.hidden_size, pol.cell, pol.num_layers, pol.value_heads) == (H, cell, layers, K)
    a, b = src.state_dict(), pol.state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


def test_from_state_dict_of_the_reference_network():
    from oracle.ref_policy import RefPolicy
    from dotaclient_b200.policy import Policy
    for H, cell in ((256, "gru"), (128, "lstm")):
        torch.manual_seed(7)
        ref = RefPolicy(H, cell)
        pol = Policy.from_state_dict(ref.state_dict())
        assert (pol.hidden_size, pol.cell, pol.num_layers, pol.value_heads) == (H, cell, 1, 1)
        sd = ref.state_dict()
        assert all(torch.equal(sd[k], v) for k, v in pol.state_dict().items())
    torch.manual_seed(7)                            # the reference's initialisation is Policy()'s
    ref = RefPolicy()
    torch.manual_seed(7)
    mine = Policy()
    assert all(torch.equal(ref.state_dict()[k], v) for k, v in mine.state_dict().items())


def test_from_state_dict_refuses_what_is_not_a_policy():
    from dotaclient_b200.policy import Policy
    sd = Policy(hidden_size=64).state_dict()
    bad = [{}, {"weight": torch.zeros(3)}, dict(sd, extra=torch.zeros(1)), {k: v for k, v in sd.items() if "ability" not in k},
           dict(sd, **{"rnn.weight_hh_l0": torch.zeros(5 * 64, 64)}),
           dict(sd, **{"affine_head_enum.weight": torch.zeros(4, 65)}),
           torch.nn.Linear(3, 4).state_dict()]
    for i, d in enumerate(bad):
        with pytest.raises(ValueError, match="not a Policy state_dict"):
            Policy.from_state_dict(d)


def test_teacher_loader_refusals(tmp_path):
    from dotaclient_b200.optimizer import load_teacher
    from dotaclient_b200.policy import Policy
    with pytest.raises(ValueError, match="no such file"):
        load_teacher(str(tmp_path / "missing.pt"))
    torch.save([1, 2, 3], str(tmp_path / "list.pt"))
    with pytest.raises(ValueError, match="does not hold a state_dict"):
        load_teacher(str(tmp_path / "list.pt"))
    torch.save(torch.nn.Linear(2, 2).state_dict(), str(tmp_path / "linear.pt"))
    with pytest.raises(ValueError, match="not a Policy state_dict"):
        load_teacher(str(tmp_path / "linear.pt"))
    torch.save(Policy(hidden_size=48).state_dict(), str(tmp_path / "w48.pt"))
    with pytest.raises(ValueError, match="multiples of 32"):
        load_teacher(str(tmp_path / "w48.pt"))
    torch.manual_seed(3)
    src = Policy(hidden_size=96, cell="lstm", num_layers=2)
    torch.save(src.state_dict(), str(tmp_path / "ok.pt"))
    t = load_teacher(str(tmp_path / "ok.pt"))
    assert (t.hidden_size, t.cell, t.num_layers) == (96, "lstm", 2)
    assert not any(p.requires_grad for p in t.parameters())
    assert all(torch.equal(src.state_dict()[k], v) for k, v in t.state_dict().items())


# ------------------------------------------------------------------------------------------------ C ABI
def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(dc_\w+)\s*\(([^;{]*?)\)\s*;", text):
        args = m.group(2).strip()
        protos[m.group(1)] = 0 if args in ("", "void") else args.count(",") + 1
    return protos


def test_header_and_lib_table_agree():
    from dotaclient_b200 import _lib
    protos = _declared()
    name = "dc_ppo_loss_fwd_bwd_teacher"
    assert name in protos and name in _lib.SIGNATURES
    assert len(_lib.SIGNATURES[name][1]) == protos[name] == protos["dc_ppo_loss_fwd_bwd_kl"] + 3
    d = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DC_[A-Z0-9_]+)\s+(-?\d+)", open(HEADER).read())}
    assert d["DC_TEACHER_STATS_SLOTS"] == _lib.TEACHER_STATS_SLOTS == 2 + len(KO.HEADS)
    assert d["DC_HPARAM_SLOTS"] == _lib.HPARAM_SLOTS == 10          # lambda is not a slot of the block


@pytest.fixture(scope="module")
def lib():
    from dotaclient_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_point_checks_its_arguments(lib):
    from dotaclient_b200 import _lib
    assert hasattr(lib, "dc_ppo_loss_fwd_bwd_teacher") and lib.dc_version() >= 113
    one = 4096
    p5 = _lib._ptr5(*[one] * 5)
    ld = (_lib._c.c_int64 * 5)(4, 9, 9, 40, 3)
    f = lib.dc_ppo_loss_fwd_bwd_teacher

    def call(rows=one, coef=one, tstats=one, hparams=one, n=8, old_rows=None, kl_out=None):
        return f(p5, ld, p5, p5, one, old_rows, rows, one, one, one, 1, None, None, n, hparams, coef, 0, p5, ld, one, 1,
                 one, one, kl_out, tstats, one, one, None)
    # null teacher operands / hyper-parameter block, and a bad token count, are refused before any CUDA call
    for kw, what in (({"rows": None}, b"teacher"), ({"coef": None}, b"teacher"), ({"tstats": None}, b"teacher"),
                     ({"hparams": None}, b"hyper-parameter"), ({"n": 0}, b"N=0")):
        assert call(**kw) == -1, kw
        assert what in lib.dc_last_error(), (kw, lib.dc_last_error())


# ------------------------------------------------------------------------------------------------ the batch field
def _batch(with_rows):
    from dotaclient_b200.optimizer import ExperienceBatch
    from dotaclient_b200.policy import Policy
    S, B = 4, 3
    obs = {k: torch.zeros(S, B, 2) for k in Policy.INPUT_KEYS}
    heads = {k: torch.zeros(S, B, n, dtype=torch.bool) for k, n in zip(KO.HEADS, KO.SIZES)}
    rows = torch.randn(S, B, 65) if with_rows else None
    return ExperienceBatch(obs, heads, dict(heads), torch.zeros(S, B, 5), torch.zeros(S, B), torch.zeros(S, B),
                           torch.zeros(1, B, 8), old_log_probs=torch.randn(S, B, 65), teacher_log_probs=rows)


def test_experience_batch_field():
    plain, t = _batch(False), _batch(True)
    assert plain.teacher_log_probs is None and t.teacher_log_probs.shape == (4, 3, 65)
    assert plain.graph_key() != t.graph_key() and t.graph_key()[:len(plain.graph_key())] == plain.graph_key()
    assert not any(f == "teacher_log_probs" for _, f, _ in plain.tensors())
    assert sum(f == "teacher_log_probs" for _, f, _ in t.tensors()) == 1
    m = t.map(lambda v: v.clone())
    assert torch.equal(m.teacher_log_probs, t.teacher_log_probs) and m.teacher_log_probs is not t.teacher_log_probs
    assert plain.map(lambda v: v.clone()).teacher_log_probs is None


def test_descriptor_budget():
    """The largest batch (every field, the teacher's rows included) still fits one gather launch."""
    from dotaclient_b200 import _lib
    from dotaclient_b200.optimizer import ExperienceBatch
    from dotaclient_b200.policy import Policy
    assert "teacher_log_probs" in ExperienceBatch.FIELDS
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
                     old_logp=torch.zeros(S, 5), teacher_log_probs=torch.full((S, 65), float(i)))
        s.advantages, s.returns = torch.zeros(S), torch.zeros(S)
        seqs.append(s)
    b = ExperienceBatch.from_sequences(seqs, torch.device("cpu"))
    assert b.teacher_log_probs.shape == (S, 2, 65) and float(b.teacher_log_probs[0, 1, 0]) == 1.0
    assert b.old_log_probs is None
    seqs[0].teacher_log_probs = None
    assert ExperienceBatch.from_sequences(seqs, torch.device("cpu")).teacher_log_probs is None


def test_oracle_is_the_kl_definition():
    """KL_T is kl_oracle's exact KL with the teacher's rows: 0 for the policy's own rows, > 0 for a tempered teacher."""
    g = torch.Generator().manual_seed(5)
    n = 64
    logits = {k: torch.randn(n, s, generator=g, dtype=torch.float64) for k, s in zip(KO.HEADS, KO.SIZES)}
    masks = {k: torch.rand(n, s, generator=g) < 0.7 for k, s in zip(KO.HEADS, KO.SIZES)}
    for k in masks:
        masks[k][:, 0] = True
    actions = {k: torch.zeros(n, s, dtype=torch.bool) for k, s in zip(KO.HEADS, KO.SIZES)}
    for k in actions:
        actions[k][::2, 0] = True
    own = TO.masked_log_rows(logits, masks)
    assert abs(float(TO.teacher_kl(logits, actions, masks, own)[0])) < 1e-12
    legal = torch.cat([masks[k] for k in KO.HEADS], dim=1)
    kl, _, t_a, _ = TO.teacher_kl(logits, actions, masks, KO.temper_rows(own, legal))
    assert float(kl) > 0 and t_a == n // 2
