"""The gradient finish (``csrc/grad_finish.cu``: has-grad divide, gradient norms, global-norm clip, Adam) against one
finish step written out in float64 from the equations, on the host.

Every step is checked on its own: the float64 reference and the fp32 calibration start from the state the kernel holds
before the step, so errors do not carry from one step to the next.  The calibration is what the reference optimizer runs:
``torch.optim.Adam(foreach=False)`` and ``torch.nn.utils.clip_grad_norm_`` in fp32, with ``.grad = None`` for a tensor
whose has-grad count is 0.  Per tensor and per kind of value:

    max|gpu - f64| <= K * max|torch32 - f64| + FLOOR * max|f64|

The parameters are judged by their update (after - before), not by their value: an error in the update disappears
against |param|.  ``test_bound_passes_fp32_and_rejects_host_mutants`` shows, without a GPU, that torch fp32 and an fp32
transcription of the finish pass the bound and that six plausible bugs fail it.

Measured on one H100 80GB HBM3 (700 W power limit), the largest ratio max|gpu - f64| / max|torch32 - f64| over 8
steps, per layout and starting state, for update / exp_avg / exp_avg_sq / clipped gradient / metrics[0..2]:
    lstm128           fresh  2.3 / 1    / 1.3  / 1 / 0.27    resumed  2.7 / 1.3 / 1   / 1 / 1.5
    lstm256           fresh 15   / 1    / 1    / 1 / 0.15    resumed  4.2 / 1   / 1   / 1 / 1
    lstm512           fresh  1.3 / 1    / 1    / 1 / 0.03    resumed  4.3 / 1.1 / 1   / 1 / 1.2
    gru256            fresh  2.0 / 1    / 1.8  / 1 / 1       resumed  2.2 / 1.1 / 1   / 1 / 4.4
    lstm128 16 layers fresh  1.5 / 1.1  / 1.0  / 1 / 1       resumed  3.0 / 1.2 / 1.2 / 1 / 1
    synthetic96       fresh  1.9 / 1.8  / 1.9  / 1 / 11      resumed  3.6 / 1.3 / 1   / 1 / 0.26
    scalar entry point, synthetic96 fresh: 2.5 / 1 / 1 / 1 / 0.02
Ratios above K pass on the floor: there torch's own error happened to be far below an ulp of the value (the metrics are
float64 sums in the kernel).  The host mutants reach ratios of 2e6 to 7e8.  Before the kernel rounded 1 - beta from
float64 as torch does, the fresh states gave update ratios of 85 to 1700 and exp_avg_sq ratios up to 1700.
"""
import math

import numpy as np
import pytest
import torch

BETAS = (0.9, 0.999)
EPS = 1e-8
ALIGN = 64                        # floats: FlatParameterSpace.ALIGN
VALUE_SLOT = 5                    # flat.VALUE_SLOT
SENTINEL = {"p": 1234.5, "m": -777.25, "v": 4096.125, "g": -31.5}    # alignment padding of the four flat buffers
# (K, FLOOR) per kind of value: allowed multiple of torch fp32's error against float64, and the floor as a fraction of
# max|f64| of the tensor
BOUNDS = {"update": (8.0, 1e-6), "exp_avg": (4.0, 1e-7), "exp_avg_sq": (4.0, 1e-7), "grad": (4.0, 1e-7),
          "metrics": (4.0, 1e-7)}
LRS = (1e-2, 3e-3, 1e-3, 3e-4, 1e-2, 5e-5, 2e-3, 1e-3)       # lr of step k, written into the hyper-parameter block
CLIP_STEPS = (0, 2, 3, 6)        # max_norm = total / 4 on these steps (clip active), 4 x total on the others
N_STEPS = 8


# ------------------------------------------------------------------------------------------------ layouts and inputs
class Layout:
    """Segments [lo, hi) of one flat buffer, each starting on an ALIGN boundary, and the head each one depends on."""

    def __init__(self, name, sizes, heads):
        self.name, self.heads = name, list(heads)
        self.lo, self.hi, cursor = [], [], 0
        for s in sizes:
            self.lo.append(cursor)
            self.hi.append(cursor + s)
            cursor = (cursor + s + ALIGN - 1) // ALIGN * ALIGN
        self.total = cursor
        self.n = len(sizes)

    def sizes(self):
        return [b - a for a, b in zip(self.lo, self.hi)]


def policy_layout(hidden, cell, num_layers=1):
    from dotaclient_b200.flat import FlatParameterSpace
    from dotaclient_b200.policy import Policy
    torch.manual_seed(0)
    flat = FlatParameterSpace(Policy(hidden_size=hidden, cell=cell, num_layers=num_layers), "cpu")
    lay = Layout("%s%d-L%d" % (cell, hidden, num_layers), [b - a for a, b in zip(flat.starts, flat.ends)],
                 flat.seg_head.tolist())
    assert lay.lo == flat.starts and lay.total == flat.total
    return lay


def synthetic_layout():
    """96 segments (kMaxSeg): lengths 1, 3, 63, 64 and 65, one of 1.2M elements (about 18 turns of the grid-stride loop
    of 2 x 132 SMs x 256 threads), the rest 1..5000; a head on every seventh, the value slot on two."""
    g = torch.Generator().manual_seed(96)
    sizes = torch.randint(1, 5000, (96,), generator=g).tolist()
    sizes[:6] = [1, 3, 63, 64, 65, 1_200_003]
    heads = [(i // 7) % 5 if i % 7 == 3 else -1 for i in range(96)]
    heads[10] = heads[50] = VALUE_SLOT
    return Layout("synthetic96", sizes, heads)


def count_plan(layout, k):
    """Has-grad count of every tensor at step k: head tensors have none on steps 0-2 and one afterwards; every fifth other
    tensor sums 2 ranks, the next 3; the rest 1."""
    counts = []
    for i, h in enumerate(layout.heads):
        if 0 <= h < VALUE_SLOT:
            counts.append(0 if k < 3 else 1)
        else:
            counts.append((1, 2, 3, 1, 1)[i % 5])
    return counts


def tensor_scales(layout, seed):
    g = torch.Generator().manual_seed(seed)
    return (10.0 ** (torch.rand(layout.n, generator=g, dtype=torch.float64) * 7.0 - 6.0)).tolist()    # 10^U(-6, 1)


def make_plan(layout, seed, n_steps=N_STEPS, clip_steps=CLIP_STEPS):
    """Per step: the fp32 gradient sums the buffer holds (the sum of `count` rank gradients; random junk the kernel must
    ignore where the count is 0), the counts, lr, and a max_norm (an fp32 value) that puts the clip on or off."""
    g = torch.Generator().manual_seed(seed)
    scale = tensor_scales(layout, seed)
    plan = []
    for k in range(n_steps):
        counts = count_plan(layout, k)
        gsum = []
        for i, n in enumerate(layout.sizes()):
            c = counts[i]
            ranks = torch.randn(max(c, 1), n, generator=g) * scale[i]
            if i % 3 == 0:                          # about 30 % exact zeros, on every rank
                ranks *= (torch.rand(n, generator=g) >= 0.3).float()
            s = ranks[0].clone()
            for r in range(1, c):
                s += ranks[r]                       # fp32, as the all-reduce sums
            gsum.append(s)
        sq = sum(float((gsum[i].double() / c).pow(2).sum()) for i, c in enumerate(counts) if c > 0)
        total = math.sqrt(sq)
        max_norm = float(np.float32(total * (0.25 if k in clip_steps else 4.0)))
        plan.append({"gsum": gsum, "counts": counts, "lr": LRS[k % len(LRS)], "max_norm": max_norm})
    return plan


def make_state(layout, seed, resumed):
    """Parameters N(0, 0.01); fresh: zero moments and counters; resumed: counters of 10^6 (head tensors 3 behind) and
    moments of the tensor's gradient scale."""
    g = torch.Generator().manual_seed(seed + 1)
    scale = tensor_scales(layout, seed)
    st = {"p": [], "m": [], "v": [], "steps": []}
    for i, n in enumerate(layout.sizes()):
        st["p"].append(torch.randn(n, generator=g) * 0.01)
        if resumed:
            st["m"].append(torch.randn(n, generator=g) * scale[i] * 0.3)
            st["v"].append((torch.rand(n, generator=g) * scale[i] + 1e-3 * scale[i]).pow(2))
            st["steps"].append(10 ** 6 - (3 if 0 <= layout.heads[i] < VALUE_SLOT else 0))
        else:
            st["m"].append(torch.zeros(n))
            st["v"].append(torch.zeros(n))
            st["steps"].append(0)
    return st


# ------------------------------------------------------------------------------------------------ references
def step_f64(st, inp):
    """One finish step in float64 from the equations, from the fp32 state ``st``."""
    b1, b2 = BETAS
    counts = inp["counts"]
    g = [inp["gsum"][i].double() / c if c > 0 else None for i, c in enumerate(counts)]
    sq = [float(x.pow(2).sum()) for x in g if x is not None]
    total = math.sqrt(sum(sq))
    mean = sum(math.sqrt(s) for s in sq) / len(sq) if sq else 0.0
    coef = min(1.0, inp["max_norm"] / (total + 1e-6))
    out = {"p": [], "m": [], "v": [], "steps": [], "g": [], "metrics": [mean, mean * coef, total, 0.0]}
    for i, c in enumerate(counts):
        p, m, v = st["p"][i].double(), st["m"][i].double(), st["v"][i].double()
        if c == 0:
            out["g"].append(None)
            out["steps"].append(st["steps"][i])
        else:
            gc = g[i] * coef
            m = b1 * m + (1.0 - b1) * gc
            v = b2 * v + (1.0 - b2) * gc * gc
            s = st["steps"][i] + 1
            bc1, bc2 = 1.0 - b1 ** s, 1.0 - b2 ** s
            p = p - inp["lr"] / bc1 * m / (v.sqrt() / math.sqrt(bc2) + EPS)
            out["g"].append(gc)
            out["steps"].append(s)
        out["p"].append(p)
        out["m"].append(m)
        out["v"].append(v)
    return out


def step_torch32(st, inp):
    """The calibration: torch.optim.Adam(foreach=False) + clip_grad_norm_ in fp32, each tensor with its own step
    counter, .grad = None where the count is 0."""
    params = [torch.nn.Parameter(p.clone()) for p in st["p"]]
    opt = torch.optim.Adam(params, lr=inp["lr"], betas=BETAS, eps=EPS, foreach=False)
    for i, p in enumerate(params):
        opt.state[p] = {"step": torch.tensor(float(st["steps"][i])), "exp_avg": st["m"][i].clone(),
                        "exp_avg_sq": st["v"][i].clone()}
        c = inp["counts"][i]
        p.grad = inp["gsum"][i] / c if c > 0 else None
    live = [p for p in params if p.grad is not None]
    norms = lambda: float(torch.stack([p.grad.norm(2) for p in live]).mean()) if live else 0.0   # noqa: E731
    unclipped = norms()
    total = float(torch.nn.utils.clip_grad_norm_(live, inp["max_norm"], foreach=False)) if live else 0.0
    clipped = norms()
    opt.step()
    out = {"p": [], "m": [], "v": [], "steps": [], "g": [], "metrics": [unclipped, clipped, total, 0.0]}
    for p in params:
        s = opt.state[p]
        out["p"].append(p.detach())
        out["m"].append(s["exp_avg"])
        out["v"].append(s["exp_avg_sq"])
        out["steps"].append(int(s["step"]))
        out["g"].append(None if p.grad is None else p.grad.detach())
    return out


def f32(x):
    return float(np.float32(x))


class HostFinish:
    """An fp32 transcription of the finish on the host, optionally with one bug (``mutant``):
    'bc_step' bias corrections with step instead of step + 1; 'bc2_no_sqrt' dividing by bc2 instead of sqrt(bc2);
    'eps_inside' eps inside the square root; 'no_clip' the clip coefficient ignored; 'no_divide_2' no divide for a
    count of 2; 'global_step' one step counter for every tensor instead of each tensor's own."""

    def __init__(self, st, mutant=None):
        self.st = {k: [t.clone() for t in v] if k != "steps" else list(v) for k, v in st.items()}
        self.mutant = mutant
        self.global_step = max(st["steps"])

    def state(self):
        return {k: [t.clone() for t in v] if k != "steps" else list(v) for k, v in self.st.items()}

    def step(self, inp):
        b1, b2, mu = BETAS[0], BETAS[1], self.mutant
        counts = inp["counts"]
        g = []
        for i, c in enumerate(counts):
            if c == 0:
                g.append(None)
            elif c == 2 and mu == "no_divide_2":
                g.append(inp["gsum"][i].clone())
            else:
                g.append(inp["gsum"][i] / c)
        sq = [float(x.double().pow(2).sum()) for x in g if x is not None]
        total = f32(math.sqrt(sum(sq)))
        mean = f32(sum(f32(math.sqrt(s)) for s in sq) / len(sq)) if sq else 0.0
        coef = min(1.0, f32(f32(inp["max_norm"]) / f32(total + f32(1e-6))))
        if mu == "no_clip":
            coef = 1.0
        out = {"g": [], "metrics": [mean, f32(mean * coef), total, 0.0]}
        self.global_step += 1
        for i, c in enumerate(counts):
            if c == 0:
                out["g"].append(None)
                continue
            gc = g[i] * f32(coef)
            m = self.st["m"][i] + (gc - self.st["m"][i]) * f32(1.0 - b1)
            v = self.st["v"][i] * f32(b2) + f32(1.0 - b2) * gc * gc
            s = (self.global_step if mu == "global_step" else self.st["steps"][i] + 1) - (1 if mu == "bc_step" else 0)
            bc1, bc2 = 1.0 - b1 ** s, 1.0 - b2 ** s
            if mu == "eps_inside":
                denom = (v / f32(bc2) + f32(EPS)).sqrt()
            else:
                denom = v.sqrt() / f32(bc2 if mu == "bc2_no_sqrt" else math.sqrt(bc2)) + f32(EPS)
            self.st["p"][i] = self.st["p"][i] - f32(inp["lr"] / bc1) * (m / denom)
            self.st["m"][i], self.st["v"][i] = m, v
            self.st["steps"][i] += 1
            out["g"].append(gc)
        out.update(self.state())
        return out


# ------------------------------------------------------------------------------------------------ the bound
def _ratio_update(ratios, key, err, cal):
    r = err / cal if cal > 0 else (0.0 if err == 0 else float("inf"))
    ratios[key] = max(ratios.get(key, 0.0), r)


def bound_one(kind, got, ref, cal, ratios, failures, where):
    k, floor = BOUNDS[kind]
    err = float((got.double() - ref).abs().max())
    c = float((cal.double() - ref).abs().max())
    scale = float(ref.abs().max())
    _ratio_update(ratios, kind, err, c)
    if not err <= k * c + floor * scale:
        failures.append("%s %s: max|err| %.3e, torch fp32 %.3e, max|f64| %.3e" % (where, kind, err, c, scale))


def check_step(k, before, got, inp, ratios, failures):
    """Compares one finish step of ``got`` (from ``before``) with the float64 reference and the fp32 calibration."""
    ref, cal = step_f64(before, inp), step_torch32(before, inp)
    for j in range(3):
        bound_one("metrics", torch.tensor([got["metrics"][j]]), torch.tensor([ref["metrics"][j]], dtype=torch.float64),
                  torch.tensor([cal["metrics"][j]]), ratios, failures, "step %d metrics[%d]" % (k, j))
    if got["metrics"][3] != 0.0:
        failures.append("step %d: NaN flag %r" % (k, got["metrics"][3]))
    for i, c in enumerate(inp["counts"]):
        where = "step %d tensor %d (count %d)" % (k, i, c)
        if got["steps"][i] != ref["steps"][i]:
            failures.append("%s: step counter %d, want %d" % (where, got["steps"][i], ref["steps"][i]))
        if c == 0:
            for n in ("p", "m", "v"):
                if not torch.equal(got[n][i], before[n][i]):
                    failures.append("%s: %s changed without a gradient" % (where, n))
            continue
        bound_one("update", got["p"][i].double() - before["p"][i].double(), ref["p"][i] - before["p"][i].double(),
                  cal["p"][i].double() - before["p"][i].double(), ratios, failures, where)
        bound_one("exp_avg", got["m"][i], ref["m"][i], cal["m"][i], ratios, failures, where)
        bound_one("exp_avg_sq", got["v"][i], ref["v"][i], cal["v"][i], ratios, failures, where)
        bound_one("grad", got["g"][i], ref["g"][i], cal["g"][i], ratios, failures, where)


def run_trajectory(device, plan):
    ratios, failures = {}, []
    for k, inp in enumerate(plan):
        before = device.state()
        got = device.step(inp)
        failures += got.pop("failures", [])
        check_step(k, before, got, inp, ratios, failures)
    return ratios, failures


# ------------------------------------------------------------------------------------------------ CPU: the bound itself
def _cpu_layout():
    return Layout("cpu12", [1, 3, 63, 64, 65, 200, 1000, 50, 7, 4096, 17, 300], [-1, -1, 0, -1, 3, -1, VALUE_SLOT, -1,
                                                                              4, -1, -1, 1])


def _early_state(layout, seed):
    """Counters at 2 with the moments two steps leave: the bias corrections are far from 1."""
    st = make_state(layout, seed, resumed=True)
    st["steps"] = [2] * layout.n
    st["v"] = [v * 0.002 for v in st["v"]]
    return st


def test_bound_passes_fp32_and_rejects_host_mutants():
    """torch fp32 and an fp32 transcription of the finish pass the bound on every step; each mutant fails it."""
    lay = _cpu_layout()
    plan = make_plan(lay, 11)
    assert any(c == 2 for c in plan[0]["counts"]) and any(c == 3 for c in plan[0]["counts"])
    for st in (make_state(lay, 11, False), _early_state(lay, 11)):
        _, over = run_trajectory(HostFinish(st), plan)
        assert not over, over[:5]

        class Torch32:
            def __init__(self):
                self.st = st

            def state(self):
                return self.st

            def step(self, inp):
                out = step_torch32(self.st, inp)
                self.st = {n: out[n] for n in ("p", "m", "v", "steps")}
                return out
        _, over = run_trajectory(Torch32(), plan)
        assert not over, over[:5]
    for mutant in ("bc_step", "bc2_no_sqrt", "eps_inside", "no_clip", "no_divide_2", "global_step"):
        _, over = run_trajectory(HostFinish(_early_state(lay, 11), mutant), plan)
        assert over, "the %s mutant passed the bound" % mutant


def test_finish_rejects_too_many_segments():
    """n_seg = 97 (one more than kMaxSeg) and 0 are refused by both entry points and by dc_grad_flags before any launch."""
    from dotaclient_b200 import _lib, build
    build.build()
    lib = _lib.load()
    one = 4096                                       # any non-null pointer: validation fails before it is used
    for n_seg in (97, 0):
        assert lib.dc_grad_finish(one, one, one, one, one, one, one, one, n_seg, 1000, 1e-3, 0.9, 0.999, 1e-8, 0.5, None,
                                  one, one, None) == -1
        assert b"n_seg=%d" % n_seg in lib.dc_last_error()
        assert lib.dc_grad_finish_dev(one, one, one, one, one, one, one, one, n_seg, 1000, one, 0.9, 0.999, 1e-8, None,
                                      one, one, None) == -1
        assert lib.dc_grad_flags(one, 1000, one, n_seg, one, None) == -1
        assert b"dc_grad_flags" in lib.dc_last_error()


# ------------------------------------------------------------------------------------------------ GPU
class GpuFinish:
    """The flat buffers of one layout on the GPU, alignment padding filled with sentinels; ``step`` runs one finish
    through ``dc_grad_finish_dev`` (lr and max_norm written into the hyper-parameter block) or ``dc_grad_finish``."""

    def __init__(self, layout, st, entry="dev"):
        from dotaclient_b200 import _lib, ops
        self.ops, self.lay, self.entry = ops, layout, entry
        d = self.dev = torch.device("cuda", 0)
        T = layout.total
        self.pad = torch.ones(T, dtype=torch.bool)
        for a, b in zip(layout.lo, layout.hi):
            self.pad[a:b] = False
        self.buf = {}
        for n in ("p", "m", "v"):
            host = torch.full((T,), SENTINEL[n])
            for i, (a, b) in enumerate(zip(layout.lo, layout.hi)):
                host[a:b] = st[n][i]
            self.buf[n] = host.to(d)
        self.grad_full = torch.full((T + layout.n,), SENTINEL["g"], device=d)
        self.steps = torch.tensor(st["steps"], dtype=torch.int32, device=d)
        self.seg_lo = torch.tensor(layout.lo, dtype=torch.int64, device=d)
        self.seg_hi = torch.tensor(layout.hi, dtype=torch.int64, device=d)
        self.seg_head = torch.tensor(layout.heads, dtype=torch.int32, device=d)
        self.loss = torch.zeros(_lib.LOSS_SLOTS, device=d)
        self.metrics = torch.zeros(4, device=d)
        self.ws = torch.zeros(_lib.FINISH_WORKSPACE_BYTES, dtype=torch.uint8, device=d)

    def _segments(self, flat):
        return [flat[a:b].clone() for a, b in zip(self.lay.lo, self.lay.hi)]

    def state(self):
        return {"p": self._segments(self.buf["p"].cpu()), "m": self._segments(self.buf["m"].cpu()),
                "v": self._segments(self.buf["v"].cpu()), "steps": self.steps.cpu().tolist()}

    def load_grads(self, inp):
        host = torch.full((self.lay.total + self.lay.n,), SENTINEL["g"])
        for i, (a, b) in enumerate(zip(self.lay.lo, self.lay.hi)):
            host[a:b] = inp["gsum"][i]
        host[self.lay.total:] = torch.tensor(inp["counts"], dtype=torch.float32)
        self.grad_full.copy_(host)
        return host

    def launch(self, inp):
        ops, T = self.ops, self.lay.total
        args = (self.buf["p"], self.grad_full, self.buf["m"], self.buf["v"], self.steps, self.seg_lo, self.seg_hi,
                self.seg_head, T)
        if self.entry == "dev":
            hp = ops.hparam_block(self.dev, lr=inp["lr"], max_grad_norm=inp["max_norm"])
            ops.grad_finish(*args, 0.0, BETAS, EPS, 0.0, self.loss, self.metrics, self.ws, hparams=hp)
        else:
            ops.grad_finish(*args, inp["lr"], BETAS, EPS, inp["max_norm"], self.loss, self.metrics, self.ws)
        torch.cuda.synchronize()

    def step(self, inp):
        host = self.load_grads(inp)
        self.launch(inp)
        out = self.state()
        g = self.grad_full.cpu()
        out["g"] = [g[a:b].clone() if c > 0 else None for (a, b), c in zip(zip(self.lay.lo, self.lay.hi), inp["counts"])]
        out["metrics"] = self.metrics.cpu().tolist()
        fails = []
        for n in ("p", "m", "v"):
            if not bool((self.buf[n].cpu()[self.pad] == SENTINEL[n]).all()):
                fails.append("%s: alignment padding overwritten" % n)
        if not (torch.equal(g[:-self.lay.n][self.pad], host[:-self.lay.n][self.pad])
                and torch.equal(g[-self.lay.n:], host[-self.lay.n:])):
            fails.append("gradient padding or has-grad counts overwritten")
        for (a, b), c in zip(zip(self.lay.lo, self.lay.hi), inp["counts"]):
            if c == 0 and not torch.equal(g[a:b], host[a:b]):
                fails.append("gradient of a tensor without a count changed")
        out["failures"] = fails
        return out


LAYOUTS = [("lstm128", (128, "lstm", 1)), ("lstm256", (256, "lstm", 1)), ("lstm512", (512, "lstm", 1)),
           ("gru256", (256, "gru", 1)), ("lstm128-16layers", (128, "lstm", 16)), ("synthetic96", None)]


def _layout(spec):
    return synthetic_layout() if spec is None else policy_layout(*spec)


@pytest.mark.gpu
@pytest.mark.parametrize("resumed", [False, True], ids=["fresh", "resumed"])
@pytest.mark.parametrize("name,spec", LAYOUTS, ids=[n for n, _ in LAYOUTS])
def test_finish_trajectory_vs_fp64(name, spec, resumed):
    """8 finish steps through dc_grad_finish_dev with lr and max_norm changing between steps, every step within the
    bound of the float64 reference; counters exact; tensors without a count and the padding sentinels untouched."""
    lay = _layout(spec)
    if spec is not None and spec[2] == 16:
        assert lay.n == 94
    if spec is None:
        assert lay.n == 96 and max(lay.sizes()) > 1_000_000
    seed = lay.total % 1000 + (7 if resumed else 0)
    plan = make_plan(lay, seed)
    ratios, failures = run_trajectory(GpuFinish(lay, make_state(lay, seed, resumed)), plan)
    print("\n%s %s ratios: %s" % (name, "resumed" if resumed else "fresh", ", ".join("%s %.3g" % kv for kv in
                                                                                     ratios.items())))
    assert not failures, failures[:10]


@pytest.mark.gpu
def test_finish_scalar_entry_point_vs_fp64():
    """dc_grad_finish (lr and max_norm as arguments) on the 96-segment layout."""
    lay = synthetic_layout()
    plan = make_plan(lay, 5)
    ratios, failures = run_trajectory(GpuFinish(lay, make_state(lay, 5, False), entry="scalar"), plan)
    print("\nscalar entry ratios: %s" % ", ".join("%s %.3g" % kv for kv in ratios.items()))
    assert not failures, failures[:10]


@pytest.mark.gpu
def test_finish_nan_guard_leaves_the_state_untouched():
    """A NaN loss, or a NaN in one gradient element, sets metrics[3] and leaves parameters, moments and counters bit for
    bit unchanged; the next finite step runs."""
    lay = policy_layout(128, "lstm")
    plan = make_plan(lay, 3, n_steps=5)
    gpu = GpuFinish(lay, make_state(lay, 3, False))
    gpu.step(plan[0])
    for case in ("loss", "grad"):
        before = [t.clone() for t in (gpu.buf["p"], gpu.buf["m"], gpu.buf["v"], gpu.steps)]
        gpu.load_grads(plan[1])
        if case == "loss":
            gpu.loss[0] = float("nan")
        else:
            i = next(i for i, c in enumerate(plan[1]["counts"]) if c > 1)
            gpu.grad_full[lay.lo[i] + (lay.hi[i] - lay.lo[i]) // 2] = float("nan")
        gpu.launch(plan[1])
        gpu.loss.zero_()
        assert float(gpu.metrics[3]) == 1.0, case
        after = (gpu.buf["p"], gpu.buf["m"], gpu.buf["v"], gpu.steps)
        assert all(torch.equal(a, b) for a, b in zip(before, after)), case
    before = gpu.state()
    got = gpu.step(plan[1])
    assert got["metrics"][3] == 0.0 and got["steps"] != before["steps"]


@pytest.mark.gpu
def test_grad_flags_vs_host():
    """dc_grad_flags writes 1 for a tensor that needs no head or whose head (the value slot included) has action rows,
    else 0, into the n_seg slots after the gradient, and nothing else."""
    from dotaclient_b200 import ops
    d = torch.device("cuda", 0)
    for lay in (policy_layout(128, "lstm"), synthetic_layout()):
        seg_head = torch.tensor(lay.heads, dtype=torch.int32, device=d)
        body = torch.randn(lay.total, device=d)
        for pattern in ([1, 2, 3, 4, 5, 1], [0, 0, 0, 0, 0, 0], [3, 0, 7, 0, 1, 0], [0, 5, 0, 2, 0, 1],
                        [0, 0, 0, 0, 0, 1], [9, 9, 9, 9, 9, 0]):
            n_actions = torch.tensor(pattern + [0, 0], dtype=torch.int32, device=d)
            grad_full = torch.cat([body, torch.full((lay.n,), 7.0, device=d)])
            ops.grad_flags(grad_full, lay.total, seg_head, n_actions)
            want = [1.0 if h < 0 or pattern[h] > 0 else 0.0 for h in lay.heads]
            assert grad_full[lay.total:].cpu().tolist() == want, pattern
            assert torch.equal(grad_full[:lay.total], body)
