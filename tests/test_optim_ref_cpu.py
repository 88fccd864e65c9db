"""The float64 optimiser reference (oracle/optim_ref.py) and its error bounds, on the CPU.

  - in float64 the reference equals torch.optim.Adam / RMSprop (foreach=False, all four RMSprop variants) and
    torch.nn.utils.clip_grad_norm_, NaN total included, given the same fp32-rounded hyperparameters;
  - the fp32 torch specifications of the kernels (oracle/ops_emul*.py) stay within every bound on the cases of
    tests/test_gpu_optim_precision.py that fit on the CPU, and within the norm-wise bound of a 50-step trajectory;
  - every C-ABI entry point is held to a float64 or exact reference by a GPU test, or is on a short exempt list.
"""
import glob
import os
import re

import pytest
import torch

from oracle import optim_ref as R
from oracle.ops_emul_a2c import A2CEmulOps
from oracle.ops_emul_dv2 import DV2EmulOps
from sheeprl_b200 import lib as L

F32 = R.f32
LR, B1, B2, EPS = F32(1e-4), F32(0.9), F32(0.999), F32(1e-8)      # Dreamer-V3's Adam (configs/optim/adam.yaml)
RMS = dict(lr=F32(7e-4), alpha=F32(0.99), eps=F32(1e-5))           # A2C's RMSprop (configs/optim/rmsprop.yaml)
FAMILIES = ("normal", "uniform", "tiny", "huge")
STEPS = (1, 2, 10, 1000, 10 ** 6)
CLIPS = ("off", "below", "at", "above", "zero_grad")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------ inputs
def grads(n, family, gen):
    """N(0, 1); U(0.5, 1) with random signs; ~1e-20 (g*g underflows to fp32 subnormals); ~1e15 (g*g ~ 1e30)"""
    x = torch.randn(n, generator=gen)
    if family == "uniform":
        return (0.5 + 0.5 * torch.rand(n, generator=gen)) * torch.sign(x + (x == 0))
    return x * {"normal": 1.0, "tiny": 1e-20, "huge": 1e15}[family]


def state(n, gen, g=None):
    """p ~ N(0, 1); m, v as after a few hundred steps on gradients like g (v > 0)"""
    p = torch.randn(n, generator=gen)
    s = 1.0 if g is None else float(g.abs().max()) or 1.0
    m = 0.1 * s * torch.randn(n, generator=gen)
    v = (s * s) * (0.01 + torch.rand(n, generator=gen)) * 0.01
    return p, m, v


def max_norm_for(clip, normsq):
    """"off": 0 (no clipping); "below" the gradient norm; "at": the fp32 norm itself (coef within one ulp of 1);
    "above": far above; "zero_grad": a clipped all-zero gradient (total = 0, coef = 1)"""
    total = float(normsq) ** 0.5
    return {"off": 0.0, "below": F32(0.3 * total), "at": F32(total), "above": F32(1e3 * total + 1),
            "zero_grad": 1.0}[clip]


def _assert_within(name, got, want, bound, factor=1.0):
    """|got - want| <= factor * bound on the finite elements; the non-finite ones must coincide"""
    got, want, bound = got.double(), want.double(), bound.double()
    fin = torch.isfinite(want)
    assert torch.equal(torch.isnan(got), torch.isnan(want)), (name, "NaN positions")
    assert torch.equal(got[torch.isinf(want)], want[torch.isinf(want)]), (name, "inf")
    err = (got[fin] - want[fin]).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / (factor * bound[fin]))
    assert bool((err <= factor * bound[fin]).all()), (name, float(ratio.max()))
    return float(ratio.max()) if ratio.numel() else 0.0


# ------------------------------------------------------------------------------------------------- against torch
def _torch_adam(p, g, m, v, t, max_norm, wd):
    P = torch.nn.Parameter(p.double().clone())
    P.grad = g.double().clone()
    if max_norm > 0:
        torch.nn.utils.clip_grad_norm_([P], max_norm, error_if_nonfinite=False)
    opt = torch.optim.Adam([P], lr=LR, betas=(B1, B2), eps=EPS, weight_decay=wd, foreach=False)
    opt.state[P] = {"step": torch.tensor(float(t - 1)), "exp_avg": m.double().clone(), "exp_avg_sq": v.double().clone()}
    opt.step()
    return P.detach(), opt.state[P]["exp_avg"], opt.state[P]["exp_avg_sq"]


def _close64(name, a, b):
    a, b = a.double(), b.double()
    assert torch.equal(torch.isnan(a), torch.isnan(b)), name
    f = torch.isfinite(b)
    err = (a[f] - b[f]).abs()
    assert bool((err <= 1e-12 * (b[f].abs() + b[f].abs().max())).all()), (name, float(err.max()))


@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("clip", ["off", "below", "at", "above"])
@pytest.mark.parametrize("t", STEPS)
def test_adam_reference_equals_torch_in_float64(wd, clip, t):
    gen = torch.Generator().manual_seed(t + 7)
    g = grads(1003, "normal", gen)
    p, m, v = state(1003, gen)
    normsq = R.sumsq64(g)
    mn = max_norm_for(clip, normsq)
    want = _torch_adam(p, g, m, v, t, mn, F32(wd))
    got = R.adam_step64(p, g, m, v, normsq, t, mn, LR, B1, B2, EPS, F32(wd))
    for k, w in zip(("p", "m", "v"), want):
        _close64(k, got[k], w)


@pytest.mark.parametrize("centered", [False, True])
@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("clip", ["off", "below"])
def test_rmsprop_reference_equals_torch_in_float64(centered, momentum, wd, clip):
    gen = torch.Generator().manual_seed(int(centered) + 2 * int(momentum > 0) + 5)
    n = 1003
    g = grads(n, "normal", gen)
    p = torch.randn(n, generator=gen)
    sq = 1.5 * (0.1 + torch.rand(n, generator=gen))
    ga = 0.3 * torch.randn(n, generator=gen) if centered else None
    buf = 0.1 * torch.randn(n, generator=gen) if momentum else None
    normsq = R.sumsq64(g)
    mn = max_norm_for(clip, normsq)
    P = torch.nn.Parameter(p.double().clone())
    P.grad = g.double().clone()
    if mn > 0:
        torch.nn.utils.clip_grad_norm_([P], mn)
    opt = torch.optim.RMSprop([P], **RMS, weight_decay=F32(wd), momentum=F32(momentum), centered=centered,
                              foreach=False)
    st = {"step": torch.tensor(0.0), "square_avg": sq.double().clone()}
    if momentum:
        st["momentum_buffer"] = buf.double().clone()
    if centered:
        st["grad_avg"] = ga.double().clone()
    opt.state[P] = st
    opt.step()
    got = R.rmsprop_step64(p, g, sq, normsq, mn, **RMS, weight_decay=F32(wd), momentum=F32(momentum), momentum_buf=buf,
                           grad_avg=ga)
    _close64("p", got["p"], P.detach())
    _close64("square_avg", got["sq"], st["square_avg"])
    if momentum:
        _close64("momentum_buffer", got["buf"], st["momentum_buffer"])
    if centered:
        _close64("grad_avg", got["gavg"], st["grad_avg"])


@pytest.mark.parametrize("case", ["below", "at", "above", "nan", "inf", "zero"])
def test_clip_coefficient_equals_clip_grad_norm(case):
    g = grads(4099, "normal", torch.Generator().manual_seed(3)).double()
    if case == "nan":
        g[17] = float("nan")
    elif case == "inf":
        g[17] = float("inf")
    elif case == "zero":
        g.zero_()
    normsq = float((g * g).sum())
    mn = {"below": 3.0, "at": normsq ** 0.5, "above": 1e6}.get(case, 3.0)
    P = torch.nn.Parameter(torch.zeros_like(g))
    P.grad = g.clone()
    total = torch.nn.utils.clip_grad_norm_([P], mn, error_if_nonfinite=False)
    coef, tot = R.clip_coef64(normsq, mn)
    assert torch.equal(tot.isnan(), total.isnan())
    assert bool(tot.isnan()) or float(tot) == pytest.approx(float(total), rel=1e-14)
    clipped = P.grad
    if case == "nan":
        assert bool(coef.isnan()) and bool(clipped.isnan().all())
    elif case == "inf":
        assert float(coef) == 0.0 and bool(clipped[17].isnan()) and not bool(clipped[:17].any())
    else:
        assert float(coef) <= 1.0
        _close64("clipped", g * coef, clipped)
    assert float(R.clip_coef64(normsq, 0.0)[0]) == 1.0                  # max_norm 0: no clipping, NaN or not


def test_fp32_betas_gap_is_the_known_one():
    """the ABI passes betas as float: 1 - 0.999f is 1.3e-5 off 0.001 (relative); the reference takes the fp32 value, so
    this gap is outside every bound and is the only difference from torch's double betas"""
    assert abs((1 - R.f32(0.999)) / 0.001 - 1) == pytest.approx(1.29e-5, rel=0.01)
    assert 1 - R.f32(0.9) == pytest.approx(0.1, rel=3e-7)


# ------------------------------------------------------------------------------------ the fp32 specification fits
def _emul_adam(p, g, m, v, normsq, t, mn, wd):
    p, m, v, out = p.clone(), m.clone(), v.clone(), torch.zeros(1)
    DV2EmulOps().adam_step(p, g, m, v, torch.tensor(normsq, dtype=torch.float64), mn, LR, B1, B2, EPS,
                           torch.tensor([t], dtype=torch.int32), out, weight_decay=wd)
    return p, m, v, out


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("clip", CLIPS)
@pytest.mark.parametrize("t", STEPS)
@pytest.mark.parametrize("wd", [0.0, 0.1])
def test_emulator_adam_within_bounds(family, clip, t, wd):
    gen = torch.Generator().manual_seed(FAMILIES.index(family) * 100 + t % 97)
    g = grads(4099, family, gen)
    if clip == "zero_grad":
        g.zero_()
    p, m, v = state(4099, gen, g)
    normsq = R.sumsq64(g)
    mn = max_norm_for(clip, normsq)
    ref = R.adam_step64(p, g, m, v, normsq, t, mn, LR, B1, B2, EPS, F32(wd))
    ep, em_, ev, out = _emul_adam(p, g, m, v, normsq, t, mn, F32(wd))
    for k, got in (("p", ep), ("m", em_), ("v", ev)):
        _assert_within(k, got, ref[k], ref["err_" + k])
    assert float(out) == float(ref["total"].float())


@pytest.mark.parametrize("centered", [False, True])
@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("clip", ["off", "below", "at"])
def test_emulator_rmsprop_within_bounds(centered, momentum, wd, family, clip):
    gen = torch.Generator().manual_seed(FAMILIES.index(family) + 11)
    n = 4099
    g = grads(n, family, gen)
    s = float(g.abs().max())
    p = torch.randn(n, generator=gen)
    sq = s * s * (0.5 + torch.rand(n, generator=gen))
    ga = 0.3 * s * torch.randn(n, generator=gen) if centered else None
    buf = 0.1 * torch.randn(n, generator=gen) if momentum else None
    normsq = R.sumsq64(g)
    mn = max_norm_for(clip, normsq)
    kw = dict(**RMS, weight_decay=F32(wd), momentum=F32(momentum))
    ref = R.rmsprop_step64(p, g, sq, normsq, mn, momentum_buf=buf, grad_avg=ga, **kw)
    e = [t.clone() if t is not None else None for t in (p, sq, buf, ga)]
    A2CEmulOps().rmsprop_step(e[0], g, e[1], e[2], e[3], torch.tensor(normsq, dtype=torch.float64), mn, kw["lr"],
                              kw["alpha"], kw["eps"], kw["weight_decay"], kw["momentum"], torch.zeros(1))
    _assert_within("p", e[0], ref["p"], ref["err_p"])
    _assert_within("sq", e[1], ref["sq"], ref["err_sq"])
    if momentum:
        _assert_within("buf", e[2], ref["buf"], ref["err_buf"])
    if centered:
        _assert_within("gavg", e[3], ref["gavg"], ref["err_gavg"])


@pytest.mark.parametrize("tau", [1.0, 0.02, 0.005])
def test_emulator_ema_within_bounds(tau):
    gen = torch.Generator().manual_seed(5)
    t, s = torch.randn(4099, generator=gen), torch.randn(4099, generator=gen) * 3
    want, bound = R.ema64(t, s, F32(tau))
    got = t.clone()
    DV2EmulOps().ema(got, s, F32(tau))
    _assert_within("ema", got, want, bound)


def test_emulator_adam_trajectory_within_norm_bound():
    """50 chained fp32 steps against 50 float64 steps from the same start, held norm-wise to twice the sum of the
    per-step bounds along the float64 trajectory (each step's own rounding of p, of order u |p|, dominates: an error
    carried in m or v is damped by b1 or b2 every step)"""
    gen = torch.Generator().manual_seed(9)
    n, T = 4099, 50
    p, m, v = torch.randn(n, generator=gen), torch.zeros(n), torch.zeros(n)
    P, M, V = p.double(), m.double(), v.double()
    tol = {"p": 0.0, "m": 0.0, "v": 0.0}
    for k in range(T):
        g = grads(n, "normal", gen) * (1 + 0.1 * k)
        normsq = R.sumsq64(g)
        p, m, v, _ = _emul_adam(p, g, m, v, normsq, k + 1, F32(10.0), F32(0.01))
        r = R.adam_step64(P, g, M, V, normsq, k + 1, F32(10.0), LR, B1, B2, EPS, F32(0.01))
        P, M, V = r["p"], r["m"], r["v"]
        for key in tol:
            tol[key] += float(r["err_" + key].norm())
    for key, got, want in (("p", p, P), ("m", m, M), ("v", v, V)):
        assert float((got.double() - want).norm()) <= 2 * tol[key], key


def test_sumsq_reference_is_exact():
    """the sum of squares is the exact sum rounded once to double, at magnitudes that a plain double sum would lose"""
    from fractions import Fraction

    x = torch.cat([torch.randn(997, generator=torch.Generator().manual_seed(1)) * 10.0 ** torch.arange(997).remainder(9),
                   torch.tensor([2.0 ** 40, 1.0, -(2.0 ** 40), 2.0 ** -30])])
    assert R.sumsq64(x) == float(sum(Fraction(float(v)) ** 2 for v in x))


# ------------------------------------------------------------------------------------------------- inventory guard
# Entry points that need no float64 check, with the reason.  Suffix / prefix rules cover the families of queries.
EXEMPT_RULES = (
    (r"_supported$|_check$|_route$", "routing / envelope query: answers from its arguments, checked by the launch-refusal"
                                     " tests and tests/test_lib_cpu.py"),
    (r"_workspace$|_workspace_bytes$|_floats$", "workspace size: an integer the launches check before running"),
    (r"^b200rl_(set|get)_", "process-wide mode switch: the precision and deterministic suites run in both modes"),
)
EXEMPT = {
    "b200rl_last_error": "returns the thread's last error message",
    "b200rl_abi_version": "a constant (tests/test_lib_cpu.py)",
    "b200rl_build_arch": "a constant string (tests/test_lib_cpu.py)",
    "b200rl_device_check": "refuses devices other than sm_90a; computes nothing",
    "b200rl_zero": "cudaMemsetAsync of zeros",
    "b200rl_increment": "integer step counter += 1",
    "b200rl_rssm_scan_error": "diagnostic: reads the scan's error word",
    "b200rl_rssm_scan_profile": "diagnostic: cycle counters of the last scan launch",
    "b200rl_deterministic_pool_fill": "diagnostic: fills the deterministic-mode slot pool for the NaN-poisoning tests",
}
# GPU suites whose checks compare against a float64 reference or an exact result (tests/test_gpu_ops.py compares most
# kernels with the fp32 emulator only and does not count).
REFERENCE_SUITES = sorted(glob.glob(os.path.join(ROOT, "tests", "test_gpu_*precision.py"))) + [
    os.path.join(ROOT, "tests", f) for f in (
        "test_gpu_rssm_scan.py",          # persistent RSSM scan against oracle/rssm_scan_ref.py
        "test_gpu_dv3_decoupled.py",      # GRU-only scan against oracle/gru_scan_ref.py
        "test_gpu_deterministic.py",      # fixed-order reductions against the float64 references
        "test_gpu_droq.py",               # dropout masks bit-exact, dropout-LayerNorm-ReLU against float64
        "test_gpu_minedojo.py",           # masked sampling against a float64 specification
        "test_gpu_tc_presplit.py",        # presplit routes bit-identical to the float64-checked tensor-core routes
        "test_gpu_buffers.py",            # replay gather / scatter: exact copies
    )]


def _wrappers():
    """entry point -> names of the CudaOps methods (sheeprl_b200/lib.py) that call it"""
    src = open(L.__file__).read()
    out = {}
    for m in re.finditer(r"\n    def (\w+)\(.*?(?=\n    def |\nclass |\Z)", src, re.S):
        for e in re.findall(r"\b(b200rl_\w+)\b", m.group(0)):
            out.setdefault(e, set()).add(m.group(1))
    return out


def test_every_entry_point_has_a_float64_or_exact_check():
    """an entry point counts as checked when a reference suite names it, or calls a CudaOps method that wraps it"""
    with open(L.HEADER_PATH) as f:
        header = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(b200rl_\w+)\s*\(", header)))
    assert set(EXEMPT) <= set(names), set(EXEMPT) - set(names)
    suites = [open(p).read() for p in REFERENCE_SUITES if os.path.exists(p)]
    wrap = _wrappers()
    missing = []
    for n in names:
        if n in EXEMPT or any(re.search(r, n) for r, _ in EXEMPT_RULES):
            continue
        pats = [r"\b" + n + r"\b"] + [r"\." + w + r"\(" for w in wrap.get(n, ())]
        if not any(re.search(pt, s) for pt in pats for s in suites):
            missing.append(n)
    assert not missing, f"entry points without a float64 or exact GPU check: {missing}"
