"""The float64 LayerNorm reference (oracle/ln_ref.py) and its error bounds, on the CPU.

  - the float64 forward and backward agree with torch autograd on float64 F.layer_norm + activation;
  - an honest fp32 implementation (EmulOps, the kernels' specification) stays within every bound with 2x headroom at
    each GPU case shape that fits on the CPU (the cases of tests/test_gpu_ln_precision.py are defined here);
  - fp32 implementations with one subtle defect each exceed the bound by at least 4x: the bounds are tight enough to
    catch the bugs a LayerNorm kernel is known to have.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import ln_ref
from oracle.ops_emul import EmulOps

EPS = (1e-3, 1e-5)                 # Dreamer-V3; PPO / SAC / DroQ
LN_FAMILIES = ("centred", "offset", "flat", "constant")
CHUNK = 1 << 22                    # elements per float64 reference chunk


# ------------------------------------------------------------------------------------------------------------ inputs
def family_rows(M, C, family, eps, gen, device):
    """centred N(0, 2^2); offset m_r + N(0, 1) with row means m_r in [500, 1500] (mean ~1000 sigma); flat m_r +
    N(0, f_r^2 eps) with f_r in [0.3, 1] (variance ~eps); constant rows of multiples of 1/64 (exact row sums, so the
    exact output is beta)."""
    n = torch.randn(M, C, generator=gen, device=device)
    r = torch.rand(M, 1, generator=gen, device=device)
    if family == "centred":
        return 2.0 * n
    if family == "offset":
        return 1000.0 * (0.5 + r) + n
    if family == "flat":
        return 0.5 * torch.randn(M, 1, generator=gen, device=device) + (0.3 + 0.7 * r) * math.sqrt(eps) * n
    assert family == "constant", family
    return (torch.randn(M, 1, generator=gen, device=device) * 128.0).round().div(64.0).expand(M, C).contiguous()


def chunks(M, C):
    step = max(1, CHUNK // max(C, 1))
    return [(r, min(M, r + step)) for r in range(0, M, step)]


def ln_inputs(M, C, family, eps, act, seed, device="cpu"):
    """(X, gamma, beta, dY): gamma = 1 + 0.3 N(0, 1), beta = 0.2 N(0, 1), dY = N(0, 1).  ReLU: rows are redrawn until no
    float64 LayerNorm output lies within 10x its forward bound of 0, so a flipped gate is a bug, not rounding."""
    gen = torch.Generator(device=device).manual_seed(seed)
    gamma = 1.0 + 0.3 * torch.randn(C, generator=gen, device=device)
    beta = 0.2 * torch.randn(C, generator=gen, device=device)
    X = family_rows(M, C, family, eps, gen, device)
    dY = torch.randn(M, C, generator=gen, device=device)
    if act == 3:
        for _ in range(100):
            bad = torch.cat([near_gate(X[a:b], gamma, beta, eps) for a, b in chunks(M, C)])
            nb = int(bad.sum())
            if nb == 0:
                break
            X[bad] = family_rows(nb, C, family, eps, gen, device)
        else:
            raise AssertionError("could not draw ReLU rows away from the gate")
    return X, gamma, beta, dY


def near_gate(X, gamma, beta, eps):
    _, _, _, xh = ln_ref.ln_act_fwd64(X, gamma, beta, eps, 0)
    ln = xh * gamma.double() + beta.double()
    return (ln.abs() <= 10 * ln_ref.ln_act_fwd_bound(X, gamma, beta, eps, 0, ln)).any(-1)


# ------------------------------------------------------------------------------------------------------------ cases
# rows per warp of the register-resident kernels (32 / lanes per row)
VEC_RPW = {32: 4, 48: 8, 64: 2, 96: 4, 128: 1, 192: 2, 256: 1, 384: 1, 512: 1, 640: 1, 768: 1, 1024: 1, 1536: 1}
GRID_ROWS = 132 * 8 * 8            # warps of one full grid of the vec / generic kernels (x rows per warp)
LAYOUTS = ("plain", "alias", "accumulate", "noparam", "strided")


def _cases():
    """case id -> (route, C, M, act, eps, family, layout).  Act, eps, family and layout cycle within each route, so every
    route meets each of them.  ReLU takes centred rows only: the other families' forward bounds (mean ~1000, rstd up
    to 1 / sqrt(eps)) put too many outputs within 10x of the gate to redraw them away."""
    shapes = {1: [], 2: [], 0: []}
    for C, rpw in VEC_RPW.items():
        shapes[1] += [(C, 1), (C, 37 * rpw + 1), (C, 2 * GRID_ROWS * rpw + 3)]
    shapes[1] += [(32, 1 << 20), (64, 1 << 20)]                       # the conv stacks' row counts
    shapes[2] += [(C, M) for C in (1540, 3072, 12288, 16384) for M in (1, 64, 4 * 132 + 5)]
    shapes[0] += [(C, 300 if C > 4096 else 2500) for C in (1, 3, 31, 33, 100, 255, 513, 1000, 1537, 2050, 16388, 20000)]
    shapes[0] += [(256, 999, "ld_odd"), (256, 999, "offset"), (3072, 77, "ld_odd"), (3072, 77, "offset")]
    out = {}
    for route, lst in shapes.items():
        for k, s in enumerate(lst):
            C, M = s[:2]
            act, fam = k % 4, LN_FAMILIES[(k + k // 4) % 4]
            if act == 3:
                fam = "centred"
            layout = s[2] if len(s) > 2 else LAYOUTS[k % len(LAYOUTS)]
            out[f"r{route}_C{C}_M{M}_act{act}_{fam}_{layout}"] = (route, C, M, act, EPS[(k // 2) % 2], fam, layout)
    return out


LN_CASES = _cases()
# the once-seen failure of tests/test_gpu_ops.py::test_ln_act_tanh_relu[2-1000-32], with that test's exact inputs
FLAKE_SHAPE = (1000, 32, 2, 1e-5)


def flake_inputs():
    M, C, _, _ = FLAKE_SHAPE

    def rnd(*shape, seed):
        return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))

    return rnd(M, C, seed=1) * 2.0, rnd(C, seed=101) + 1.0, rnd(C, seed=201), rnd(M, C, seed=301)


# ------------------------------------------------------------------------------------------------------------ metrics
def ratio(got, ref, bound):
    """max |got - ref| / bound; an element whose bound is 0 must be exact; NaN counts as infinitely wrong"""
    d = (got.double() - ref).abs()
    r = torch.where(d == 0, torch.zeros_like(d), d / bound)
    return float("inf") if bool(r.isnan().any()) else float(r.max()) if r.numel() else 0.0


def margins(X, gamma, beta, eps, act, dY, Y, dX, dgamma=None, dbeta=None, prior_g=None, prior_b=None):
    """{"y", "dX", "dgamma", "dbeta"}: worst error / bound of an fp32 result, the float64 reference and its bounds computed
    in row chunks (dgamma / dbeta: their sums over the chunks).  prior_*: the values the gradients were added to."""
    M, C = X.shape
    out = {"y": 0.0, "dX": 0.0}
    dev = X.device
    sums = [torch.zeros(C, dtype=torch.float64, device=dev) for _ in range(6)]
    for a, b in chunks(M, C):
        x, dy = X[a:b], dY[a:b]
        y64, *_ = ln_ref.ln_act_fwd64(x, gamma, beta, eps, act)
        out["y"] = max(out["y"], ratio(Y[a:b], y64, ln_ref.ln_act_fwd_bound(x, gamma, beta, eps, act, y64)))
        del y64
        dx64, dg64, db64, mag = ln_ref.ln_act_bwd64(x, gamma, beta, eps, act, dy)
        b_dx, p_g, p_b = ln_ref.ln_act_bwd_bound(x, gamma, beta, eps, act, dy)
        out["dX"] = max(out["dX"], ratio(dX[a:b], dx64, b_dx))
        del dx64, b_dx
        for s, v in zip(sums, (dg64, db64, mag["dgamma"], mag["dbeta"], p_g, p_b)):
            s += v
    dg64, db64, mg, mb, p_g, p_b = sums
    if prior_g is not None:
        dg64, db64 = dg64 + prior_g.double(), db64 + prior_b.double()
    if dgamma is not None:
        out["dgamma"] = ratio(dgamma, dg64, ln_ref.param_bound(M, mg, p_g, prior_g))
        out["dbeta"] = ratio(dbeta, db64, ln_ref.param_bound(M, mb, p_b, prior_b))
    return out


def emul_margins(X, gamma, beta, eps, act, dY):
    em = EmulOps()
    M, C = X.shape
    Y, dX, dg, db = torch.empty(M, C), torch.empty(M, C), torch.empty(C), torch.empty(C)
    em.ln_act_fwd(X, gamma, beta, eps, act, Y)
    em.ln_act_bwd(X, gamma, beta, eps, act, dY, dX, dg, db)
    return margins(X, gamma, beta, eps, act, dY, Y, dX, dg, db)


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_float64_reference_matches_autograd(act):
    g = torch.Generator().manual_seed(act)
    M, C, eps = 9, 37, 1e-3
    X = (torch.randn(M, C, generator=g, dtype=torch.float64) * 2 + 0.5).requires_grad_(True)
    gamma = (1 + 0.3 * torch.randn(C, generator=g, dtype=torch.float64)).requires_grad_(True)
    beta = (0.2 * torch.randn(C, generator=g, dtype=torch.float64)).requires_grad_(True)
    dY = torch.randn(M, C, generator=g, dtype=torch.float64)
    ln = F.layer_norm(X, (C,), gamma, beta, eps)
    y = {0: ln, 1: F.silu(ln), 2: torch.tanh(ln), 3: torch.relu(ln)}[act]
    y.backward(dY)
    y64, mu, rstd, xh = ln_ref.ln_act_fwd64(X, gamma, beta, eps, act)
    dx64, dg64, db64, mag = ln_ref.ln_act_bwd64(X, gamma, beta, eps, act, dY)
    for got, want in ((y64, y), (dx64, X.grad), (dg64, gamma.grad), (db64, beta.grad),
                      (mu.squeeze(1), X.mean(1)), (rstd.squeeze(1), (X.var(1, unbiased=False) + eps).rsqrt())):
        assert float((got - want.detach()).abs().max()) <= 1e-12 * (1 + float(want.abs().max()))
    assert bool((mag["dbeta"] >= db64.abs()).all()) and bool((mag["dgamma"] >= dg64.abs()).all())
    s, sa = ln_ref.col_sum64(dY)
    assert torch.allclose(s, dY.sum(0), rtol=0, atol=1e-12) and torch.equal(sa, dY.abs().sum(0))


def test_gather_reference_matches_the_dense_product():
    g = torch.Generator().manual_seed(0)
    M, S, K, A, N = 5, 3, 4, 2, 8
    z = F.one_hot(torch.randint(0, K, (M, S), generator=g), K).float().reshape(M, S * K)
    act, WT = torch.randn(M, A, generator=g), torch.randn(S * K + A, N, generator=g)
    pre, mag = ln_ref.gather64(z, act, WT, S, K)
    x = torch.cat([z, act], 1).double()
    assert torch.allclose(pre, x @ WT.double(), rtol=0, atol=1e-12)
    assert torch.allclose(mag, x.abs() @ WT.double().abs(), rtol=0, atol=1e-12)


CPU_CASES = [c for c, (_, C, M, *_) in LN_CASES.items() if M * C <= 1 << 20]


@pytest.mark.parametrize("case", CPU_CASES)
def test_emulator_is_within_the_bounds(case):
    """the fp32 specification at the GPU case's shape, act, eps and family: every bound with 2x headroom"""
    _, C, M, act, eps, fam, _ = LN_CASES[case]
    X, gamma, beta, dY = ln_inputs(M, C, fam, eps, act, seed=len(case))
    m = emul_margins(X, gamma, beta, eps, act, dY)
    assert max(m.values()) <= 0.5, m


def test_emulator_at_the_once_failed_shape():
    M, C, act, eps = FLAKE_SHAPE
    X, gamma, beta, dY = flake_inputs()
    m = emul_margins(X, gamma, beta, eps, act, dY)
    assert max(m.values()) <= 0.5, m


# ------------------------------------------------------------------------------------------------------------ mutants
def fp32_ln(X, gamma, beta, eps, act, dY, mutant=None):
    """EmulOps's fp32 forward / backward written out, with one defect switched on by `mutant`"""
    C = X.shape[-1]
    mu = X.mean(-1, keepdim=True)
    if mutant == "one_pass_variance":
        var = (X * X).mean(-1, keepdim=True) - mu * mu
    else:
        var = ((X - mu) ** 2).mean(-1, keepdim=True)
    rstd = torch.rsqrt(var) if mutant == "no_eps" else torch.rsqrt(var + eps)
    if mutant == "rstd_1e-4":
        rstd = rstd * (1 + 1e-4)
    xh = (X - mu) * rstd
    ln = xh * gamma + beta
    Y = {0: ln, 1: F.silu(ln), 2: torch.tanh(ln), 3: torch.relu(ln)}[act]
    at = F.silu(ln) if mutant == "silu_prime_at_output" else ln
    if act == 1:
        s = torch.sigmoid(at)
        dln = dY * (s * (1 + at * (1 - s)))
    elif act == 2:
        dln = dY * (1 - torch.tanh(at) ** 2)
    elif act == 3:
        dln = dY * (at > 0).float()
    else:
        dln = dY.clone()
    rows = dln[:-1] if mutant == "drop_last_row_group" else dln
    dg, db = (rows * xh[:rows.shape[0]]).sum(0), rows.sum(0)
    dxh = dln * gamma
    n1 = C - 1 if mutant == "mean_gg_over_C_minus_1" else C
    n2 = C - 1 if mutant == "mean_ggxh_over_C_minus_1" else C
    dX = rstd * (dxh - dxh.sum(-1, keepdim=True) / n1 - xh * (dxh * xh).sum(-1, keepdim=True) / n2)
    return Y, dX, dg, db


# mutant -> (M, C, family, eps, act, outputs that must reject it)
MUTANTS = {
    "one_pass_variance": (64, 256, "offset", 1e-3, 0, ("y",)),
    "no_eps": (64, 64, "flat", 1e-3, 0, ("y",)),
    "mean_gg_over_C_minus_1": (64, 1024, "centred", 1e-3, 0, ("dX",)),
    "mean_ggxh_over_C_minus_1": (64, 1024, "centred", 1e-3, 0, ("dX",)),
    "drop_last_row_group": (1001, 32, "centred", 1e-5, 0, ("dgamma", "dbeta")),
    "silu_prime_at_output": (64, 128, "centred", 1e-3, 1, ("dX", "dgamma", "dbeta")),
    "rstd_1e-4": (64, 64, "centred", 1e-3, 0, ("y",)),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_bounds_reject_subtly_wrong_implementations(mutant):
    M, C, fam, eps, act, rejected = MUTANTS[mutant]
    X, gamma, beta, dY = ln_inputs(M, C, fam, eps, act, seed=7)
    honest = margins(X, gamma, beta, eps, act, dY, *fp32_ln(X, gamma, beta, eps, act, dY))
    assert max(honest.values()) <= 0.5, honest
    wrong = margins(X, gamma, beta, eps, act, dY, *fp32_ln(X, gamma, beta, eps, act, dY, mutant))
    for k in rejected:
        assert wrong[k] >= 4.0, (k, wrong)
