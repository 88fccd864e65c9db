"""The optimiser kernels (csrc/optim.cu: `b200rl_adam_step`, `b200rl_adam_step_wd`, `b200rl_rmsprop_step`,
`b200rl_ema`, `b200rl_sumsq`) and the element-wise / data-movement entry points (`b200rl_copy2d`, `b200rl_axpy`,
`b200rl_affine`, `b200rl_symlog`, `b200rl_tanh_fwd`, `b200rl_tanh_bwd`, csrc/conv.cu: `b200rl_obs_prep`,
`b200rl_transpose_batched`, `b200rl_transpose2d`, csrc/ppo.cu: `b200rl_im2col`, `b200rl_col2im`) against float64
references (oracle/optim_ref.py and the expressions below) with first-order per-element bounds, or bit for bit where
the operation moves data only.

Every optimiser step starts from the kernel's own previous state, so each step is a one-step error check against its
bound; a 50-step trajectory is held norm-wise.  Views sit between guard floats that must stay untouched, at a 16-byte
aligned base (float4 body + scalar tail) and one float off it (scalar path only).  The largest error / bound ratio of
each output is printed at the end of the module."""
import math

import pytest
import torch

from oracle import optim_ref as R
from oracle.simt_ref import U
from tests.test_optim_ref_cpu import (B1, B2, CLIPS, EPS, F32, FAMILIES, LR, RMS, STEPS, _assert_within, grads,
                                      max_norm_for, state)

pytestmark = pytest.mark.gpu

ONE_PASS = 132 * 8 * 256 * 4        # floats one vectorised grid-stride pass covers (stream_grid's cap of 132*8 CTAs)
SHAPES = [1, 2, 3, 5, 1003, 4096, ONE_PASS + 7, 5_000_003]
GUARD = 8
FILL = 7.0
RATIOS = {}


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    ops = CudaOps()
    yield ops
    if RATIOS:
        print("\nlargest error / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(RATIOS.items())))


def within(name, got, want, bound):
    r = _assert_within(name, got, want, bound)
    RATIOS[name] = max(RATIOS.get(name, 0.0), r)


def guarded(x, offset=0):
    """(buffer, view): x on the device inside GUARD floats of FILL on each side; offset 1 misaligns the view"""
    n = x.numel()
    buf = torch.full((n + 2 * GUARD + offset,), FILL, device="cuda")
    view = buf[GUARD + offset:GUARD + offset + n]
    view.copy_(x)
    return buf, view


def assert_guards(buf, n, offset=0):
    assert bool((buf[:GUARD + offset] == FILL).all()) and bool((buf[GUARD + offset + n:] == FILL).all()), "guard"


def d(t):
    return t.detach().to(device="cuda", dtype=torch.float64)


# ------------------------------------------------------------------------------------------------------- Adam
def run_adam(cu, n, offset, family, clip, t, wd, steps=2, seed=0, nan_at=None, inf_at=None):
    gen = torch.Generator().manual_seed(seed)
    g = grads(n, family, gen)
    p, m, v = state(n, gen, g)
    bufs = {k: guarded(x, offset) for k, x in (("p", p), ("m", m), ("v", v), ("g", g))}
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    normsq, out = torch.zeros((), dtype=torch.float64, device="cuda"), torch.zeros(1, device="cuda")
    name = "adam_wd" if wd else "adam"
    for s in range(steps):
        if s:
            g = grads(n, family, gen)
        if clip == "zero_grad":
            g = torch.zeros(n)
        if nan_at is not None:
            g[nan_at] = float("nan")
        if inf_at is not None:
            g[inf_at] = float("inf")
        bufs["g"][1].copy_(g)
        ns = R.sumsq64(g)
        normsq.fill_(ns)
        mn = max_norm_for(clip, ns if math.isfinite(ns) else 1.0)
        cur = {k: d(bufs[k][1]) for k in "pmv"}
        ref = R.adam_step64(cur["p"], d(g), cur["m"], cur["v"], ns, t + s, mn, LR, B1, B2, EPS, F32(wd))
        step.fill_(t + s)
        cu.adam_step(bufs["p"][1], bufs["g"][1], bufs["m"][1], bufs["v"][1], normsq, mn, LR, B1, B2, EPS, step, out,
                     weight_decay=F32(wd))
        for k in "pmv":
            within(f"{name} {k}", bufs[k][1], ref[k], ref["err_" + k])
        tot = float(ref["total"].float())
        assert float(out) == tot or (math.isnan(tot) and math.isnan(float(out))), "norm_out"
    for k, (buf, _) in bufs.items():
        assert_guards(buf, n, offset)
    return {k: bufs[k][1] for k in "pmv"}


@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("n", SHAPES)
def test_adam_shapes(cu, n, offset, wd):
    """n = 1 (SAC / DroQ's log_alpha), every float4 tail length, one grid-stride pass + 7, several passes"""
    run_adam(cu, n, offset, "normal", "below", 10, wd, seed=n + offset)


@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("t", STEPS)
@pytest.mark.parametrize("clip", CLIPS)
def test_adam_clip_and_bias_correction(cu, clip, t, wd):
    run_adam(cu, 4099, 0, "normal", clip, t, wd, seed=t % 101)


@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("clip", ["off", "below"])
@pytest.mark.parametrize("family", FAMILIES)
def test_adam_gradient_magnitudes(cu, family, clip, wd):
    """~1e-20: g*g lands among the fp32 subnormals; ~1e15: g*g ~ 1e30"""
    run_adam(cu, 4099, 1, family, clip, 3, wd, seed=7)


def test_adam_trajectory_norm_wise(cu):
    """50 chained steps against the float64 chain from the same start, norm-wise within twice the sum of the per-step
    bounds (the CPU test holds the fp32 specification to the same)"""
    n, T = 100_003, 50
    gen = torch.Generator().manual_seed(9)
    p0 = torch.randn(n, generator=gen)
    p, m, v = p0.cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    P, M, V = d(p0), torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    g, step = torch.empty(n, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    normsq, out = torch.zeros((), dtype=torch.float64, device="cuda"), torch.zeros(1, device="cuda")
    tol = {"p": 0.0, "m": 0.0, "v": 0.0}
    for k in range(T):
        gk = grads(n, "normal", gen) * (1 + 0.1 * k)
        g.copy_(gk)
        cu.sumsq(g, normsq)
        cu.increment(step)
        cu.adam_step(p, g, m, v, normsq, F32(100.0), LR, B1, B2, EPS, step, out, weight_decay=F32(0.01))
        r = R.adam_step64(P, d(gk), M, V, R.sumsq64(gk), k + 1, F32(100.0), LR, B1, B2, EPS, F32(0.01))
        P, M, V = r["p"], r["m"], r["v"]
        for key in tol:
            tol[key] += float(r["err_" + key].norm())
    for key, got, want in (("p", p, P), ("m", m, M), ("v", v, V)):
        err = float((d(got) - want).norm())
        RATIOS[f"adam trajectory {key}"] = err / tol[key]
        assert err <= 2 * tol[key], key


# ------------------------------------------------------------------------------------------------------- RMSprop
def run_rmsprop(cu, n, offset, family, clip, centered, momentum, wd, steps=2, seed=0, nan_at=None, inf_at=None):
    gen = torch.Generator().manual_seed(seed)
    g = grads(n, family, gen)
    s = float(g.abs().max()) or 1.0
    init = {"p": torch.randn(n, generator=gen), "g": g, "sq": s * s * (0.5 + torch.rand(n, generator=gen))}
    if momentum:
        init["buf"] = 0.1 * torch.randn(n, generator=gen)
    if centered:
        init["gavg"] = 0.3 * s * torch.randn(n, generator=gen)
    bufs = {k: guarded(x, offset) for k, x in init.items()}
    normsq, out = torch.zeros((), dtype=torch.float64, device="cuda"), torch.zeros(1, device="cuda")
    kw = dict(**RMS, weight_decay=F32(wd), momentum=F32(momentum))
    name = f"rmsprop{'_centered' if centered else ''}{'_momentum' if momentum else ''}{'_wd' if wd else ''}"
    for st in range(steps):
        if st:
            g = grads(n, family, gen)
        if nan_at is not None:
            g[nan_at] = float("nan")
        if inf_at is not None:
            g[inf_at] = float("inf")
        bufs["g"][1].copy_(g)
        ns = R.sumsq64(g)
        normsq.fill_(ns)
        mn = max_norm_for(clip, ns if math.isfinite(ns) else 1.0)
        cur = {k: d(b[1]) for k, b in bufs.items()}
        ref = R.rmsprop_step64(cur["p"], d(g), cur["sq"], ns, mn, momentum_buf=cur.get("buf"), grad_avg=cur.get("gavg"),
                               **kw)
        v = {k: (b[1] if b else None) for k, b in ((k, bufs.get(k)) for k in ("p", "g", "sq", "buf", "gavg"))}
        cu.rmsprop_step(v["p"], v["g"], v["sq"], v["buf"], v["gavg"], normsq, mn, kw["lr"], kw["alpha"], kw["eps"],
                        kw["weight_decay"], kw["momentum"], out)
        for k in ("p", "sq", "buf", "gavg"):
            if k in bufs:
                within(f"{name} {k}", bufs[k][1], ref[k], ref["err_" + k])
        tot = float(ref["total"].float())
        assert float(out) == tot or (math.isnan(tot) and math.isnan(float(out))), "norm_out"
    for k, (buf, _) in bufs.items():
        assert_guards(buf, n, offset)
    return {k: b[1] for k, b in bufs.items()}


VARIANTS = [(False, 0.0), (False, 0.9), (True, 0.0), (True, 0.9)]          # (centered, momentum): the four kernels


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("clip", ["off", "below", "at"])
@pytest.mark.parametrize("centered,momentum", VARIANTS)
@pytest.mark.parametrize("n,offset", [(1003, 0), (1003, 1), (5, 0), (ONE_PASS + 7, 0)])
def test_rmsprop(cu, n, offset, centered, momentum, clip, wd):
    run_rmsprop(cu, n, offset, "normal", clip, centered, momentum, wd, seed=n + offset)


@pytest.mark.parametrize("centered,momentum", VARIANTS)
@pytest.mark.parametrize("family", FAMILIES)
def test_rmsprop_gradient_magnitudes(cu, family, centered, momentum):
    run_rmsprop(cu, 4099, 0, family, "below", centered, momentum, 0.0, seed=3)


@pytest.mark.parametrize("momentum", [0.0, 0.9])
def test_rmsprop_centered_at_a_constant_gradient(cu, momentum):
    """After a long run on a constant gradient, grad_avg = g and square_avg = g^2 up to rounding, so the centered variance
    square_avg - grad_avg^2 is a few ulps from 0 and its fp32 value can be negative.  The kernel then takes sqrtf of a
    negative number and the parameter turns NaN in that element, as torch's fp32 RMSprop does (square_avg.addcmul(
    grad_avg, grad_avg, value=-1).sqrt_()).  What is asserted: the moments follow their float64 bounds; an element is
    NaN only where the exact variance of the kernel's own new state is within one rounding of zero or below it, and is
    NaN wherever that variance is negative by more than a rounding; every other element of p is the float64 step from
    the kernel's own new state, within the bound of the variance's rounding."""
    n = 4096
    gen = torch.Generator().manual_seed(5)
    g = torch.randn(n, generator=gen)
    p, sq, ga = torch.randn(n, generator=gen), g * g, g.clone()
    bufs = {"p": p.cuda(), "g": g.cuda(), "sq": sq.cuda(), "gavg": ga.cuda()}
    bufs["buf"] = (0.1 * torch.randn(n, generator=gen)).cuda() if momentum else None
    kw = dict(**RMS, weight_decay=0.0, momentum=F32(momentum))
    ns = R.sumsq64(g)
    ref = R.rmsprop_step64(d(p), d(g), d(sq), ns, 0.0, momentum_buf=None if bufs["buf"] is None else d(bufs["buf"]),
                           grad_avg=d(ga), **kw)
    buf0 = None if bufs["buf"] is None else d(bufs["buf"])
    normsq, out = torch.full((), ns, dtype=torch.float64, device="cuda"), torch.zeros(1, device="cuda")
    cu.rmsprop_step(bufs["p"], bufs["g"], bufs["sq"], bufs["buf"], bufs["gavg"], normsq, 0.0, kw["lr"], kw["alpha"],
                    kw["eps"], 0.0, kw["momentum"], out)
    within("rmsprop_constant sq", bufs["sq"], ref["sq"], ref["err_sq"])
    within("rmsprop_constant gavg", bufs["gavg"], ref["gavg"], ref["err_gavg"])
    sq1, ga1 = d(bufs["sq"]), d(bufs["gavg"])
    var = sq1 - ga1 * ga1                                   # exact: ga1^2 has 48 significant bits, sq1 and it are close
    slack = U * ga1 * ga1                                   # the fp32 product's rounding, if not fused
    nan = bufs["p"].isnan()
    assert bool((var[nan] <= slack[nan]).all()), "NaN where the variance is clearly positive"
    assert bool(nan[var < -slack].all()), "a clearly negative variance gave a number"
    ok = ~nan
    e_var = slack + U * var.abs()
    root = var.clamp_min(0).sqrt()
    avg = root + kw["eps"]
    e_avg = torch.minimum(e_var / (2 * root), e_var.sqrt()) + U * root + U * avg
    q = d(g) / avg
    e_q = q.abs() * e_avg / avg + U * q.abs()
    if momentum:
        b1 = buf0 * kw["momentum"] + q
        within("rmsprop_constant buf", bufs["buf"][ok], b1[ok], (e_q + U * (buf0 * kw["momentum"]).abs() + U * b1.abs())[ok])
        step, e_step = b1, e_q + U * (buf0 * kw["momentum"]).abs() + U * b1.abs()
    else:
        step, e_step = q, e_q
    p1 = d(p) - kw["lr"] * step
    within("rmsprop_constant p", bufs["p"][ok], p1[ok], (kw["lr"] * e_step + U * (kw["lr"] * step).abs() + U * p1.abs())[ok])
    print(f"\ncentered RMSprop at a constant gradient (momentum {momentum}): {int(nan.sum())} of {n} elements NaN")


# --------------------------------------------------------------------------------------------------- non-finite
OPTIMS = ["adam", "adam_wd", "rmsprop", "rmsprop_momentum", "rmsprop_centered", "rmsprop_centered_momentum"]


def run_optim(cu, which, clip, **kw):
    if which.startswith("adam"):
        return run_adam(cu, 1003, 0, "normal", clip, 5, 0.1 if which == "adam_wd" else 0.0, steps=1, **kw)
    return run_rmsprop(cu, 1003, 0, "normal", clip, "centered" in which, 0.9 if "momentum" in which else 0.0, 0.01,
                       steps=1, **kw)


@pytest.mark.parametrize("which", OPTIMS)
def test_nan_gradient_poisons_the_clipped_group(cu, which):
    """clip_grad_norm_ multiplies every gradient by a NaN coefficient when the total norm is NaN, so the reference's
    whole group turns NaN; the kernel must not step the finite elements unclipped"""
    st = run_optim(cu, which, "below", nan_at=17)
    assert bool(st["p"].isnan().all())


@pytest.mark.parametrize("which", OPTIMS)
@pytest.mark.parametrize("kind", ["nan", "inf"])
@pytest.mark.parametrize("clip", ["off", "below"])
def test_non_finite_gradient_element_matches_reference(cu, which, kind, clip):
    """element by element against the reference (inside run_*): an inf element makes the coefficient 0 and itself NaN;
    without clipping a non-finite element stays in its own element"""
    run_optim(cu, which, clip, **{f"{kind}_at": 17})


# ---------------------------------------------------------------------------------------------------- sumsq, EMA
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("n", SHAPES)
def test_sumsq(cu, n, det):
    """double accumulation: relative error <= 1e-12 of the exact sum (every term is non-negative)"""
    x = grads(n, "normal", torch.Generator().manual_seed(n))
    buf, view = guarded(x)
    out = torch.full((), float("nan"), dtype=torch.float64, device="cuda")
    try:
        cu.set_deterministic(det)
        cu.sumsq(view, out)
    finally:
        cu.set_deterministic(False)
    want = R.sumsq64(x)
    err = abs(float(out) - want) / want
    RATIOS["sumsq rel err / 1e-12"] = max(RATIOS.get("sumsq rel err / 1e-12", 0.0), err / 1e-12)
    assert err <= 1e-12, err


@pytest.mark.parametrize("det", [False, True])
def test_sumsq_64bit_indexing(cu, det):
    """n > 2^31: nonzero elements on both sides of 2^31 and at the end; a wrapped 32-bit index would drop them or count
    x[0] twice.  Needs 8.6 GB of free device memory (the machines are shared)."""
    n = (1 << 31) + 5
    free, _ = torch.cuda.mem_get_info()
    if free < 4 * n + (2 << 30):
        pytest.skip(f"needs {4 * n / 2 ** 30:.1f} GiB free, {free / 2 ** 30:.1f} GiB are")
    x = torch.zeros(n, device="cuda")
    for i, val in ((0, 8.0), ((1 << 31) - 1, 1.0), (1 << 31, 2.0), (n - 1, 4.0)):
        x[i] = val
    out = torch.zeros((), dtype=torch.float64, device="cuda")
    try:
        cu.set_deterministic(det)
        cu.sumsq(x, out)
    finally:
        cu.set_deterministic(False)
    torch.cuda.synchronize()
    del x
    assert float(out) == 64.0 + 1.0 + 4.0 + 16.0


@pytest.mark.parametrize("tau", [1.0, 0.02, 0.005])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("n", [1, 3, 1003, ONE_PASS + 7])
def test_ema(cu, n, offset, tau):
    gen = torch.Generator().manual_seed(n)
    t, s = torch.randn(n, generator=gen), 3 * torch.randn(n, generator=gen)
    tb, tv = guarded(t, offset)
    sb, sv = guarded(s, offset)
    cu.ema(tv, sv, F32(tau))
    if tau == 1.0:
        assert torch.equal(tv.cpu(), s)                      # the hard copy of the target critic's first update
    want, bound = R.ema64(d(t), d(s), F32(tau))
    within("ema", tv, want, bound)
    assert_guards(tb, n, offset), assert_guards(sb, n, offset)


# ------------------------------------------------------------------------------------------- element-wise kernels
SPECIAL = [0.0, -0.0, 1e-30, -1e-30, 1e-9, -1e-9, 1.0, -1.0, 20.0, -20.0, 1e30, -1e30, 3.4e38, -3.4e38]


def special_rows(M, C, seed, scale):
    x = torch.randn(M, C, generator=torch.Generator().manual_seed(seed)) * scale
    x.view(-1)[:len(SPECIAL)] = torch.tensor(SPECIAL)
    return x


def test_symlog(cu):
    """sign(x) log(1 + |x|) (sheeprl/utils/utils.py:148) into a column slice, from a strided source: the rounding of
    1 + |x| is an absolute u after the log; logf is within 1 ulp (CUDA Math API)"""
    x = special_rows(37, 9, 1, 30.0)
    src, dst = torch.zeros(37, 13, device="cuda"), torch.full((37, 16), FILL, device="cuda")
    src[:, 2:11] = x.cuda()
    cu.symlog(src[:, 2:11], dst[:, 4:13])
    x64 = d(x)
    want = torch.sign(x64) * torch.log1p(x64.abs())
    within("symlog", dst[:, 4:13], want, U + 2 * U * want.abs())
    assert bool((dst[:, :4] == FILL).all()) and bool((dst[:, 13:] == FILL).all())
    assert bool((dst[:, 4:13][x.cuda() == 0] == 0).all())


def test_tanh_fwd(cu):
    """tanhf is within 2 ulp (CUDA Math API); tanh(+-0) = +-0 with its sign, saturation gives exactly +-1"""
    x = torch.cat([torch.tensor(SPECIAL), torch.randn(10_000, generator=torch.Generator().manual_seed(2)) * 3]).cuda()
    y = torch.empty_like(x)
    cu.tanh_fwd(x, y)
    want = torch.tanh(d(x))
    within("tanh_fwd", y, want, 4 * U * want.abs() + R.TINY)
    assert torch.equal(torch.signbit(y[:2]), torch.tensor([False, True], device="cuda")) and bool((y[:2] == 0).all())
    assert bool((y[x.abs() >= 20] == torch.sign(x[x.abs() >= 20])).all())


@pytest.mark.parametrize("accumulate", [False, True])
def test_tanh_bwd(cu, accumulate):
    """dx (+)= dy (1 - y^2): the product y*y, the difference, the product with dy (and the sum)"""
    gen = torch.Generator().manual_seed(3)
    y = torch.tanh(torch.randn(10_003, generator=gen) * 3)
    y[:5] = torch.tensor([1.0, -1.0, 0.0, -0.0, 0.9999999])
    dy = torch.randn(10_003, generator=gen) * 10
    dx0 = torch.randn(10_003, generator=gen)
    dx = dx0.cuda()
    cu.tanh_bwd(y.cuda(), dy.cuda(), dx, accumulate)
    y64, dy64 = d(y), d(dy)
    t = 1 - y64 * y64
    r = dy64 * t
    bound = dy64.abs() * (U * y64 * y64 + U * t.abs()) + U * r.abs()
    if accumulate:
        r = r + d(dx0)
        bound = bound + U * r.abs()
    within(f"tanh_bwd acc={int(accumulate)}", dx, r, bound + R.TINY)


def test_axpy_and_affine(cu):
    """axpy: one fmaf, a single rounding; affine: alpha x + beta, at most two"""
    gen = torch.Generator().manual_seed(4)
    x = torch.cat([torch.tensor(SPECIAL[:12]), torch.randn(10_001, generator=gen) * 100])
    y = torch.cat([torch.tensor([-0.0, 0.0] * 6), torch.randn(10_001, generator=gen)])
    for alpha in (F32(0.5), F32(-3.7e-3), F32(1e3)):
        yg = y.cuda()
        cu.axpy(x.cuda(), yg, alpha)
        want = alpha * d(x) + d(y)
        within("axpy", yg, want, U * want.abs() + R.TINY)
        for beta in (0.0, F32(1.3)):
            out = torch.empty_like(yg)
            cu.affine(x.cuda(), out, alpha, beta)
            want = alpha * d(x) + beta
            within("affine", out, want, U * (alpha * d(x)).abs() + U * want.abs() + R.TINY)


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _odd_values(*shape, seed=0):
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(seed))
    flat = x.view(-1)
    k = min(5, flat.numel())
    flat[:k] = torch.tensor([float("nan"), -0.0, 1e-45, -3e-39, float("inf")])[:k]
    return x


@pytest.mark.parametrize("M,C,lds,ldd", [(33, 20, 20, 20), (1, 1003, 1003, 1003), (33, 20, 27, 50), (7, 5, 5, 9),
                                         (1000, 3, 8, 3), (1, 1, 1, 1)])
def test_copy2d_is_bit_exact(cu, M, C, lds, ldd):
    """lds = ldd = C takes the cudaMemcpyAsync branch, any other stride the kernel.  NaN, -0 and subnormals keep their
    bits; the destination's other columns and the guards stay untouched."""
    src = _odd_values(M, lds, seed=M).cuda()[:, :C]
    dbuf = torch.full((M * ldd + 2 * GUARD,), FILL, device="cuda")
    rows = dbuf[GUARD:GUARD + M * ldd].view(M, ldd)
    cu.copy(src, rows[:, :C])
    assert torch.equal(_bits(rows[:, :C]), _bits(src))
    assert bool((rows[:, C:] == FILL).all())
    assert_guards(dbuf, M * ldd)


@pytest.mark.parametrize("NB,a,b", [(7, 16, 40), (3, 33, 65), (1, 1, 1), (2, 100, 3), (65, 31, 97)])
def test_transpose_batched_is_bit_exact(cu, NB, a, b):
    X = _odd_values(NB, a, b, seed=a).cuda()
    Y = torch.full((NB * a * b + 2 * GUARD,), FILL, device="cuda")
    cu.transpose_batched(X, Y[GUARD:GUARD + NB * a * b].view(NB, b, a))
    assert torch.equal(_bits(Y[GUARD:GUARD + NB * a * b].view(NB, b, a)), _bits(X.transpose(1, 2)))
    assert_guards(Y, NB * a * b)


@pytest.mark.parametrize("rows,cols,ldx,ldy", [(40, 70, 70, 40), (33, 65, 80, 37), (1, 1, 1, 1), (3, 300, 301, 5),
                                               (1025, 3, 4, 1030)])
def test_transpose2d_is_bit_exact(cu, rows, cols, ldx, ldy):
    X = _odd_values(rows, ldx, seed=rows).cuda()
    Y = torch.full((cols, ldy), FILL, device="cuda")
    cu.transpose2d(X[:, :cols], Y[:, :rows])
    assert torch.equal(_bits(Y[:, :rows]), _bits(X[:, :cols].t()))
    assert bool((Y[:, rows:] == FILL).all())


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
@pytest.mark.parametrize("shape", [(3, 1, 8, 12), (2, 3, 16, 16), (2, 4, 20, 20), (2, 12, 84, 84),      # 4-pixel kernels
                                   (2, 3, 5, 5), (3, 12, 7, 9), (2, 5, 6, 6), (1, 2, 4, 4)])         # the generic one
def test_obs_prep(cu, shape, dtype):
    """out [N,H,W,C] = obs [N,C,H,W] / 255 - 0.5 (dreamer_v3.py:98): the division and the shift are one rounding each,
    u of the quotient plus u of the result (the shift cancels near 127.5).  The 4-pixel kernels (C in 1, 3, 4, 12, HW a
    multiple of 4, aligned rows) give the generic kernel's bits, which an output one float off its alignment forces."""
    NB, C, H, W = shape
    g = torch.Generator().manual_seed(C * H)
    obs = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    if dtype == torch.float32:
        obs = obs.float()
        obs.view(-1)[::7] += 0.5                             # float observations need not be integers
    og = obs.cuda()
    n = obs.numel()
    out = torch.full((n + 2 * GUARD,), FILL, device="cuda")
    cu.obs_prep(og, out[GUARD:GUARD + n].view(NB, H, W, C))
    q = d(obs).permute(0, 2, 3, 1) / 255.0
    want = q - 0.5
    within("obs_prep", out[GUARD:GUARD + n].view(NB, H, W, C), want, U * q + U * want.abs())
    assert_guards(out, n)
    generic = torch.full((n + 2 * GUARD + 1,), FILL, device="cuda")
    cu.obs_prep(og, generic[GUARD + 1:GUARD + 1 + n].view(NB, H, W, C))
    assert torch.equal(_bits(generic[GUARD + 1:GUARD + 1 + n]), _bits(out[GUARD:GUARD + n]))
    assert_guards(generic, n, 1)


def _patches(x, k, s):
    """[B, Ho, Wo, k, k, C] views of the k x k patches of x [B, H, W, C] at stride s"""
    B, H, W, C = x.shape
    Ho, Wo = (H - k) // s + 1, (W - k) // s + 1
    return Ho, Wo, torch.stack([torch.stack([x[:, ky:ky + s * (Ho - 1) + 1:s, kx:kx + s * (Wo - 1) + 1:s, :]
                                             for kx in range(k)], 3) for ky in range(k)], 3)


@pytest.mark.parametrize("B,H,C,k,s", [(3, 84, 12, 8, 4), (3, 20, 32, 4, 2), (3, 9, 64, 3, 1), (2, 11, 5, 3, 2),
                                       (2, 7, 3, 7, 1), (2, 10, 3, 2, 3), (1, 5, 1, 1, 1), (2, 21, 7, 5, 2)])
def test_im2col_col2im(cu, B, H, C, k, s):
    """im2col is a gather: bit-exact.  col2im sums the patches overlapping each pixel (up to ceil(k/s)^2 terms) in
    fp32: within (terms - 1) u of the sum of their magnitudes, and exactly 0 where the ReLU mask is off."""
    gen = torch.Generator().manual_seed(H + k)
    x = torch.randn(B, H, H, C, generator=gen)
    Ho, Wo, pt = _patches(x, k, s)
    col = torch.full((B * Ho * Wo * k * k * C + 2 * GUARD,), FILL, device="cuda")
    cv = col[GUARD:GUARD + B * Ho * Wo * k * k * C].view(B * Ho * Wo, k * k * C)
    cu.im2col(x.cuda(), cv, k, s)
    assert torch.equal(cv.cpu(), pt.reshape(B * Ho * Wo, k * k * C)) and bool((col[:GUARD] == FILL).all())
    assert bool((col[-GUARD:] == FILL).all())
    dcol = torch.randn(B * Ho * Wo, k * k * C, generator=gen)
    act = torch.randn(B, H, H, C, generator=gen).clamp_min(0)
    dc = d(dcol).view(B, Ho, Wo, k, k, C)
    sums, mags, terms = (torch.zeros(B, H, H, C, dtype=torch.float64, device="cuda") for _ in range(3))
    for ky in range(k):
        for kx in range(k):
            sl = (slice(None), slice(ky, ky + s * (Ho - 1) + 1, s), slice(kx, kx + s * (Wo - 1) + 1, s))
            sums[sl] += dc[:, :, :, ky, kx]
            mags[sl] += dc[:, :, :, ky, kx].abs()
            terms[sl] += 1
    bound = (terms - 1).clamp_min(0) * U * mags
    for a in (None, act):
        dx = torch.full((B, H, H, C), FILL, device="cuda")
        cu.col2im(dcol.cuda(), None if a is None else a.cuda(), dx, k, s)
        want = sums if a is None else sums * (d(a) > 0)
        within(f"col2im{'' if a is None else ' masked'}", dx, want, bound)
        if a is not None:
            assert bool((dx[a.cuda() <= 0] == 0).all())
