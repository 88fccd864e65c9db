"""Every Dreamer-V3 objective kernel (csrc/losses.cu, csrc/dv3_cont.cu, the KL of csrc/rssm.cu) against the float64
reference of oracle/loss_ref.py, across each launch's warp, block and grid edges.

Each case runs the kernel twice and checks:
  - error <= bound element by element (not relative to the largest entry, so one small wrong entry fails);
  - the two runs bit-identical: none of these kernels uses float atomics;
  - nothing outside the output views written (guard values around the rows and in the padding between nb and ldd).
moments_update is held to fp32 torch.quantile: equal order statistics, the lerp within 2 ulp, NaN where torch gives NaN.
Cases, input families and the emulator's margins are in tests/test_loss_ref_cpu.py, which also shows the bounds reject
a softmax without max shift, swapped two-hot weights, exp(m) in twohot_mean_bwd, an uncentred KL gradient, a unimix
chain rule through s, the entropy gradient without +ent, a late lambda-return carry, a naive BCE and a clip factor that
is differentiated.
"""
import json
import math
import os

import pytest
import torch

from oracle import loss_ref as R
from tests.test_gpu_ln_precision import Guarded
from tests.test_loss_ref_cpu import (ACTOR_HEADS, CONT_ARGS, CONT_AS, HIGH, KL_CASES, LAMBDA_CASES, LOW, TWOHOT_CASES,
                                     actor_inputs, cont_inputs, gen, kl_inputs, lambda_inputs, logit_rows,
                                     moments_inputs, quantile_ok, ratio, twohot_inputs, worst)

pytestmark = pytest.mark.gpu

MARGINS = {}                     # case id -> worst error / bound per output, kept for reporting
CHUNK = 1 << 22                  # elements per float64 reference chunk


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    yield CudaOps("cuda")
    path = os.environ.get("LOSS_PRECISION_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(MARGINS, f, indent=1, sort_keys=True)


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def twice(run):
    """run() -> dict of fresh output tensors, guards checked inside; the two runs must agree bit for bit"""
    first, again = run(), run()
    for k in first:
        assert same_bits(first[k], again[k]), f"{k}: rerun is not bit-identical"
    return first


def guarded(M, C, ld=None, fill=math.nan):
    return Guarded(M, C, ld or C, fill=torch.full((M, C), fill, device="cuda"))


def row(n, fill=math.nan):
    return guarded(1, n, fill=fill)


def record(case, m):
    MARGINS[case] = m
    assert max(m.values()) <= 1.0, m


def chunked(M, width):
    """row ranges of at most CHUNK elements, for the float64 reference"""
    step = max(1, CHUNK // max(width, 1))
    return [(a, min(M, a + step)) for a in range(0, M, step)]


# ------------------------------------------------------------------------------------------------------------ two-hot
@pytest.mark.parametrize("case", list(TWOHOT_CASES))
def test_twohot_precision(cu, case):
    """twohot_loss_grad (plain / strided ldl and ldd / accumulate / weight), twohot_mean and twohot_mean_bwd"""
    M, nb, fam, xf, layout = TWOHOT_CASES[case]
    logits, x, w = twohot_inputs(M, nb, fam, xf, layout, seed=len(case), device="cuda")
    strided = layout == "strided"
    ldl, ldd = (nb + 3, nb + 5) if strided else (nb, nb)
    lg = Guarded(M, nb, ldl, fill=logits)
    acc = layout == "accumulate"
    g = gen(2, "cuda")
    prior_l = torch.randn(M, generator=g, device="cuda") if acc else None
    prior_d = torch.randn(M, nb, generator=g, device="cuda") * 1e-3 if acc else None
    dm = torch.randn(M, generator=g, device="cuda")

    def run():
        loss = Guarded(1, M, M, fill=prior_l.reshape(1, M) if acc else torch.full((1, M), math.nan, device="cuda"))
        d = Guarded(M, nb, ldd, fill=prior_d if acc else torch.full((M, nb), math.nan, device="cuda"))
        cu.twohot_loss_grad(lg.view, x, w, 0.25, LOW, HIGH, loss.view[0], d.view, accumulate=acc)
        mean = row(M)
        cu.twohot_mean(lg.view, LOW, HIGH, mean.view[0])
        mg = guarded(M, nb, ldd)
        cu.twohot_mean_bwd(lg.view, dm, LOW, HIGH, mg.view)
        for b in (loss, d, mean, mg, lg):
            assert b.outside_untouched(), "write outside the output view"
        assert torch.equal(lg.view, logits), "the logits were written"
        return {"loss": loss.view[0].clone(), "grad": d.view.clone(), "mean": mean.view[0].clone(),
                "mean_grad": mg.view.clone()}

    out = twice(run)
    m = {}
    for a, b in chunked(M, nb):
        ref, bd = R.twohot_loss(logits[a:b], x[a:b], None if w is None else w[a:b], 0.25, LOW, HIGH)
        if acc:
            ref["loss"], bd["loss"] = ref["loss"] + prior_l[a:b].double(), R.acc_bound(bd["loss"], prior_l[a:b],
                                                                                        ref["loss"])
            bd["grad"] = R.acc_bound(bd["grad"], prior_d[a:b], ref["grad"])
            ref["grad"] = ref["grad"] + prior_d[a:b].double()
        r2, b2 = R.twohot_mean(logits[a:b], LOW, HIGH, dm[a:b])
        ref.update(mean=r2["mean"], mean_grad=r2["grad"])
        bd.update(mean=b2["mean"], mean_grad=b2["grad"])
        got = {k: v[a:b] for k, v in out.items()}
        for k, v in worst(got, ref, bd).items():
            m[k] = max(m.get(k, 0.0), v)
    record(f"twohot_{case}", m)


# ------------------------------------------------------------------------------------------------------------ bce / mse
@pytest.mark.parametrize("M", [1, 7, 8, 9, 1000, 1 << 20])
def test_bce_precision(cu, M):
    g = gen(M, "cuda")
    l = 4 * torch.randn(M, generator=g, device="cuda")
    edge = torch.tensor([0.0, 1e-9, -1e-9, 17.5, -17.5, 40.0, -40.0, 90.0], device="cuda")
    l[:min(M, 8)] = edge[:min(M, 8)]
    y = (torch.rand(M, generator=g, device="cuda") > 0.5).float()

    def run():
        lr, dl = row(M), row(M)
        cu.bce_loss_grad(l, y, 1.0, 1.0 / 4096, lr.view[0], dl.view[0])
        assert lr.outside_untouched() and dl.outside_untouched()
        return {"loss": lr.view[0].clone(), "grad": dl.view[0].clone()}

    ref, bd = R.bce(l, y, 1.0, 1.0 / 4096)
    record(f"bce_M{M}", worst(twice(run), ref, bd))


@pytest.mark.parametrize("alias", [True, False], ids=["grad_is_pred", "separate"])
@pytest.mark.parametrize("MP", [(1, 1), (7, 33), (9, 256), (1000, 1000), (1 << 16, 77)], ids=str)
def test_mse_precision(cu, MP, alias):
    """the engine passes grad = pred: every element is read before the same thread writes it"""
    M, P = MP
    g = gen(P, "cuda")
    pred, tgt = torch.randn(M, P, generator=g, device="cuda"), torch.randn(M, P, generator=g, device="cuda") + 0.5

    def run():
        p = guarded(M, P, fill=0.0)
        p.view.copy_(pred)
        gr = p if alias else guarded(M, P)
        lr = row(M)
        cu.mse_loss_grad(p.view, tgt, 1.0 / M, lr.view[0], gr.view)
        assert lr.outside_untouched() and gr.outside_untouched() and p.outside_untouched()
        if not alias:
            assert torch.equal(p.view, pred), "pred was written"
        return {"loss": lr.view[0].clone(), "grad": gr.view.clone()}

    ref, bd = R.mse(pred, tgt, 1.0 / M)
    record(f"mse_M{M}_P{P}_{'alias' if alias else 'separate'}", worst(twice(run), ref, bd))


# ------------------------------------------------------------------------------------------------------------ KL
@pytest.mark.parametrize("case", list(KL_CASES))
def test_kl_precision(cu, case):
    G, K, fam = KL_CASES[case]
    M = 300
    post, prior, free = kl_inputs(M, G, K, fam, seed=len(case), device="cuda")
    C = G * K
    strided = len(case) % 2 == 1
    ld = C + 3 if strided else C
    pg, qg = Guarded(M, C, ld, fill=post), Guarded(M, C, ld + 2 if strided else C, fill=prior)

    def run():
        dp, dq = guarded(M, C, C + 5 if strided else C), guarded(M, C, C + 1 if strided else C)
        rows = guarded(M, 4)
        cu.kl_loss_grad(pg.view, qg.view, G, K, 0.5, 0.1, free, 1.0, 1.0 / M, dp.view, dq.view, rows.view)
        for b in (dp, dq, rows, pg, qg):
            assert b.outside_untouched(), "write outside the output view"
        return {"rows": rows.view.clone(), "d_post": dp.view.clone(), "d_prior": dq.view.clone()}

    ref, bd = R.kl_loss(post, prior, G, K, 0.5, 0.1, free, 1.0, 1.0 / M)
    record(f"kl_{case}{'_strided' if strided else ''}", worst(twice(run), ref, bd))


# ------------------------------------------------------------------------------------------------------------ actor
@pytest.mark.parametrize("unimix", [0.0, 0.01])
@pytest.mark.parametrize("M", [1, 9, 1000, 1 << 18])
@pytest.mark.parametrize("heads", list(ACTOR_HEADS))
def test_actor_loss_precision(cu, heads, M, unimix):
    hd = ACTOR_HEADS[heads]
    raw, acts, lam, val, disc, mom, A = actor_inputs(M, hd, seed=len(heads) + M, device="cuda")

    def run():
        rows, draw = row(M), guarded(M, A)
        cu.actor_loss_grad(raw, acts, lam, val, disc, mom, hd, unimix, 3e-4, 1.0 / M, rows.view[0], draw.view)
        assert rows.outside_untouched() and draw.outside_untouched()
        return {"rows": rows.view[0].clone(), "draw": draw.view.clone()}

    out = twice(run)
    m = {}
    for a, b in chunked(M, A):
        ref, bd = R.actor_loss(raw[a:b], acts[a:b], lam[a:b], val[a:b], disc[a:b], mom, hd, unimix, 3e-4, 1.0 / M)
        for k, v in worst({k: o[a:b] for k, o in out.items()}, ref, bd).items():
            m[k] = max(m.get(k, 0.0), v)
    record(f"actor_{heads}_M{M}_u{unimix}", m)


# ------------------------------------------------------------------------------------------------------------ lambda
@pytest.mark.parametrize("case", list(LAMBDA_CASES))
def test_lambda_returns_precision(cu, case):
    """lambda_returns, then lambda_returns_bwd on the kernel's own lam and discount"""
    H, N, gamma, lmbda = LAMBDA_CASES[case]
    gamma, lmbda = R.f32(gamma), R.f32(lmbda)
    rew, val, cl, tc = lambda_inputs(H, N, seed=len(case), device="cuda")
    ent = torch.randn(H * N, generator=gen(3, "cuda"), device="cuda")
    mom = torch.tensor([0.5, 3.0], device="cuda")
    scale = 1.0 / (H * N)

    def run():
        lam, disc = guarded(H, N), guarded(H + 1, N)
        cu.lambda_returns(rew, val, cl, tc, gamma, lmbda, lam.view, disc.view)
        dv, dr, rows = guarded(H + 1, N), guarded(H + 1, N), guarded(H, N)
        cu.lambda_returns_bwd(cl, disc.view, mom, lam.view, val, ent, gamma, lmbda, 3e-4, scale, dv.view, dr.view,
                              rows.view)
        for b in (lam, disc, dv, dr, rows):
            assert b.outside_untouched(), "write outside the output view"
        return {"lam": lam.view.clone(), "discount": disc.view.clone(), "rows": rows.view.clone(),
                "d_val": dv.view.clone(), "d_rew": dr.view.clone()}

    out = twice(run)
    ref, bd = R.lambda_returns(rew, val, cl, tc, gamma, lmbda)
    m = worst({"lam": out["lam"], "discount": out["discount"]}, ref, bd)
    ref, bd = R.lambda_returns_bwd(cl, out["discount"], mom, out["lam"], val, ent, gamma, lmbda, 3e-4, scale)
    m.update(worst({k: out[k] for k in ref}, ref, bd))
    record(f"lambda_{case}", m)


# ------------------------------------------------------------------------------------------------------------ cont_action
@pytest.mark.parametrize("M", [1, 9, 1000, 1 << 16])
@pytest.mark.parametrize("A", CONT_AS)
def test_cont_action_precision(cu, A, M):
    """cont_action_fwd into a strided action view (lda), cont_action_bwd from a strided d_action (ldd); about a third of
    the actions pass action_clip"""
    head, eps, dact, disc = cont_inputs(M, A, seed=A + M, device="cuda")
    dg = Guarded(M, A, A + 3, fill=dact)

    def run():
        act, ent = guarded(M, A, A + 2), row(M)
        cu.cont_action_fwd(head, eps, act.view, ent.view[0], *CONT_ARGS)
        dh = guarded(M, 2 * A)
        cu.cont_action_bwd(head, eps, dg.view, disc, dh.view, *CONT_ARGS, -0.01)
        for b in (act, ent, dh, dg):
            assert b.outside_untouched(), "write outside the output view"
        return {"action": act.view.clone(), "ent": ent.view[0].clone(), "dhead": dh.view.clone()}

    out = twice(run)
    ref, bd = R.cont_action(head, eps, *CONT_ARGS, dact, disc, -0.01)
    if M >= 1000:
        assert bool((ref["action"].abs() >= CONT_ARGS[3]).any()), "no action reaches the clip"
    record(f"cont_A{A}_M{M}", worst(out, ref, bd))


# ------------------------------------------------------------------------------------------------------------ moments
MOMENT_NS = (1, 2, 1023, 1024, 1025, 122880, 1 << 24)
MOMENT_FAMILIES = ("random", "ties", "equal", "zeros", "nan")


def run_moments(cu, x, state, decay, q_lo=0.05, q_hi=0.95):
    def run():
        st, out = Guarded(1, 2, 2, fill=state.reshape(1, 2)), row(2)
        cu.moments_update(x, st.view[0], decay, 1e8, q_lo, q_hi, out.view[0])
        assert st.outside_untouched() and out.outside_untouched()
        return {"state": st.view[0].clone(), "out": out.view[0].clone()}

    return twice(run)


@pytest.mark.parametrize("family", MOMENT_FAMILIES)
@pytest.mark.parametrize("n", MOMENT_NS)
def test_moments_update_matches_torch_quantile(cu, n, family):
    """decay 0: the state is the kernel's quantiles; decay 0.99: the EMA within its bound"""
    x = moments_inputs(n, family, seed=n, device="cuda")
    lo, hi = R.quantiles32(x, 0.05, 0.95)
    got = run_moments(cu, x, torch.zeros(2, device="cuda"), 0.0)["state"]
    assert quantile_ok(got[0], lo) and quantile_ok(got[1], hi), (got.tolist(), float(lo), float(hi))
    for q, v in ((0.05, lo), (0.95, hi)):
        rank = torch.tensor(q, dtype=torch.float32) * (n - 1)
        if float(rank) == math.floor(float(rank)):                   # an order statistic itself: exact
            assert float(got[0 if q < 0.5 else 1]) == float(v) or math.isnan(float(v))
    state = torch.tensor([-0.3, 1.7], device="cuda")
    out = run_moments(cu, x, state, 0.99)
    (st, o), _, (b_st, b_o) = R.moments(x, state, 0.99, 1e8, 0.05, 0.95)
    m = {"state": ratio(out["state"], st, b_st), "out": ratio(out["out"], o, b_o)}
    record(f"moments_n{n}_{family}", m)


@pytest.mark.parametrize("q", [0.95, 0.05, 0.5, 0.0, 1.0])
def test_moments_update_inf_next_to_an_integral_rank(cu, q):
    """x = 0..19 and +inf, shuffled (and -inf at the bottom for q = 0.05): q (n - 1) is integral in fp32 for q = 0.95
    and 0.05, so the quantile is an element, not NaN from 0 * inf.  q = 0 / 1 select +-inf itself, where ATen's
    lerp(inf, inf, 0) is NaN."""
    x = torch.cat([torch.arange(20.0), torch.tensor([math.inf])])
    if q == 0.05 or q == 0.0:
        x = torch.cat([torch.tensor([-math.inf]), torch.arange(1.0, 20.0), torch.tensor([math.inf])])
    x = x[torch.randperm(x.numel(), generator=torch.Generator().manual_seed(0))].cuda()
    want = torch.quantile(x.cpu(), q)
    got = run_moments(cu, x, torch.zeros(2, device="cuda"), 0.0, q, q)["state"]
    assert quantile_ok(got[0], want) and quantile_ok(got[1], want), (got.tolist(), float(want))


def test_moments_update_extreme_range(cu):
    """[-3e38, 3e38] at q = 0: rank 0 is integral, so the result is -3e38, not a lerp through b - a = inf"""
    x = torch.tensor([3e38, -3e38], device="cuda")
    got = run_moments(cu, x, torch.zeros(2, device="cuda"), 0.0, 0.0, 1.0)["state"]
    assert float(got[0]) == R.f32(-3e38) and float(got[1]) == R.f32(3e38), got.tolist()


def test_moments_update_nan_gives_nan(cu):
    """a NaN anywhere (either sign) makes both quantiles, the state and the invscale NaN, as torch.quantile and
    torch.max do"""
    for sign in (1.0, -1.0):
        x = torch.randn(1025, generator=torch.Generator().manual_seed(1))
        x[77] = sign * math.nan
        out = run_moments(cu, x.cuda(), torch.zeros(2, device="cuda"), 0.99)
        assert bool(out["state"].isnan().all()) and bool(out["out"].isnan().all()), out


# ------------------------------------------------------------------------------------------------------------ sums
@pytest.mark.parametrize("MC", [(1, 1), (7, 3), (1000, 255), (1 << 20, 3), (9, 1000)], ids=str)
def test_sum_rows_precision(cu, MC):
    M, C = MC
    X = logit_rows(M, C, "s2", gen(M, "cuda"), "cuda") + 1.0
    xg = Guarded(M, C, C + 7, fill=X)

    def run():
        o = row(C)
        cu.sum_rows(xg.view, o.view[0], 0.5)
        assert o.outside_untouched()
        return {"sum": o.view[0].clone()}

    s, b = R.sum_rows(X, 0.5)
    record(f"sum_rows_M{M}_C{C}", {"sum_rows": ratio(twice(run)["sum"], s, b)})


@pytest.mark.parametrize("n", [1, 1000, 1023, 1 << 20])
def test_weighted_mean_precision(cu, n):
    g = gen(n, "cuda")
    x, w = torch.randn(n, generator=g, device="cuda") + 0.3, torch.rand(n, generator=g, device="cuda")

    def run():
        o = row(1)
        cu.weighted_mean(x, w, 1.0 / n, o.view[0])
        assert o.outside_untouched()
        return {"out": o.view[0].clone()}

    s, b = R.weighted_mean(x, w, 1.0 / n)
    record(f"weighted_mean_n{n}", {"weighted_mean": ratio(twice(run)["out"], s.reshape(1), b.reshape(1))})
