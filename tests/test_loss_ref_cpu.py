"""The float64 reference of the Dreamer-V3 objective kernels (oracle/loss_ref.py) and its error bounds, on the CPU.

  - the reference is the reference's semantics: it reproduces, to ~1e-12, a fixture made by running the reference's own
    classes in float64 with autograd (oracle/make_golden_loss_ref.py -> tests/golden/dv3_loss_ref.pt), and re-runs the
    comparison live when the reference package is importable;
  - an honest fp32 implementation (EmulOps, the kernels' specification) stays within every bound with 2x headroom at
    each GPU case shape that fits on the CPU (the cases of tests/test_gpu_loss_precision.py are defined here);
  - fp32 implementations with one plausible defect each exceed the bound by at least 4x.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import loss_ref as R
from oracle.ops_emul import EmulOps

LOW, HIGH = -20.0, 20.0
U = R.U
GOLDEN = "tests/golden/dv3_loss_ref.pt"


# ------------------------------------------------------------------------------------------------------------ inputs
def gen(seed, device="cpu"):
    return torch.Generator(device=device).manual_seed(seed)


def logit_rows(M, K, family, g, device="cpu"):
    """s0.1 / s2 / s30: N(0, sigma); offset: N(0, 2) + 1000 (softmax-invariant: only a max shift survives it);
    dominant: N(0, 1) with one class raised until p ~ 1 - 1e-7"""
    n = torch.randn(M, K, generator=g, device=device)
    if family.startswith("s"):
        return float(family[1:]) * n
    if family == "offset":
        return 2.0 * n + 1000.0
    assert family == "dominant", family
    hot = torch.randint(0, K, (M,), generator=g, device=device)
    return n + F.one_hot(hot, K).float() * (math.log(max(K - 1, 1) / 1e-7) + 3.0)


def twohot_x(M, nb, family, g, device="cpu"):
    """cont: symexp of U(-21, 21); at_bin: the fp32 symexp of a bin; near_bin: one fp32 ulp either side of it (symlog
    within about an ulp of the bin); edges: +-20, +-0, +-1e9 and their neighbours"""
    if family == "cont":
        return R.symexp64(42.0 * torch.rand(M, generator=g, device=device, dtype=torch.float64) - 21.0).float()
    b32 = torch.linspace(LOW, HIGH, nb, device=device)
    pick = b32[torch.randint(0, nb, (M,), generator=g, device=device)]
    at = torch.sign(pick) * (torch.exp(pick.abs()) - 1)
    if family == "at_bin":
        return at
    if family == "near_bin":
        up = torch.rand(M, generator=g, device=device) < 0.5
        return torch.where(up, torch.nextafter(at, torch.full_like(at, math.inf)),
                           torch.nextafter(at, torch.full_like(at, -math.inf)))
    assert family == "edges", family
    e = torch.tensor([20.0, -20.0, 0.0, -0.0, 1e9, -1e9, 4.8e8, -4.8e8], device=device)
    return e[torch.randint(0, e.numel(), (M,), generator=g, device=device)]


# ------------------------------------------------------------------------------------------------------------ metrics
def ratio(got, ref, bound):
    """max |got - ref| / bound; an element whose bound is 0 must be exact; NaN on one side only counts as infinitely
    wrong, NaN on both sides as agreement"""
    got, ref = got.double().reshape(ref.shape), ref
    both = got.isnan() & ref.isnan()
    d = (got - ref).abs()
    d = torch.where(both | (got == ref), torch.zeros_like(d), d)
    r = torch.where(d == 0, torch.zeros_like(d), d / bound)
    return float("inf") if bool(r.isnan().any()) else float(r.max()) if r.numel() else 0.0


def worst(got: dict, ref: dict, bound: dict):
    return {k: ratio(got[k], ref[k], bound[k]) for k in ref}


# ------------------------------------------------------------------------------------------------------------ cases
# The GPU file runs every case; this file holds EmulOps to the same bounds at the ones that fit on the CPU.
ROW_COUNTS = (1, 7, 8, 9, 1000, 1 << 20)
NBS = (2, 31, 32, 33, 255, 256, 1000)
LOGIT_FAMILIES = ("s0.1", "s2", "s30", "offset", "dominant")
X_FAMILIES = ("cont", "at_bin", "near_bin", "edges")


def _twohot_cases():
    out, k = {}, 0
    for nb in NBS:
        for M in ROW_COUNTS:
            if M * nb > (1 << 20) * 256:
                continue
            fam, xf = LOGIT_FAMILIES[k % 5], X_FAMILIES[(k + k // 5) % 4]
            layout = ("plain", "strided", "accumulate", "weight")[k % 4]
            out[f"nb{nb}_M{M}_{fam}_{xf}_{layout}"] = (M, nb, fam, xf, layout)
            k += 1
    return out


TWOHOT_CASES = _twohot_cases()
KL_CASES = {f"G{G}_K{K}_{fam}": (G, K, fam) for i, (G, K) in enumerate((G, K) for G in (1, 7, 8, 9, 32, 64)
                                                                       for K in (2, 31, 32, 33, 64))
            for fam in (("s2", "near_free") if i % 2 else ("s0.1", "offset", "dominant") if i % 3 else ("s30",))}
ACTOR_HEADS = {"2": (2,), "18": (18,), "3x2": (3, 2), "40": (40,), "16heads": tuple(range(2, 18))}
LAMBDA_CASES = {f"H{H}_N{N}_g{g}_l{l}": (H, N, g, l) for i, (H, N) in enumerate((H, N) for H in (1, 15, 64)
                                                                               for N in (1, 127, 128, 129, 16384))
                for g, l in (((0.997, 0.95), (1.0, 0.0)) if i % 2 else ((0.997, 1.0), (1.0, 0.95)))}
CONT_AS = (1, 6, 32, 33, 64)


def cont_logits(shape, g, device="cpu"):
    """continue logits: random N(0, 4) with exact 0 and +-1e-9 mixed in"""
    c = 4.0 * torch.randn(shape, generator=g, device=device)
    pick = torch.rand(shape, generator=g, device=device)
    c = torch.where(pick < 0.1, torch.zeros_like(c), c)
    return torch.where((pick >= 0.1) & (pick < 0.2), torch.sign(c) * 1e-9, c)


# ------------------------------------------------------------------------------------------------------------ case inputs
def twohot_inputs(M, nb, fam, xf, layout, seed, device="cpu"):
    g = gen(seed, device)
    logits = logit_rows(M, nb, fam, g, device)
    x = twohot_x(M, nb, xf, g, device)
    w = torch.rand(M, generator=g, device=device) + 0.5 if layout == "weight" else None
    return logits, x, w


def kl_inputs(M, G, K, fam, seed, device="cpu"):
    """(post, prior, free_nats).  near_free: posterior = prior + s_m d with s_m bisected so the row's KL is
    free_nats (1 + 1e-3 (-1)^m), a fixed margin on each side of the switch; otherwise free_nats is the middle of the
    widest gap between the KLs of the middle half of the rows, so no row sits on the switch."""
    g = gen(seed, device)
    prior = logit_rows(M, G * K, fam if fam != "near_free" else "s2", g, device)
    if fam == "near_free":
        d = torch.randn(M, G * K, generator=g, device=device, dtype=torch.float64)
        free = 1.0
        want = free * (1 + 1e-3 * (1 - 2 * (torch.arange(M, device=device) % 2)).double())
        lo, hi = torch.zeros(M, 1, dtype=torch.float64, device=device), torch.full((M, 1), 64.0, dtype=torch.float64,
                                                                                  device=device)
        for _ in range(80):
            mid = (lo + hi) / 2
            kl = R.kl_rows64((prior.double() + mid * d).float(), prior, G, K)
            more = kl.unsqueeze(-1) > want.unsqueeze(-1)
            hi, lo = torch.where(more, mid, hi), torch.where(more, lo, mid)
        post = (prior.double() + lo * d).float()
        return post, prior, free
    post = logit_rows(M, G * K, fam, g, device) if fam != "offset" else prior + torch.randn(M, G * K, generator=g,
                                                                                            device=device)
    kl = R.kl_rows64(post, prior, G, K)
    if M == 1:
        return post, prior, float(kl[0]) * 0.5
    srt = kl.sort().values
    lo, hi = M // 4, max(M // 4 + 1, 3 * M // 4)
    i = lo + int((srt[lo + 1:hi + 1] - srt[lo:hi]).argmax())
    return post, prior, float((srt[i] + srt[i + 1]) / 2)


def actor_inputs(M, heads, seed, device="cpu"):
    g = gen(seed, device)
    A = sum(heads)
    raw = torch.cat([logit_rows(M, K, LOGIT_FAMILIES[i % 5] if LOGIT_FAMILIES[i % 5] != "offset" else "s2", g, device)
                     for i, K in enumerate(heads)], 1)
    acts = torch.cat([F.one_hot(torch.randint(0, K, (M,), generator=g, device=device), K).float() for K in heads], 1)
    lam, val = torch.randn(M, generator=g, device=device) * 3, torch.randn(M, generator=g, device=device) * 3
    disc = torch.rand(M, generator=g, device=device)
    mom = torch.tensor([0.3, 2.5], device=device)
    return raw.contiguous(), acts, lam, val, disc, mom, A


def lambda_inputs(H, N, seed, device="cpu"):
    g = gen(seed, device)
    rew, val = torch.randn(H + 1, N, generator=g, device=device), 5 * torch.randn(H + 1, N, generator=g, device=device)
    cl = cont_logits((H + 1, N), g, device)
    tc = (torch.rand(N, generator=g, device=device) > 0.1).float()
    return rew, val, cl, tc


def cont_inputs(M, A, seed, device="cpu"):
    """head = [mean | std_raw]; eps large enough that some actions pass action_clip = 1"""
    g = gen(seed, device)
    head = torch.randn(M, 2 * A, generator=g, device=device) * 2
    eps = torch.randn(M, A, generator=g, device=device) * 1.5
    dact = torch.randn(M, A, generator=g, device=device)
    disc = torch.rand(M, generator=g, device=device)
    return head, eps, dact, disc


CONT_ARGS = (0.1, 1.0, 2.0, 1.0)          # min_std, max_std, init_std, action_clip


# ------------------------------------------------------------------------------------------------------------ emulator
em = EmulOps()


def emul_twohot(logits, x, w, layout, scale=0.25):
    M, nb = logits.shape
    lr, d = torch.empty(M), torch.empty(M, nb)
    em.twohot_loss_grad(logits, x, w, scale, LOW, HIGH, lr, d)
    return {"loss": lr, "grad": d}


CPU_TWOHOT = [c for c, (M, nb, *_) in TWOHOT_CASES.items() if M * nb <= 1 << 18]


@pytest.mark.parametrize("case", CPU_TWOHOT)
def test_emulator_twohot_within_bounds(case):
    M, nb, fam, xf, layout = TWOHOT_CASES[case]
    logits, x, w = twohot_inputs(M, nb, fam, xf, layout, seed=len(case))
    ref, bd = R.twohot_loss(logits, x, w, 0.25, LOW, HIGH)
    m = worst(emul_twohot(logits, x, w, layout), ref, bd)
    out = torch.empty(M)
    em.twohot_mean(logits, LOW, HIGH, out)
    dm = torch.randn(M, generator=gen(1))
    dl = torch.empty(M, nb)
    em.twohot_mean_bwd(logits, dm, LOW, HIGH, dl)
    r2, b2 = R.twohot_mean(logits, LOW, HIGH, dm)
    m.update(worst({"mean": out, "mean_grad": dl}, {"mean": r2["mean"], "mean_grad": r2["grad"]},
                   {"mean": b2["mean"], "mean_grad": b2["grad"]}))
    assert max(m.values()) <= 0.5, m


@pytest.mark.parametrize("case", [c for c, (G, K, _) in KL_CASES.items()])
def test_emulator_kl_within_bounds(case):
    G, K, fam = KL_CASES[case]
    M = 64
    post, prior, free = kl_inputs(M, G, K, fam, seed=len(case))
    ref, bd = R.kl_loss(post, prior, G, K, 0.5, 0.1, free, 1.0, 1.0 / M)
    dp, dq, rows = torch.empty(M, G * K), torch.empty(M, G * K), torch.empty(M, 4)
    em.kl_loss_grad(post, prior, G, K, 0.5, 0.1, free, 1.0, R.f32(1.0 / M), dp, dq, rows)
    m = worst({"rows": rows, "d_post": dp, "d_prior": dq}, ref, bd)
    assert max(m.values()) <= 0.5, m


@pytest.mark.parametrize("unimix", [0.0, 0.01])
@pytest.mark.parametrize("heads", list(ACTOR_HEADS))
def test_emulator_actor_within_bounds(heads, unimix):
    hd = ACTOR_HEADS[heads]
    M = 300
    raw, acts, lam, val, disc, mom, A = actor_inputs(M, hd, seed=len(heads))
    ref, bd = R.actor_loss(raw, acts, lam, val, disc, mom, hd, unimix, 3e-4, 1.0 / M)
    rows, draw = torch.empty(M), torch.empty(M, A)
    em.actor_loss_grad(raw, acts, lam, val, disc, mom, hd, unimix, 3e-4, R.f32(1.0 / M), rows, draw)
    m = worst({"rows": rows, "draw": draw}, ref, bd)
    assert max(m.values()) <= 0.5, m


CPU_LAMBDA = [c for c, (H, N, *_) in LAMBDA_CASES.items() if H * N <= 1 << 16]


@pytest.mark.parametrize("case", CPU_LAMBDA)
def test_emulator_lambda_within_bounds(case):
    H, N, gamma, lmbda = LAMBDA_CASES[case]
    rew, val, cl, tc = lambda_inputs(H, N, seed=len(case))
    lam, disc = torch.empty(H, N), torch.empty(H + 1, N)
    gamma, lmbda = R.f32(gamma), R.f32(lmbda)
    em.lambda_returns(rew, val, cl, tc, gamma, lmbda, lam, disc)
    ref, bd = R.lambda_returns(rew, val, cl, tc, gamma, lmbda)
    m = worst({"lam": lam, "discount": disc}, ref, bd)
    ent = torch.randn(H * N, generator=gen(2))
    mom = torch.tensor([0.5, 3.0])
    dv, dr, rows = torch.empty(H + 1, N), torch.empty(H + 1, N), torch.empty(H, N)
    em.lambda_returns_bwd(cl, disc, mom, lam, val, ent, gamma, lmbda, 3e-4, R.f32(1.0 / (H * N)), dv, dr, rows)
    ref, bd = R.lambda_returns_bwd(cl, disc, mom, lam, val, ent, gamma, lmbda, 3e-4, 1.0 / (H * N))
    m.update(worst({"rows": rows, "d_val": dv, "d_rew": dr}, ref, bd))
    assert max(m.values()) <= 0.5, m


@pytest.mark.parametrize("A", CONT_AS)
def test_emulator_cont_action_within_bounds(A):
    M = 777
    head, eps, dact, disc = cont_inputs(M, A, seed=A)
    act, ent, dh = torch.empty(M, A), torch.empty(M), torch.empty(M, 2 * A)
    em.cont_action_fwd(head, eps, act, ent, *CONT_ARGS)
    em.cont_action_bwd(head, eps, dact, disc, dh, *CONT_ARGS, -0.01)
    ref, bd = R.cont_action(head, eps, *CONT_ARGS, dact, disc, -0.01)
    m = worst({"action": act, "ent": ent, "dhead": dh}, ref, bd)
    assert max(m.values()) <= 0.5, m


def test_emulator_bce_mse_reductions_within_bounds():
    g = gen(5)
    M, P = 4097, 77
    l = torch.cat([torch.randn(M, generator=g) * 3, torch.tensor([0.0, 1e-9, -1e-9, 20.0, -20.0, 40.0, -40.0])])
    y = (torch.rand(l.numel(), generator=g) > 0.5).float()
    lr, dl = torch.empty(l.numel()), torch.empty(l.numel())
    em.bce_loss_grad(l, y, 1.0, R.f32(1.0 / M), lr, dl)
    ref, bd = R.bce(l, y, 1.0, 1.0 / M)
    m = worst({"loss": lr, "grad": dl}, ref, bd)
    pred, tgt = torch.randn(M, P, generator=g), torch.randn(M, P, generator=g)
    lr, gr = torch.empty(M), torch.empty(M, P)
    em.mse_loss_grad(pred, tgt, R.f32(1.0 / M), lr, gr)
    ref, bd = R.mse(pred, tgt, 1.0 / M)
    m.update({"mse_" + k: v for k, v in worst({"loss": lr, "grad": gr}, ref, bd).items()})
    o = torch.empty(P)
    em.sum_rows(pred, o, 0.5)
    s, b = R.sum_rows(pred, 0.5)
    m["sum_rows"] = ratio(o, s, b)
    o = torch.empty(1)
    em.weighted_mean(pred[:, 0].contiguous(), tgt[:, 0].contiguous(), 0.1, o)
    s, b = R.weighted_mean(pred[:, 0], tgt[:, 0], 0.1)
    m["weighted_mean"] = ratio(o, s.reshape(1), b.reshape(1))
    assert max(m.values()) <= 0.5, m


# ------------------------------------------------------------------------------------------------------------ moments
def moments_inputs(n, family, seed, device="cpu"):
    """random N(0, 4); ties: 7 distinct values; equal: one value; zeros: mixed +-0 with a few +-1; inf_rank: 0..n-2
    and +inf (rank q (n - 1) is integral for q = 0.95 when n = 21); nan: one NaN among random values"""
    g = gen(seed, device)
    if family == "random":
        return 4 * torch.randn(n, generator=g, device=device)
    if family == "ties":
        return torch.randint(-3, 4, (n,), generator=g, device=device).float()
    if family == "equal":
        return torch.full((n,), 2.5, device=device)
    if family == "zeros":
        s = torch.where(torch.rand(n, generator=g, device=device) < 0.5, -1.0, 1.0)
        z = s * 0.0
        z[: max(1, n // 100)] = s[: max(1, n // 100)]
        return z[torch.randperm(n, generator=g, device=device)]
    if family == "inf_rank":
        x = torch.arange(n, device=device, dtype=torch.float32)
        x[-1] = math.inf
        x[0] = -math.inf
        return x[torch.randperm(n, generator=g, device=device)]
    assert family == "nan", family
    x = torch.randn(n, generator=g, device=device)
    x[int(torch.randint(0, n, (1,), generator=g, device=device))] = math.nan
    return x


def quantile_ok(got, want):
    """equal (NaN = NaN, -0 = +0) or within 2 ulp of fp32 torch.quantile"""
    g, w = float(got), float(want)
    if math.isnan(w) or math.isnan(g):
        return math.isnan(w) and math.isnan(g)
    if g == w:
        return True
    ulp = float(torch.nextafter(torch.tensor(abs(w)), torch.tensor(math.inf)) - abs(w))
    return abs(g - w) <= 2 * ulp


def test_emulator_moments_matches_quantile_at_the_edges():
    """EmulOps is fp32 torch.quantile itself; this pins the families' torch answers the kernel is held to: NaN for a
    NaN anywhere, and the integral-rank element itself (not NaN) next to +-inf"""
    for fam, q, want in (("inf_rank", 0.95, 19.0), ("inf_rank", 0.05, 1.0), ("nan", 0.5, math.nan)):
        x = moments_inputs(21, fam, seed=3)
        assert quantile_ok(torch.quantile(x, q), want), (fam, q)
    lo, hi = R.quantiles32(torch.tensor([-3e38, 3e38]), 0.0, 1.0)
    assert float(lo) == R.f32(-3e38) and float(hi) == R.f32(3e38)
    (st, out), _, _ = R.moments(moments_inputs(21, "nan", 3), torch.zeros(2), 0.99, 1e8, 0.05, 0.95)
    assert bool(st.isnan().all()) and bool(out.isnan().all())


# ------------------------------------------------------------------------------------------------------------ fixture
def _compare_fixture(fx):
    """loss_ref on the fixture's inputs against the reference's float64 outputs"""
    worst_err = {}
    for name, case in fx.items():
        got = reference_outputs(name, case["args"])
        for k, want in case["out"].items():
            w = want.double()
            err = float((got[k].double() - w).abs().max()) / (1.0 + float(w.abs().max()))
            worst_err[f"{name}.{k}"] = err
    return worst_err


def reference_outputs(name, a):
    """loss_ref's outputs for one fixture entry, keyed like the fixture"""
    if name == "twohot":
        o, _ = R.twohot_loss(a["logits"], a["x"], a["weight"], a["scale"], LOW, HIGH)
        m, _ = R.twohot_mean(a["logits"], LOW, HIGH, a["d_mean"])
        return {"loss": o["loss"], "grad": o["grad"], "mean": m["mean"], "mean_grad": m["grad"]}
    if name == "mse":
        return R.mse(a["pred"], a["target"], a["scale"])[0]
    if name == "bce":
        return R.bce(a["logit"], a["target"], a["loss_scale"], a["scale"])[0]
    if name == "kl":
        return R.kl_loss(a["post"], a["prior"], a["groups"], a["K"], 0.5, 0.1, a["free"], 1.0, a["scale"])[0]
    if name == "lambda":
        o, _ = R.lambda_returns(a["rew"], a["val"], a["cont_logit"], a["true_cont"], a["gamma"], a["lmbda"])
        b, _ = R.lambda_returns_bwd(a["cont_logit"], o["discount"].float(), a["moments"], o["lam"].float(), a["val"],
                                    a["ent"], a["gamma"], a["lmbda"], a["ent_coef"], a["scale"])
        return {"lam": o["lam"], "discount": o["discount"], "rows": b["rows"], "d_val": b["d_val"], "d_rew": b["d_rew"]}
    if name == "moments":
        (st, out), _, _ = R.moments(a["x"], a["state"], a["decay"], a["max"], 0.05, 0.95)
        return {"state": st, "out": out}
    if name.startswith("actor"):
        return R.actor_loss(a["raw"], a["actions"], a["lam"], a["val"], a["discount"], a["moments"], a["heads"],
                            a["unimix"], a["ent_coef"], a["scale"])[0]
    assert name == "cont", name
    return R.cont_action(a["head"], a["eps"], *a["cfg"], a["d_action"], a["discount"], a["ent_scale"])[0]


def test_reference_matches_the_committed_fixture():
    fx = torch.load(GOLDEN, weights_only=False)
    errs = _compare_fixture(fx)
    assert max(errs.values()) <= 1e-12, errs


def test_reference_matches_the_reference_live():
    from oracle.ref_harness import reference_available

    if not reference_available():
        pytest.skip("reference package not present")
    from oracle.make_golden_loss_ref import make

    errs = _compare_fixture(make())
    assert max(errs.values()) <= 1e-12, errs


# ------------------------------------------------------------------------------------------------------------ mutants
def fp32_twohot(logits, x, scale, mutant=None):
    """the two-hot gradient (softmax - target) scale in fp32, with one defect switched on"""
    M, nb = logits.shape
    t, below, above, _ = R.twohot_target(x, nb, LOW, HIGH)
    t = t.float()
    if mutant == "swapped_weights":
        r, lo, hi = torch.arange(M), below.squeeze(-1), above.squeeze(-1)
        w_lo, w_hi = t[r, lo], t[r, hi]
        same = lo == hi
        t = torch.zeros_like(t)
        t[r, lo] += torch.where(same, 0.5, w_hi)
        t[r, hi] += torch.where(same, 0.5, w_lo)
    if mutant == "no_max_shift":
        e = torch.exp(logits)
        p = e / e.sum(-1, keepdim=True)
    else:
        p = torch.softmax(logits, -1)
    return {"grad": (p - t) * scale}


def fp32_mean_bwd(logits, dm, mutant=None):
    nb = logits.shape[-1]
    bins = torch.linspace(LOW, HIGH, nb)
    p = torch.softmax(logits, -1)
    m = (p * bins).sum(-1, keepdim=True)
    amp = torch.exp(m) if mutant == "exp_m_not_abs" else torch.exp(m.abs())
    return dm.reshape(-1, 1) * amp * p * (bins - m)


def fp32_kl(post, prior, G, K, free, scale, mutant=None):
    M = post.shape[0]
    dp, dq, rows = torch.empty(M, G * K), torch.empty(M, G * K), torch.empty(M, 4)
    em.kl_loss_grad(post, prior, G, K, 0.5, 0.1, free, 1.0, scale, dp, dq, rows)
    if mutant == "no_klg_centring":
        lp = post.reshape(M, G, K).log_softmax(-1)
        lq = prior.reshape(M, G, K).log_softmax(-1)
        live = (rows[:, 0] > free).float().reshape(M, 1, 1) * scale
        dp = (0.1 * live * lp.exp() * (lp - lq)).reshape(M, -1)
    return {"rows": rows, "d_post": dp, "d_prior": dq}


def fp32_actor(raw, acts, lam, val, disc, mom, heads, unimix, ent_coef, scale, mutant=None):
    M = raw.shape[0]
    adv = (lam - mom[0]) / mom[1] - (val - mom[0]) / mom[1]
    draw = torch.empty_like(raw)
    o = 0
    for K in heads:
        x = raw[:, o:o + K]
        s = torch.softmax(x, -1)
        pm = (1 - unimix) * s + unimix / K
        mix = torch.log(pm.clamp(R.FP32_EPS, 1 - R.FP32_EPS))
        lg = mix - torch.logsumexp(mix, -1, keepdim=True)
        p = torch.exp(lg)
        a = acts[:, o:o + K].argmax(-1)
        ent = -(p * lg).sum(-1, keepdim=True)
        dent = -p * lg if mutant == "entropy_grad_without_ent" else -p * (lg + ent)
        g = (-(scale * disc)).unsqueeze(-1) * (adv.unsqueeze(-1) * (F.one_hot(a, K).float() - p) + ent_coef * dent)
        if unimix > 0:
            ds = g * (1 - unimix) / (s if mutant == "unimix_divides_by_s" else pm)
            draw[:, o:o + K] = s * (ds - (s * ds).sum(-1, keepdim=True))
        else:
            draw[:, o:o + K] = g
        o += K
    rows = torch.empty(M)
    em.actor_loss_grad(raw, acts, lam, val, disc, mom, heads, unimix, ent_coef, scale, rows, torch.empty_like(raw))
    return {"rows": rows, "draw": draw}


def fp32_lambda_bwd(cl, disc, mom, lam, val, ent, gamma, lmbda, ent_coef, scale, mutant=None):
    H, N = lam.shape
    dv, dr, rows = torch.empty(H + 1, N), torch.empty(H + 1, N), torch.empty(H, N)
    em.lambda_returns_bwd(cl, disc, mom, lam, val, ent, gamma, lmbda, ent_coef, scale, dv, dr, rows)
    if mutant == "G_one_step_late":
        c = (torch.sigmoid(cl) > 0.5).float() * gamma
        G = torch.zeros(N)
        dr.zero_()
        for t in range(H):
            dr[t + 1] = G                                    # the carry before this step's update
            G = -scale * disc[t] / mom[1] + (c[t] * lmbda * G if t > 0 else 0.0)
    return {"rows": rows, "d_val": dv, "d_rew": dr}


def fp32_bce(l, y, loss_scale, scale, mutant=None):
    lr, dl = torch.empty_like(l), torch.empty_like(l)
    em.bce_loss_grad(l, y, loss_scale, scale, lr, dl)
    if mutant == "naive_log_sigmoid":
        s = torch.sigmoid(l)
        lr = -loss_scale * (y * torch.log(s) + (1 - y) * torch.log(1 - s))
    return {"loss": lr, "grad": dl}


def fp32_cont_bwd(head, eps, dact, disc, mutant=None):
    M, A = eps.shape
    dh = torch.empty(M, 2 * A)
    em.cont_action_bwd(head, eps, dact, disc, dh, *CONT_ARGS, -0.01)
    if mutant == "through_the_clip_factor":
        h = head.clone().requires_grad_(True)
        mn, mx, init, clip = CONT_ARGS
        std = (mx - mn) * torch.sigmoid(h[:, A:] + init) + mn
        a = torch.tanh(h[:, :A]) + std * eps
        a = a * (clip / torch.maximum(torch.full_like(a, clip), a.abs()))          # not detached
        ent = (R.HALF_LOG_2PI_E + std.log()).sum(-1)
        ((a * dact).sum() + (-0.01 * disc * ent).sum()).backward()
        dh = h.grad
    return {"dhead": dh}


def _twohot_mutant(mutant):
    M, nb = 200, 255
    logits, x, _ = twohot_inputs(M, nb, "offset" if mutant == "no_max_shift" else "s2", "cont", "plain", seed=11)
    ref, bd = R.twohot_loss(logits, x, None, 0.25, LOW, HIGH)
    ref, bd = {"grad": ref["grad"]}, {"grad": bd["grad"]}
    return worst(fp32_twohot(logits, x, 0.25), ref, bd), worst(fp32_twohot(logits, x, 0.25, mutant), ref, bd)


def _mean_mutant(mutant):
    M, nb = 200, 255
    logits = logit_rows(M, nb, "s2", gen(12)) - 0.05 * torch.arange(nb).float()     # means well below 0
    dm = torch.randn(M, generator=gen(13))
    ref, bd = R.twohot_mean(logits, LOW, HIGH, dm)
    assert bool((ref["mean"] < -1).all())
    return (worst({"grad": fp32_mean_bwd(logits, dm)}, {"grad": ref["grad"]}, {"grad": bd["grad"]}),
            worst({"grad": fp32_mean_bwd(logits, dm, mutant)}, {"grad": ref["grad"]}, {"grad": bd["grad"]}))


def _kl_mutant(mutant):
    G, K, M = 8, 32, 64
    post, prior, free = kl_inputs(M, G, K, "s2", seed=14)
    ref, bd = R.kl_loss(post, prior, G, K, 0.5, 0.1, free, 1.0, 1.0 / M)
    s = R.f32(1.0 / M)
    return (worst(fp32_kl(post, prior, G, K, free, s), ref, bd),
            worst(fp32_kl(post, prior, G, K, free, s, mutant), ref, bd))


def _actor_mutant(mutant):
    """the entropy term's +ent is a constant shift per head, which the softmax Jacobian of the unimix chain removes:
    that defect shows without unimix only"""
    M, heads = 300, (18,)
    unimix = 0.0 if mutant == "entropy_grad_without_ent" else 0.01
    raw, acts, lam, val, disc, mom, _ = actor_inputs(M, heads, seed=15)
    ref, bd = R.actor_loss(raw, acts, lam, val, disc, mom, heads, unimix, 3e-4, 1.0 / M)
    s = R.f32(1.0 / M)
    return (worst(fp32_actor(raw, acts, lam, val, disc, mom, heads, unimix, 3e-4, s), ref, bd),
            worst(fp32_actor(raw, acts, lam, val, disc, mom, heads, unimix, 3e-4, s, mutant), ref, bd))


def _lambda_mutant(mutant):
    H, N = 15, 129
    rew, val, cl, tc = lambda_inputs(H, N, seed=16)
    gamma, lmbda = R.f32(0.997), R.f32(0.95)
    o, _ = R.lambda_returns(rew, val, cl, tc, gamma, lmbda)
    lam, disc = o["lam"].float(), o["discount"].float()
    ent, mom, s = torch.randn(H * N, generator=gen(17)), torch.tensor([0.5, 3.0]), R.f32(1.0 / (H * N))
    ref, bd = R.lambda_returns_bwd(cl, disc, mom, lam, val, ent, gamma, lmbda, 3e-4, s)
    return (worst(fp32_lambda_bwd(cl, disc, mom, lam, val, ent, gamma, lmbda, 3e-4, s), ref, bd),
            worst(fp32_lambda_bwd(cl, disc, mom, lam, val, ent, gamma, lmbda, 3e-4, s, mutant), ref, bd))


def _bce_mutant(mutant):
    g = gen(18)
    l = torch.cat([torch.randn(100, generator=g) * 3, torch.tensor([18.0, 25.0, -18.0, -25.0])])
    y = torch.cat([(torch.rand(100, generator=g) > 0.5).float(), torch.tensor([0.0, 0.0, 1.0, 1.0])])
    ref, bd = R.bce(l, y, 1.0, 0.01)
    return worst(fp32_bce(l, y, 1.0, 0.01), ref, bd), worst(fp32_bce(l, y, 1.0, 0.01, mutant), ref, bd)


def _cont_mutant(mutant):
    head, eps, dact, disc = cont_inputs(300, 6, seed=19)
    ref, bd = R.cont_action(head, eps, *CONT_ARGS, dact, disc, -0.01)
    ref, bd = {"dhead": ref["dhead"]}, {"dhead": bd["dhead"]}
    return (worst(fp32_cont_bwd(head, eps, dact, disc), ref, bd),
            worst(fp32_cont_bwd(head, eps, dact, disc, mutant), ref, bd))


MUTANTS = {
    "no_max_shift": _twohot_mutant,                 # softmax of the +1000 family without the max shift
    "swapped_weights": _twohot_mutant,              # two-hot weights on the wrong bins
    "exp_m_not_abs": _mean_mutant,                  # twohot_mean_bwd with exp(m) for exp(|m|), negative means
    "no_klg_centring": _kl_mutant,                  # the KL d_post without its - klg centring
    "unimix_divides_by_s": _actor_mutant,           # the unimix chain rule dividing by s instead of pm
    "entropy_grad_without_ent": _actor_mutant,      # the entropy gradient without its + ent term
    "G_one_step_late": _lambda_mutant,              # lambda_returns_bwd writing G one step late
    "naive_log_sigmoid": _bce_mutant,               # bce as -log sigmoid(l), |l| > 17
    "through_the_clip_factor": _cont_mutant,        # cont_action_bwd differentiating the clip factor
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_bounds_reject_subtly_wrong_implementations(mutant):
    honest, wrong = MUTANTS[mutant](mutant)
    assert max(honest.values()) <= 0.5, honest
    assert max(wrong.values()) >= 4.0, wrong
