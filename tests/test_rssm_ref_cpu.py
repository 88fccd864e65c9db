"""The float64 reference of the RSSM sampling, gate and masking kernels (oracle/rssm_ref.py) and the executable
specification of the device noise (oracle/philox_ref.py), on the CPU.

  - the references follow the reference's semantics: rssm_ref reproduces, to ~1e-12, a fixture made by running the
    reference's own classes in float64 with autograd (oracle/make_golden_rssm_ref.py -> tests/golden/dv3_rssm_ref.pt),
    re-run live when the reference package is importable; philox_ref reproduces the Random123 known-answer vectors;
  - an honest fp32 implementation (EmulOps, the kernels' specification, fed the spec's noise) stays within every bound
    with 2x headroom at each GPU case that fits on the CPU (the cases of tests/test_gpu_rssm_precision.py are here);
  - fp32 implementations with one plausible defect each exceed their bound by at least 4x, or fail the sample criterion;
  - the spec's noise is distributed as specified (fixed seeds: deterministic).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy import stats

from oracle import philox_ref as P
from oracle import rssm_ref as R
from oracle.ops_emul import EmulOps
from tests.test_loss_ref_cpu import LOGIT_FAMILIES, gen, logit_rows, ratio, worst

GOLDEN = "tests/golden/dv3_rssm_ref.pt"
U = R.U
em = EmulOps()

# ------------------------------------------------------------------------------------------------------------ cases
# The GPU file runs every case; this file holds EmulOps to the same bounds at the ones that fit on the CPU.
CAT_ROWS = (1, 7, 8, 9, 1024, 15360)
CAT_GK = ((32, 32), (1, 1), (1, 2), (6, 5), (4, 31), (4, 33), (2, 40), (2, 64), (1, 1000))
UNIMIXES = (0.0, 0.01, 0.5)
BWD_MODES = ("dz", "dmix", "both")
CAT_LAYOUTS = ("plain", "strided", "mix_only", "sample_only")


def _cat_cases():
    out, k = {}, 0
    for G, K in CAT_GK:
        for M in CAT_ROWS:
            fam = LOGIT_FAMILIES[k % 5]
            unimix, mode = UNIMIXES[k % 3], BWD_MODES[(k // 3) % 3]
            layout, noisy = CAT_LAYOUTS[(k + k // 4) % 4], (k // 2) % 2 == 1
            out[f"G{G}_K{K}_M{M}_{fam}_u{unimix}_{mode}_{layout}{'_noise' if noisy else ''}"] = \
                (M, G, K, fam, unimix, mode, layout, noisy)
            k += 1
    return out


CAT_CASES = _cat_cases()
HEAD_KINS = (4, 36, 128, 512, 1020, 1024)
HEAD_AS = (1, 2, 17, 31, 32)
HEAD_ROWS = (1, 9, 1024, 15360)
HEAD_CASES = {f"Kin{Kin}_A{A}_M{HEAD_ROWS[k % 4]}_{'bias' if k % 2 else 'nobias'}_{'noise' if (k // 2) % 2 else 'mode'}":
              (Kin, A, HEAD_ROWS[k % 4], k % 2 == 1, (k // 2) % 2 == 1, (0.01, 0.0)[(k // 4) % 2])
              for k, (Kin, A) in enumerate((Kin, A) for Kin in HEAD_KINS for A in HEAD_AS)}
GRU_SHAPES = ((1, 1), (3, 7), (16, 512), (1024, 24), (64, 4096))
GRU_FAMILIES = ("n1", "n30", "sat100")
GRU_CASES = {f"M{M}_R{Rr}_{fam}": (M, Rr, fam) for M, Rr in GRU_SHAPES for fam in GRU_FAMILIES}
MASK_SHAPES = ((1, 1), (16, 100), (1024, 1536))
MASK_CASES = {f"M{M}_C{C}_{first}": (M, C, first) for M, C in MASK_SHAPES for first in ("zeros", "ones", "mixed")}
OL_S, OL_K, OL_A, OL_N = (1, 32, 64), (1, 32, 33, 40), (0, 1, 32), (1, 255, 256, 257, 1536)
OL_CASES = {f"S{S}_K{K}_A{A}_N{OL_N[k % 5]}": (S, K, A, OL_N[k % 5])
            for k, (S, K, A) in enumerate((S, K, A) for S in OL_S for K in OL_K for A in OL_A)}
FILL_NS = (1, 2, 3, 4, 5, 1023, (1 << 20) + 3, 3 * (1 << 20) + 1)
FILL_COUNTERS = (None, 0, 1, (1 << 31) - 1)
FILL_SEEDS = ((1234, 0), (0x9E3779B97F4A7C15, 7), (42, (1 << 32) - 1))       # (seed, stream id)
FILL_CASES = {f"n{n}_c{FILL_COUNTERS[k % 4]}_s{k % 3}": (n, FILL_COUNTERS[k % 4], *FILL_SEEDS[k % 3])
              for k, n in enumerate(FILL_NS)}
CLAMP_EDGE = (1e-9, 64)            # unimix, K: u / K < FP32_EPS, so the unimix clamp is reached from below


# ------------------------------------------------------------------------------------------------------------ inputs
def spec_exponential(shape, seed, stream, counter=0, device="cpu"):
    n = int(np.prod(shape))
    return torch.from_numpy(P.exponential(n, seed, stream, counter)[0].astype(np.float32)).reshape(shape).to(device)


def cat_inputs(M, G, K, fam, noisy, seed, device="cpu"):
    g = gen(seed, device)
    raw = logit_rows(M * G, K, fam, g, device).reshape(M, G * K)
    noise = spec_exponential((M, G * K), seed, 0, device=device) if noisy else None
    dz = torch.randn(M, G * K, generator=g, device=device)
    dmix = torch.randn(M, G * K, generator=g, device=device)
    return raw, noise, dz, dmix


def bwd_args(mode, dz, dmix):
    return (dz if mode != "dmix" else None), (dmix if mode != "dz" else None)


def head_inputs(M, Kin, A, bias, noisy, seed, device="cpu"):
    g = gen(seed, device)
    X = torch.randn(M, Kin, generator=g, device=device)
    W = torch.randn(A, Kin, generator=g, device=device) / math.sqrt(Kin) * 3
    b = torch.randn(A, generator=g, device=device) if bias else None
    noise = spec_exponential((M, A), seed, 2, device=device) if noisy else None
    return X, W, b, noise


def gru_inputs(M, Rr, fam, seed, device="cpu"):
    """n1 / n30: G ~ N(0, 1) / N(0, 30); sat100: G = +-100 (expf(-x) overflows to inf for x = -100)"""
    g = gen(seed, device)
    G = torch.randn(M, 3 * Rr, generator=g, device=device)
    if fam == "n30":
        G = 30 * G
    elif fam == "sat100":
        G = torch.where(G > 0, 100.0, -100.0)
    return G, torch.randn(M, Rr, generator=g, device=device), torch.randn(M, Rr, generator=g, device=device)


def mask_inputs(M, C, first, seed, device="cpu"):
    g = gen(seed, device)
    f = {"zeros": torch.zeros(M, device=device), "ones": torch.ones(M, device=device),
         "mixed": (torch.rand(M, generator=g, device=device) < 0.5).float()}[first]
    return (torch.randn(M, C, generator=g, device=device), torch.randn(C, generator=g, device=device), f,
            torch.randn(M, C, generator=g, device=device), torch.randn(C, generator=g, device=device))


def ol_inputs(M, S, K, A, N, seed, device="cpu"):
    """z: S one-hot groups, every third group's hot class in the second ballot chunk (>= 32) when K > 32"""
    g = gen(seed, device)
    hot = torch.randint(0, K, (M, S), generator=g, device=device)
    if K > 32:
        hot[:, ::3] = 32 + torch.randint(0, K - 32, (M, (S + 2) // 3), generator=g, device=device)
    z = F.one_hot(hot, K).float().reshape(M, S * K)
    act = torch.randn(M, A, generator=g, device=device) if A else None
    WT = torch.randn(S * K + A, N, generator=g, device=device)
    return z, act, WT


def tie_rows(K, device="cpu"):
    """rows of one group whose exact fp32 ties decide the mode: (logits [n, K], expected class [n]).  Classes c and
    c + 32 (one lane of the strided kernel), classes 3 and 17 (two lanes), the whole row (-> class 0)"""
    rows, want = [], []
    base = torch.linspace(-3.0, -1.0, K, device=device)
    rows.append(torch.zeros(K, device=device))
    want.append(0)
    if K > 17:
        r = base.clone()
        r[3] = r[17] = 2.0
        rows.append(r)
        want.append(3)
    if K > 32:
        c = min(5, K - 33)
        r = base.clone()
        r[c] = r[c + 32] = 2.0
        rows.append(r)
        want.append(c)
    return torch.stack(rows), torch.tensor(want, device=device)


# ------------------------------------------------------------------------------------------------------------ emulator
def emul_cat(raw, noise, unimix, G, K):
    M = raw.shape[0]
    oh, mx = torch.empty(M, G * K), torch.empty(M, G * K)
    em.cat_sample(raw, noise, R.f32(unimix), G, K, oh, mx)
    return oh, mx


def cat_margins(raw, noise, unimix, G, K, onehot, mix):
    ref, bd = R.cat_sample(raw, noise, unimix, G, K)
    fmt, w, nonarg = R.judge_sample(onehot, ref, noise)
    assert fmt, "not an exact one-hot"
    return {"mix": ratio(mix, ref["mix"], bd["mix"]), "sample": w}, nonarg


CPU_CAT = [c for c, (M, G, K, *_) in CAT_CASES.items() if M * G * K <= 1 << 18]


@pytest.mark.parametrize("case", CPU_CAT)
def test_emulator_cat_sample_within_bounds(case):
    M, G, K, fam, unimix, mode, _, noisy = CAT_CASES[case]
    raw, noise, dz, dmix = cat_inputs(M, G, K, fam, noisy, seed=len(case))
    oh, mx = emul_cat(raw, noise, unimix, G, K)
    m, _ = cat_margins(raw, noise, unimix, G, K, oh, mx)
    a, b = bwd_args(mode, dz, dmix)
    dr = torch.empty(M, G * K)
    em.cat_sample_bwd(raw, a, b, R.f32(unimix), G, K, dr)
    ref, bd = R.cat_sample_bwd(raw, a, b, unimix, G, K)
    m["draw"] = ratio(dr, ref, bd)
    assert max(m.values()) <= 0.5, m


def test_emulator_cat_sample_bwd_at_the_clamp_edge():
    """unimix 1e-9, K = 64: u / K < FP32_EPS, so pm crosses the clamp's lower edge inside the dominant family"""
    unimix, K = CLAMP_EDGE
    raw, _, dz, dmix = cat_inputs(512, 1, K, "dominant", False, seed=3)
    _, _, pm, _, _, _ = R.unimix_fwd_err(raw.double(), R.f32(unimix))
    assert bool((pm < R.FP32_EPS).any()) and bool((pm > R.FP32_EPS).any())
    for mode in BWD_MODES:
        a, b = bwd_args(mode, dz, dmix)
        dr = torch.empty_like(raw)
        em.cat_sample_bwd(raw, a, b, R.f32(unimix), 1, K, dr)
        ref, bd = R.cat_sample_bwd(raw, a, b, unimix, 1, K)
        assert ratio(dr, ref, bd) <= 0.5, mode


@pytest.mark.parametrize("K", [32, 40, 1000])
def test_emulator_ties_pick_the_lowest_index(K):
    rows, want = tie_rows(K)
    oh, _ = emul_cat(rows, None, 0.0, 1, K)
    assert torch.equal(oh.argmax(-1), want)


CPU_HEAD = [c for c, (Kin, A, M, *_) in HEAD_CASES.items() if M * Kin <= 1 << 20]


@pytest.mark.parametrize("case", CPU_HEAD)
def test_emulator_head_sample_within_bounds(case):
    Kin, A, M, bias, noisy, unimix = HEAD_CASES[case]
    X, W, b, noise = head_inputs(M, Kin, A, bias, noisy, seed=len(case))
    raw, oh = torch.empty(M, A), torch.empty(M, A)
    em.head_sample(X, W, b, noise, R.f32(unimix), raw, oh)
    r64, br = R.head_raw(X, W, b)
    m = {"raw": ratio(raw, r64, br)}
    ref, _ = R.cat_sample(raw, noise, unimix, 1, A)
    fmt, m["sample"], _ = R.judge_sample(oh, ref, noise)
    assert fmt and max(m.values()) <= 0.5, m


def emul_gru(G, Hin, dH):
    h, dG, dHin = torch.empty_like(Hin), torch.empty_like(G), torch.empty_like(Hin)
    em.gru_gate_fwd(G, Hin, h)
    em.gru_gate_bwd(G, Hin, dH, dG, dHin)
    return {"h": h, "dG": dG, "dHin": dHin}


@pytest.mark.parametrize("case", list(GRU_CASES))
def test_emulator_gru_gate_within_bounds(case):
    M, Rr, fam = GRU_CASES[case]
    G, Hin, dH = gru_inputs(M, Rr, fam, seed=len(case))
    ref, bd = R.gru_gate(G, Hin, dH)
    m = worst(emul_gru(G, Hin, dH), ref, bd)
    assert max(m.values()) <= 0.5, m


@pytest.mark.parametrize("case", list(MASK_CASES))
def test_emulator_masks_exact_and_within_bounds(case):
    M, C, first = MASK_CASES[case]
    prev, init, f, dIn, d0 = mask_inputs(M, C, first, seed=len(case))
    out = torch.empty(M, C)
    em.mask_mix(prev, init, f, out)
    assert torch.equal(out.double(), R.mask_mix(prev, init, f))
    em.mask_rows(prev, f, out)
    assert torch.equal(out.double(), R.mask_mix(prev, None, f))
    for start in (None, torch.zeros(C), d0):
        dp, di = torch.empty(M, C), None if start is None else start.clone()
        em.mask_bwd(dIn, f, dp, di)
        rp, ri, bi = R.mask_bwd(dIn, f, start)
        assert torch.equal(dp.double(), rp)
        if start is not None:
            assert ratio(di, ri, bi) <= 0.5


CPU_OL = [c for c, (S, K, A, N) in OL_CASES.items() if N <= 257]


@pytest.mark.parametrize("case", CPU_OL)
def test_emulator_onehot_linear_within_bounds(case):
    S, K, A, N = OL_CASES[case]
    M = 64
    z, act, WT = ol_inputs(M, S, K, A, N, seed=len(case))
    out = torch.empty(M, N)
    em.onehot_linear(z, act if A else torch.empty(M, 0), WT, out, S, K)
    ref, bd = R.onehot_linear(z, act, WT, S, K)
    assert ratio(out, ref, bd) <= 0.5


def fp32_exponential(u, mutant=None):
    """the kernel's transform in fp32, each operation correctly rounded"""
    u32 = torch.from_numpy(u).float()
    return torch.clamp(-torch.log(u32), min=P.EXP_FLOOR).double().numpy()


def fp32_normal(u1, u2, mutant=None):
    r = torch.sqrt(-2 * torch.log(torch.from_numpy(u1).float()))
    c, s = P._cospi_sinpi(2.0 * u2)
    if mutant == "cos_sin_swapped":
        c, s = s, c
    trig = np.where(np.arange(u1.size) % 2 == 0, c, s)           # element 4 i + j: cos for even j, sin for odd
    return (r * torch.from_numpy(trig).float()).double().numpy()


def np_ratio(got, want, bound):
    d = np.abs(got - want)
    return float(np.max(np.where(d == 0, 0.0, d / bound))) if d.size else 0.0


CPU_FILL = [c for c, (n, *_) in FILL_CASES.items() if n <= (1 << 20) + 3]


@pytest.mark.parametrize("case", CPU_FILL)
def test_fp32_noise_transforms_within_bounds(case):
    n, ctr, seed, stream = FILL_CASES[case]
    v, b, u = P.exponential(n, seed, stream, ctr or 0)
    v2, b2, u1, u2 = P.normal(n, seed, stream, ctr or 0)
    m = {"exp": np_ratio(fp32_exponential(u), v, b), "normal": np_ratio(fp32_normal(u1, u2), v2, b2)}
    assert max(m.values()) <= 0.5, m
    assert v.max() <= P.EXP_MAX + 1e-9 and np.abs(v2).max() <= P.NORMAL_MAX + 1e-9


def test_case_lists_straddle_the_kernel_switches():
    """cat_sample runs one class per lane for K <= 32 and a strided loop above; onehot_linear ballots 32 classes at
    a time; the fills run a grid-stride loop of 132 * 8 blocks of 256 threads, four elements each"""
    ks = {K for _, K in CAT_GK}
    assert 32 in ks and 33 in ks and 1 in ks and max(ks) > 64
    assert {32, 33}.issubset(OL_K) and max(n for n, *_ in FILL_CASES.values()) > 132 * 8 * 256 * 4
    assert any(s == (1 << 32) - 1 for *_, s in FILL_CASES.values())
    assert any(seed >> 32 for _, _, seed, _ in FILL_CASES.values())


# ------------------------------------------------------------------------------------------------------------ fixture
def _compare_fixture(fx):
    errs = {}
    for name, case in fx.items():
        a, out = case["args"], case["out"]
        if name.startswith("cat"):
            G, K, u = a["G" if "G" in a else "groups"], a["K"], a["unimix"]
            ref, _ = R.cat_sample(a["raw"], None, u, G, K)
            got = {"mix": ref["mix"], "probs": ref["p"].reshape(out["probs"].shape),
                   "mode": F.one_hot(ref["r"].argmax(-1), K).double().reshape(out["mode"].shape)}
            for mode in BWD_MODES:
                got[f"draw_{mode}"] = R.cat_sample_bwd(a["raw"], *bwd_args(mode, a["dz"], a["dmix"]), u, G, K)[0]
        else:
            ref, _ = R.gru_gate(a["G"], a["Hin"], a["dH"])
            got = ref
        for k, want in out.items():
            w = want.double()
            errs[f"{name}.{k}"] = float((got[k].double().reshape(w.shape) - w).abs().max()) / (1 + float(w.abs().max()))
    return errs


def test_reference_matches_the_committed_fixture():
    errs = _compare_fixture(torch.load(GOLDEN, weights_only=False))
    assert max(errs.values()) <= 1e-12, errs


def test_reference_matches_the_reference_live():
    from oracle.ref_harness import reference_available

    if not reference_available():
        pytest.skip("reference package not present")
    from oracle.make_golden_rssm_ref import make

    errs = _compare_fixture(make())
    assert max(errs.values()) <= 1e-12, errs


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
], ids=["zero", "ones", "pi"])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(w) for w in P.philox4x32_10(ctr, key)) == want


def test_philox_layout_and_index_high_word():
    """element 4 i + j is word j of counter {i lo, i hi, stream, counter} keyed by {seed lo, seed hi}: checked past
    2^32 blocks (the index high word), which no device buffer reaches"""
    seed, stream, ctr = 0x0123456789ABCDEF, 5, 77
    i = (1 << 32) + 3
    w = P.words(8, seed, stream, ctr, start=4 * i)
    blk = P.philox4x32_10((i & 0xffffffff, i >> 32, stream, ctr), (seed & 0xffffffff, seed >> 32))
    blk2 = P.philox4x32_10(((i + 1) & 0xffffffff, (i + 1) >> 32, stream, ctr), (seed & 0xffffffff, seed >> 32))
    assert np.array_equal(w, np.concatenate([blk, blk2]))
    assert not np.array_equal(P.words(4, seed, stream, ctr, start=4 * 3), blk)


def test_value_edges_of_the_noise():
    """u = 1 is reachable: the exponential's floor 1e-20f and the normal's r = 0"""
    c = P.find_counter(1234, 0, 3, lambda w: (w >> 8) == 0xFFFFFF)
    assert c == 413469
    v, _, u = P.exponential(4, 1234, 0, c)
    assert u[3] == 1.0 and v[3] == P.EXP_FLOOR
    c = P.find_counter(1234, 0, 2, lambda w: (w >> 8) == 0xFFFFFF)
    assert c == 2183629
    v, _, u1, _ = P.normal(4, 1234, 0, c)
    assert u1[2] == 1.0 and v[2] == 0.0 and v[3] == 0.0


# ------------------------------------------------------------------------------------------------------------ mutants
def fp32_gru(G, Hin, dH, mutant=None):
    out = emul_gru(G, Hin, dH)
    gr, gc, gu = torch.chunk(G, 3, -1)
    r, u = torch.sigmoid(gr), torch.sigmoid(gu - 1)
    c = torch.tanh(r * gc)
    if mutant == "gate_without_shift":
        us = torch.sigmoid(gu)
        out["h"] = us * c + (1 - us) * Hin
    elif mutant == "dHin_is_dh_u":
        out["dHin"] = dH * u
    elif mutant == "reset_grad_uses_update":
        drc = dH * u * (1 - c * c)
        out["dG"] = torch.cat((drc * gc * u * (1 - u), drc * r, dH * (c - Hin) * u * (1 - u)), -1)
    return out


def _gru_mutant(mutant):
    G, Hin, dH = gru_inputs(256, 24, "n1", seed=21)
    ref, bd = R.gru_gate(G, Hin, dH)
    return worst(fp32_gru(G, Hin, dH), ref, bd), worst(fp32_gru(G, Hin, dH, mutant), ref, bd)


def fp32_cat_bwd(raw, dz, dmix, unimix, G, K, mutant=None):
    M = raw.shape[0]
    dr = torch.empty(M, G * K)
    em.cat_sample_bwd(raw, dz, dmix, unimix, G, K, dr)
    if mutant is None:
        return dr
    x = raw.reshape(M, G, K)
    s = torch.softmax(x, -1)
    pm = (1 - unimix) * s + unimix / K
    pmc = pm.clamp(R.FP32_EPS, 1 - R.FP32_EPS)
    mix = torch.log(pmc) if unimix > 0 else x
    p = torch.softmax(mix, -1)
    d = torch.zeros_like(x) if dz is None else dz.reshape(M, G, K)
    g = (0 if dmix is None else dmix.reshape(M, G, K)) + (p * d if mutant == "uncentred_straight_through"
                                                          else p * (d - (p * d).sum(-1, keepdim=True)))
    if unimix > 0:
        inside = (pm >= R.FP32_EPS) & (pm <= 1 - R.FP32_EPS)
        ds = g * (1 - unimix) / pmc
        if mutant != "grad_outside_the_clamp":
            ds = torch.where(inside, ds, torch.zeros_like(ds))
        g = s * (ds - (s * ds).sum(-1, keepdim=True))
    return g.reshape(M, -1)


def _cat_bwd_mutant(mutant):
    """the missing - sum p dz is a constant shift per group, which the softmax Jacobian of the unimix chain removes:
    that defect shows without unimix only"""
    if mutant == "grad_outside_the_clamp":
        unimix, K, fam = *CLAMP_EDGE, "dominant"
    else:
        unimix, K, fam = 0.0, 32, "s2"
    raw, _, dz, dmix = cat_inputs(256, 1, K, fam, False, seed=22)
    ref, bd = R.cat_sample_bwd(raw, dz, None if mutant == "uncentred_straight_through" else dmix, unimix, 1, K)
    b = None if mutant == "uncentred_straight_through" else dmix
    u = R.f32(unimix)
    return ({"draw": ratio(fp32_cat_bwd(raw, dz, b, u, 1, K), ref, bd)},
            {"draw": ratio(fp32_cat_bwd(raw, dz, b, u, 1, K, mutant), ref, bd)})


def fp32_sample(raw, noise, unimix, G, K, mutant=None):
    oh, mx = emul_cat(raw, noise, unimix, G, K)
    if mutant is None:
        return oh
    M = raw.shape[0]
    p = torch.softmax(mx.reshape(M, G, K), -1)
    if mutant == "noise_times_p":
        p = p * noise.reshape(M, G, K)
    else:                                                   # ties_to_highest: argmax of the reversed row
        assert mutant == "ties_to_highest"
        p = p / noise.reshape(M, G, K) if noise is not None else p
        p = p.flip(-1)
        return F.one_hot(K - 1 - p.argmax(-1), K).float().reshape(M, -1)
    return F.one_hot(p.argmax(-1), K).float().reshape(M, -1)


def _sample_mutant(mutant):
    """the sample criterion: within the margin of the float64 argmax of p / E, and exact ties to the lowest index"""
    if mutant == "ties_to_highest":
        rows, want = tie_rows(40)
        ok = torch.equal(fp32_sample(rows, None, 0.0, 1, 40).argmax(-1), want)
        bad = torch.equal(fp32_sample(rows, None, 0.0, 1, 40, mutant).argmax(-1), want)
        return {"ties": 0.0 if ok else math.inf}, {"ties": 0.0 if bad else math.inf}
    raw, noise, _, _ = cat_inputs(256, 4, 33, "s2", True, seed=23)
    ref, _ = R.cat_sample(raw, noise, 0.01, 4, 33)
    return ({"sample": R.judge_sample(fp32_sample(raw, noise, 0.01, 4, 33), ref, noise)[1]},
            {"sample": R.judge_sample(fp32_sample(raw, noise, 0.01, 4, 33, mutant), ref, noise)[1]})


def _noise_mutant(mutant):
    n, seed, stream, ctr = 4096, 1234, 1, 3
    v, b, u = P.exponential(n, seed, stream, ctr)
    v2, b2, u1, u2 = P.normal(n, seed, stream, ctr)
    honest = {"exp": np_ratio(fp32_exponential(u), v, b), "normal": np_ratio(fp32_normal(u1, u2), v2, b2)}
    if mutant == "cos_sin_swapped":
        return honest, {"normal": np_ratio(fp32_normal(u1, u2, mutant), v2, b2)}
    _, _, um = P.exponential(n, seed, stream, ctr, mutant=mutant)
    wrong = {"exp": np_ratio(fp32_exponential(um), v, b)}
    if mutant != "u_half_open":
        _, _, m1, m2 = P.normal(n, seed, stream, ctr, mutant=mutant)
        wrong["normal"] = np_ratio(fp32_normal(m1, m2), v2, b2)
    return honest, wrong


MUTANTS = {
    "gate_without_shift": _gru_mutant,              # update = sigmoid(update) without the -1
    "dHin_is_dh_u": _gru_mutant,                    # dHin = dh u instead of dh (1 - u)
    "reset_grad_uses_update": _gru_mutant,          # r (1 - r) taken as u (1 - u) in the reset gradient
    "uncentred_straight_through": _cat_bwd_mutant,  # p dz without the - sum p dz
    "grad_outside_the_clamp": _cat_bwd_mutant,      # the unimix chain rule ignoring the clamp
    "ties_to_highest": _sample_mutant,              # exact ties broken to the highest index
    "noise_times_p": _sample_mutant,                # argmax p E instead of p / E
    "key_bumped_first": _noise_mutant,              # Philox key bumped before each round
    "stream_counter_swapped": _noise_mutant,        # stream id and device counter in each other's word
    "u_half_open": _noise_mutant,                   # exponential u on [0, 1)
    "cos_sin_swapped": _noise_mutant,               # Box-Muller with cos and sin swapped
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_bounds_reject_subtly_wrong_implementations(mutant):
    honest, wrong = MUTANTS[mutant](mutant)
    assert max(honest.values()) <= 0.5, honest
    assert max(wrong.values()) >= 4.0, wrong


# ------------------------------------------------------------------------------------------------------------ distribution
N_DIST = 1 << 20


def test_spec_noise_matches_its_distributions():
    """KS of 2^20 exponentials and normals against scipy.stats (the grid truncation's tail mass is far below what a
    KS test of this size resolves)"""
    e = P.exponential(N_DIST, 2024, 0, 5)[0]
    z = P.normal(N_DIST, 2024, 0, 5)[0]
    assert stats.kstest(e, "expon").pvalue > 1e-6
    assert stats.kstest(z, "norm").pvalue > 1e-6
    assert abs(z.mean()) < 5 / math.sqrt(N_DIST) and abs(z.var() - 1) < 5 * math.sqrt(2 / N_DIST)


def test_spec_streams_and_counters_are_uncorrelated():
    """|corr| <= 5 / sqrt(n) between streams 0 and 1 and between counters 0 and 1, and between the words of one block"""
    lim = 5 / math.sqrt(N_DIST)
    a = P.exponential(N_DIST, 99, 0, 0)[2]
    for b in (P.exponential(N_DIST, 99, 1, 0)[2], P.exponential(N_DIST, 99, 0, 1)[2]):
        assert abs(np.corrcoef(a, b)[0, 1]) <= lim
    w = a.reshape(-1, 4)
    for j in range(1, 4):
        assert abs(np.corrcoef(w[:, 0], w[:, j])[0, 1]) <= 5 / math.sqrt(w.shape[0])


def chi_square_pvalue(counts, p):
    counts, p = np.asarray(counts, dtype=np.float64), np.asarray(p, dtype=np.float64)
    return float(stats.chisquare(counts, counts.sum() * p / p.sum()).pvalue)


def test_spec_race_samples_the_unimix_categorical():
    """argmax p / E over 2^20 spec draws of one K = 32 unimix row: class frequencies against p64"""
    K, n = 32, N_DIST
    raw = logit_rows(1, K, "s2", gen(31))
    ref, _ = R.cat_sample(raw, None, 0.01, 1, K)
    p = ref["p"].reshape(K)
    counts = np.zeros(K)
    for c0 in range(0, n, n // 4):
        E = P.exponential(n // 4 * K, 555, 0, 0, start=c0 * K)[0].reshape(-1, K)
        counts += np.bincount(np.argmax(p.numpy() / E, -1), minlength=K)
    assert chi_square_pvalue(counts, p.numpy()) > 1e-6
