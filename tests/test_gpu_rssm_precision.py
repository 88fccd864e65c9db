"""The RSSM sampling, gate and masking kernels of csrc/rssm.cu and the noise fills of csrc/optim.cu against the float64
reference of oracle/rssm_ref.py and the executable noise specification of oracle/philox_ref.py.

Each case runs the kernels twice and checks:
  - error <= bound element by element; a categorical sample is an exact one-hot whose class is within the sample
    margin of the float64 argmax of p / E (rssm_ref.judge_sample); the masks' forward and dPrev are exact;
  - the two runs bit-identical: none of these kernels uses atomics;
  - nothing outside the output views written (guard rows, and the padding between the width and the row stride).
The noise: every element within its bound of the spec's transform of the spec's uniform, and where the documented
1-ulp error of logf cannot reach halfway to a neighbouring grid point, the exponential's uniform is recovered from
the output and must be the spec's.  End to end, fill_exponential -> cat_sample / head_sample over 2^22 draws of one
logits row must sample the unimix categorical (chi-square p > 1e-6, deterministic for the fixed seeds).
Cases, input families and the emulator's margins are in tests/test_rssm_ref_cpu.py, which also shows the bounds reject
a gate without its -1 shift, dHin = dh u, a reset gradient through u (1 - u), an uncentred straight-through gradient, a
gradient through the clamp, ties to the highest index, noise as p E, a Philox key bumped early, swapped stream and
counter words, an exponential uniform on [0, 1) and a Box-Muller with cos and sin swapped.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import philox_ref as P
from oracle import rssm_ref as R
from tests.test_gpu_ln_precision import Guarded
from tests.test_gpu_loss_precision import chunked, guarded, same_bits, twice
from tests.test_loss_ref_cpu import gen, logit_rows, ratio, worst
from tests.test_rssm_ref_cpu import (CAT_CASES, CLAMP_EDGE, FILL_CASES, GRU_CASES, HEAD_CASES, MASK_CASES, OL_CASES,
                                     BWD_MODES, bwd_args, cat_inputs, chi_square_pvalue, gru_inputs, head_inputs,
                                     mask_inputs, ol_inputs, tie_rows)

pytestmark = pytest.mark.gpu

MARGINS = {}                     # case id -> worst error / bound per output, kept for reporting
NON_ARGMAX = {}                  # case id -> picks that differ from the float64 argmax (inside the margin)
CHI2 = {}                        # end-to-end case id -> chi-square p-value of the class frequencies


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    yield CudaOps("cuda")
    path = os.environ.get("RSSM_PRECISION_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump({"margins": MARGINS, "non_argmax_picks": NON_ARGMAX, "chi2_pvalues": CHI2}, f, indent=1,
                      sort_keys=True)


def record(case, m, nonarg=None):
    MARGINS[case] = m
    if nonarg is not None:
        NON_ARGMAX[case] = nonarg
    assert max(m.values()) <= 1.0, m


def device_noise(cu, M, C, ld, seed, stream):
    """fill_exponential noise [M, C] inside rows of ld"""
    buf = torch.empty(M * ld, device="cuda")
    cu.fill_exponential(buf, seed, stream)
    return buf.view(M, ld)[:, :C]


def merge(m, new):
    for k, v in new.items():
        m[k] = max(m.get(k, 0.0), v)


# ------------------------------------------------------------------------------------------------------------ cat_sample
@pytest.mark.parametrize("case", list(CAT_CASES))
def test_cat_sample_precision(cu, case):
    """cat_sample (lane-per-class for K <= 32, strided above) and cat_sample_bwd; layouts: plain, strided (raw, noise,
    dz, dmix and every output inside wider rows, as the engine slices them), mix_only (onehot None: the prior's call),
    sample_only (mix_out None)"""
    M, G, K, fam, unimix, mode, layout, noisy = CAT_CASES[case]
    C = G * K
    raw, _, dz, dmix = cat_inputs(M, G, K, fam, False, seed=len(case), device="cuda")
    st = layout == "strided"
    noise = device_noise(cu, M, C, C + 5 if st else C, seed=len(case), stream=0) if noisy else None
    rg = Guarded(M, C, C + 3 if st else C, fill=raw)
    dzg, dmg = Guarded(M, C, C + 1 if st else C, fill=dz), Guarded(M, C, C + 6 if st else C, fill=dmix)
    a, b = bwd_args(mode, dzg.view, dmg.view)
    want_hot, want_mix = layout != "mix_only", layout != "sample_only"

    def run():
        oh = guarded(M, C, C + 2 if st else C) if want_hot else None
        mx = guarded(M, C, C + 7 if st else C) if want_mix else None
        cu.cat_sample(rg.view, noise, unimix, G, K, oh.view if oh else None, mx.view if mx else None)
        dr = guarded(M, C, C + 4 if st else C)
        cu.cat_sample_bwd(rg.view, a, b, unimix, G, K, dr.view)
        for t in (oh, mx, dr, rg, dzg, dmg):
            assert t is None or t.outside_untouched(), "write outside the output view"
        assert torch.equal(rg.view, raw), "raw was written"
        out = {"draw": dr.view.clone()}
        if oh:
            out["onehot"] = oh.view.clone()
        if mx:
            out["mix"] = mx.view.clone()
        return out

    out = twice(run)
    m, nonarg = {}, 0
    for lo, hi in chunked(M, 8 * C):
        nz = None if noise is None else noise[lo:hi]
        ref, bd = R.cat_sample(raw[lo:hi], nz, unimix, G, K)
        if want_mix:
            merge(m, {"mix": ratio(out["mix"][lo:hi], ref["mix"], bd["mix"])})
        if want_hot:
            fmt, w, n = R.judge_sample(out["onehot"][lo:hi], ref, nz)
            assert fmt, "the sample is not an exact one-hot"
            merge(m, {"sample": w})
            nonarg += n
        d, bd = R.cat_sample_bwd(raw[lo:hi], *bwd_args(mode, dz[lo:hi], dmix[lo:hi]), unimix, G, K)
        merge(m, {"draw": ratio(out["draw"][lo:hi], d, bd)})
    record(f"cat_{case}", m, nonarg if want_hot else None)


@pytest.mark.parametrize("K", [1, 32, 33, 40, 64, 1000])
def test_cat_sample_exact_ties_pick_the_lowest_index(cu, K):
    """bit-equal p / E: classes c and c + 32 (one lane of the strided kernel), 3 and 17 (two lanes), the whole row
    (-> class 0); with no noise and with a noise row that is equal on the tied classes"""
    rows, want = tie_rows(K, "cuda")
    n = rows.shape[0]
    for noise in (None, torch.full((n, K), 0.75, device="cuda")):
        oh = torch.empty(n, K, device="cuda")
        cu.cat_sample(rows, noise, 0.0, 1, K, oh)
        assert torch.equal(oh.sum(-1), torch.ones(n, device="cuda")) and torch.equal(oh.argmax(-1), want), oh.argmax(-1)


@pytest.mark.parametrize("mode", BWD_MODES)
def test_cat_sample_bwd_at_the_clamp_edge(cu, mode):
    """unimix 1e-9, K = 64: pm falls below FP32_EPS in the dominant family, so the clamp is live and elements near
    its edge may take either branch (rssm_ref bounds them for both)"""
    unimix, K = CLAMP_EDGE
    M = 4096
    raw, _, dz, dmix = cat_inputs(M, 1, K, "dominant", False, seed=3, device="cuda")
    a, b = bwd_args(mode, dz, dmix)

    def run():
        dr = guarded(M, K)
        cu.cat_sample_bwd(raw, a, b, unimix, 1, K, dr.view)
        assert dr.outside_untouched()
        return {"draw": dr.view.clone()}

    d, bd = R.cat_sample_bwd(raw, a, b, unimix, 1, K)
    record(f"cat_bwd_clamp_edge_{mode}", {"draw": ratio(twice(run)["draw"], d, bd)})


# ------------------------------------------------------------------------------------------------------------ head_sample
@pytest.mark.parametrize("case", list(HEAD_CASES))
def test_head_sample_precision(cu, case):
    """raw = X W^T + b within its bound; the sample judged on the kernel's own raw, and bit-equal to cat_sample's on
    that raw with the same noise; every operand in rows wider than its width (ldx, ldw, ldr, ldn, ldo)"""
    Kin, A, M, bias, noisy, unimix = HEAD_CASES[case]
    X, W, b, _ = head_inputs(M, Kin, A, bias, False, seed=len(case), device="cuda")
    noise = device_noise(cu, M, A, A + 3, seed=len(case), stream=2) if noisy else None
    xg, wg = Guarded(M, Kin, Kin + 4, fill=X), Guarded(A, Kin, Kin + 8, fill=W)
    assert cu.head_sample_supported(xg.view, wg.view)

    def run():
        raw, oh = guarded(M, A, A + 1), guarded(M, A, A + 2)
        cu.head_sample(xg.view, wg.view, b, noise, unimix, raw.view, oh.view)
        for t in (raw, oh, xg, wg):
            assert t.outside_untouched(), "write outside the output view"
        return {"raw": raw.view.clone(), "onehot": oh.view.clone()}

    out = twice(run)
    r64, br = R.head_raw(X, W, b)
    m = {"raw": ratio(out["raw"], r64, br)}
    ref, _ = R.cat_sample(out["raw"], noise, unimix, 1, A)
    fmt, m["sample"], nonarg = R.judge_sample(out["onehot"], ref, noise)
    assert fmt, "the sample is not an exact one-hot"
    again = torch.empty(M, A, device="cuda")
    cu.cat_sample(out["raw"], noise, unimix, 1, A, again)
    assert same_bits(again, out["onehot"]), "head_sample and cat_sample disagree on the same raw and noise"
    record(f"head_{case}", m, nonarg)


# ------------------------------------------------------------------------------------------------------------ GRU gate
@pytest.mark.parametrize("case", list(GRU_CASES))
def test_gru_gate_precision(cu, case):
    M, Rr, fam = GRU_CASES[case]
    G, Hin, dH = gru_inputs(M, Rr, fam, seed=len(case), device="cuda")
    gg, hg, dg_in = Guarded(M, 3 * Rr, 3 * Rr + 1, fill=G), Guarded(M, Rr, Rr + 2, fill=Hin), \
        Guarded(M, Rr, Rr + 5, fill=dH)

    def run():
        h, dG, dHin = guarded(M, Rr, Rr + 3), guarded(M, 3 * Rr, 3 * Rr + 2), guarded(M, Rr, Rr + 1)
        cu.gru_gate_fwd(gg.view, hg.view, h.view)
        cu.gru_gate_bwd(gg.view, hg.view, dg_in.view, dG.view, dHin.view)
        for t in (h, dG, dHin, gg, hg, dg_in):
            assert t.outside_untouched(), "write outside the output view"
        return {"h": h.view.clone(), "dG": dG.view.clone(), "dHin": dHin.view.clone()}

    out = twice(run)
    ref, bd = R.gru_gate(G, Hin, dH)
    record(f"gru_{case}", worst(out, ref, bd))


# ------------------------------------------------------------------------------------------------------------ masks
@pytest.mark.parametrize("case", list(MASK_CASES))
def test_masks_exact_and_within_bounds(cu, case):
    """mask_mix and mask_rows exact; mask_bwd's dPrev exact, dInit += sum f dIn from a zero start, a nonzero start
    and with dInit None"""
    M, C, first = MASK_CASES[case]
    prev, init, f, dIn, d0 = mask_inputs(M, C, first, seed=len(case), device="cuda")
    pg, dg = Guarded(M, C, C + 3, fill=prev), Guarded(M, C, C + 1, fill=dIn)
    m = {}
    for start in ("none", "zero", "nonzero"):
        s0 = None if start == "none" else torch.zeros(C, device="cuda") if start == "zero" else d0

        def run():
            mix, rows, dp = guarded(M, C, C + 2), guarded(M, C, C + 4), guarded(M, C, C + 5)
            cu.mask_mix(pg.view, init, f, mix.view)
            cu.mask_rows(pg.view, f, rows.view)
            di = None if s0 is None else Guarded(1, C, C, fill=s0.reshape(1, C))
            cu.mask_bwd(dg.view, f, dp.view, None if di is None else di.view[0])
            for t in (mix, rows, dp, di, pg, dg):
                assert t is None or t.outside_untouched(), "write outside the output view"
            out = {"mix": mix.view.clone(), "rows": rows.view.clone(), "dPrev": dp.view.clone()}
            if di is not None:
                out["dInit"] = di.view[0].clone()
            return out

        out = twice(run)
        assert torch.equal(out["mix"].double(), R.mask_mix(prev, init, f))
        assert torch.equal(out["rows"].double(), R.mask_mix(prev, None, f))
        rp, ri, bi = R.mask_bwd(dIn, f, s0)
        assert torch.equal(out["dPrev"].double(), rp)
        if s0 is not None:
            merge(m, {f"dInit_{start}": ratio(out["dInit"], ri, bi)})
    record(f"mask_{case}", m or {"exact": 0.0})


# ------------------------------------------------------------------------------------------------------------ onehot_linear
@pytest.mark.parametrize("case", list(OL_CASES))
def test_onehot_linear_precision(cu, case):
    """the gather form with z an exact one-hot inside a wider row (the hot class of every third group in the second
    ballot chunk when K > 32) and act None (A = 0)"""
    S, K, A, N = OL_CASES[case]
    M = 257
    z, act, WT = ol_inputs(M, S, K, A, N, seed=len(case), device="cuda")
    zg = Guarded(M, S * K, S * K + 3, fill=z)
    ag = Guarded(M, A, A + 2, fill=act) if A else None
    a_view = ag.view if A else torch.empty(M, 0, device="cuda")

    def run():
        out = guarded(M, N, N + 1)
        cu.onehot_linear(zg.view, a_view, WT, out.view, S, K)
        for t in (out, zg, ag):
            assert t is None or t.outside_untouched(), "write outside the output view"
        return {"out": out.view.clone()}

    ref, bd = R.onehot_linear(z, act, WT, S, K)
    record(f"onehot_linear_{case}", {"out": ratio(twice(run)["out"], ref, bd)})


# ------------------------------------------------------------------------------------------------------------ noise
def _exp_pinned(u):
    """half the gap to the nearer neighbouring grid point in -ln u, and whether it exceeds 1 ulp of the fp32 result
    (the documented logf error): there the output identifies u"""
    k = np.round(u / P.U)
    t = -np.log(u)
    lo = -np.log(np.maximum(k - 1, 0.5) * P.U)             # k - 1 = 0 does not exist: a wide gap
    hi = np.where(k < 2 ** 24, -np.log(np.minimum(k + 1, 2 ** 24) * P.U), t - 1.0)
    half = np.minimum(lo - t, t - hi) / 2
    ulp = np.spacing(np.maximum(t, P.EXP_FLOOR).astype(np.float32)).astype(np.float64)
    return half, half > ulp


@pytest.mark.parametrize("case", list(FILL_CASES))
def test_fill_noise_matches_the_spec(cu, case):
    """fill_exponential / fill_normal over the grid-stride loop's edges: every element within its bound of the spec,
    the exponential's uniform recovered exactly wherever the output pins it, nothing past n written"""
    n, ctr, seed, stream = FILL_CASES[case]
    counter = None if ctr is None else torch.tensor([ctr], dtype=torch.int32, device="cuda")
    m = {}
    for kind in ("exponential", "normal"):
        def run():
            buf = guarded(1, n)
            getattr(cu, f"fill_{kind}")(buf.view[0], seed, stream, counter)
            assert buf.outside_untouched(), "write past n"
            return {"x": buf.view[0].clone()}

        got = twice(run)["x"].double().cpu().numpy()
        if kind == "exponential":
            v, b, u = P.exponential(n, seed, stream, ctr or 0)
            half, pinned = _exp_pinned(u)
            assert np.all(np.abs(got - v)[pinned] < half[pinned]), "an exponential's uniform is not the spec's"
            assert pinned.mean() > 0.5 or n < 64
        else:
            v, b, _, _ = P.normal(n, seed, stream, ctr or 0)
        d = np.abs(got - v)
        m[kind] = float(np.max(np.where(d == 0, 0.0, d / b)))
    record(f"fill_{case}", m)


def test_noise_value_edges(cu):
    """u = 1, located with the spec: the exponential's floor 1e-20f, and the normal's r = 0 on both of its pair"""
    c = P.find_counter(1234, 0, 3, lambda w: (w >> 8) == 0xFFFFFF)
    out = torch.empty(4, device="cuda")
    cu.fill_exponential(out, 1234, 0, torch.tensor([c], dtype=torch.int32, device="cuda"))
    assert float(out[3]) == P.EXP_FLOOR, out.tolist()
    c = P.find_counter(1234, 0, 2, lambda w: (w >> 8) == 0xFFFFFF)
    cu.fill_normal(out, 1234, 0, torch.tensor([c], dtype=torch.int32, device="cuda"))
    assert float(out[2]) == 0.0 and float(out[3]) == 0.0, out.tolist()


# ------------------------------------------------------------------------------------------------------------ end to end
E2E_ROWS = 1 << 22


@pytest.mark.parametrize("path,K", [("cat_sample", 32), ("cat_sample", 40), ("head_sample", 32)])
def test_device_race_samples_the_unimix_categorical(cu, path, K):
    """fill_exponential -> cat_sample / head_sample over 2^22 rows of one logits row, unimix 0.01: class frequencies
    against the float64 probabilities (chi-square p > 1e-6)"""
    unimix, n = 0.01, E2E_ROWS
    noise = torch.empty(n, K, device="cuda")
    cu.fill_exponential(noise.view(-1), 4321, 3 if path == "head_sample" else K)
    oh = torch.empty(n, K, device="cuda")
    if path == "cat_sample":
        row = logit_rows(1, K, "s2", gen(K, "cuda"), "cuda")
        cu.cat_sample(row.expand(n, K).contiguous(), noise, unimix, 1, K, oh)
    else:
        g = gen(5, "cuda")
        X = torch.randn(1, 64, generator=g, device="cuda").expand(n, 64).contiguous()
        W = torch.randn(K, 64, generator=g, device="cuda") / 4
        raw = torch.empty(n, K, device="cuda")
        cu.head_sample(X, W, None, noise, unimix, raw, oh)
        row = raw[:1].clone()
        assert torch.equal(raw, row.expand(n, K)), "rows of equal inputs gave different logits"
        del raw, X
    ref, _ = R.cat_sample(row, None, unimix, 1, K)
    assert torch.equal(oh.sum(-1), torch.ones(n, device="cuda"))
    counts = oh.sum(0).double().cpu().numpy()
    pv = chi_square_pvalue(counts, ref["p"].reshape(K).cpu().numpy())
    CHI2[f"race_{path}_K{K}"] = pv
    assert pv > 1e-6, pv
