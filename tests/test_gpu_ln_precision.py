"""Every stand-alone LayerNorm route of csrc/norm.cu, the column sums, and the gather + LayerNorm + SiLU of
`onehot_linear_ln` (csrc/rssm.cu) against the float64 reference of oracle/ln_ref.py.

Each LayerNorm case runs forward and backward twice and checks:
  - the intended route, through b200rl_ln_act_route (0 warp per row, 1 register-resident rows, 2 one CTA per row);
  - error <= bound element by element for y and dX, column by column for dgamma / dbeta (not relative to the largest
    entry of the output, so one small wrong row or column fails);
  - y and dX bit-identical between the runs; dgamma / dbeta are summed with atomics (not bit-reproducible) and each
    run is held to the bound;
  - nothing outside the output views is written (guard values around and between the rows).
Cases, input families and their shapes are defined in tests/test_ln_ref_cpu.py, which holds the emulator to the same
bounds and shows that they reject one-pass variance, a missing eps, a wrong mean, a lost row group, a misplaced SiLU'
and a 1e-4 error in rstd.
"""
import json
import math
import os

import pytest
import torch

from oracle import ln_ref
from oracle.simt_ref import tau1
from tests.test_ln_ref_cpu import FLAKE_SHAPE, LN_CASES, flake_inputs, ln_inputs, margins, ratio

pytestmark = pytest.mark.gpu

GUARD = -7.0
MARGINS = {}          # case id -> worst error / bound per output, kept for reporting


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    yield CudaOps("cuda")
    path = os.environ.get("LN_PRECISION_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(MARGINS, f, indent=1, sort_keys=True)


class Guarded:
    """an [M, C] view with row stride ld, `off` floats into a buffer of GUARD values (pad rows before and after)"""

    def __init__(self, M, C, ld, off=0, pad=64, fill=None):
        self.buf = torch.full((pad + M * ld + pad,), GUARD, device="cuda")
        self.view = self.buf[pad + off:pad + off + M * ld].view(M, ld)[:, :C]
        self.mask = torch.zeros_like(self.buf, dtype=torch.bool)
        self.mask[pad + off:pad + off + M * ld].view(M, ld)[:, :C] = True
        if fill is not None:
            self.view.copy_(fill)

    def outside_untouched(self):
        return bool((self.buf[~self.mask] == GUARD).all())


def run_ln(cu, X, gamma, beta, eps, act, dY, layout, prior_g, prior_b):
    """one forward + backward in `layout`; returns (Y, dX, dgamma, dbeta) as fresh tensors, guards checked"""
    M, C = X.shape
    ld = {"strided": C + 4, "ld_odd": C + 1}.get(layout, C)
    off = 1 if layout == "offset" else 0
    x = Guarded(M, C, ld, off, fill=X)
    y = Guarded(M, C, ld, off)
    cu.ln_act_fwd(x.view, gamma, beta, eps, act, y.view)
    dy = Guarded(M, C, ld, off, fill=dY)
    dx = dy if layout == "alias" else Guarded(M, C, ld, off)
    dg = db = None
    if layout != "noparam":
        dg, db = Guarded(1, C, C, fill=prior_g), Guarded(1, C, C, fill=prior_b)
    cu.ln_act_bwd(x.view, gamma, beta, eps, act, dy.view, dx.view, None if dg is None else dg.view[0],
                  None if db is None else db.view[0], accumulate=layout == "accumulate")
    for g in (x, y, dy, dx) + ((dg, db) if dg is not None else ()):
        assert g.outside_untouched(), "write outside the output view"
    assert torch.equal(x.view, X), "the input was written"
    return (y.view.clone(), dx.view.clone(), None if dg is None else dg.view[0].clone(),
            None if db is None else db.view[0].clone())


def route_of(cu, X, layout):
    M, C = X.shape
    ld = {"strided": C + 4, "ld_odd": C + 1}.get(layout, C)
    off = 1 if layout == "offset" else 0
    base = torch.empty(64, device="cuda").data_ptr()         # 256-byte aligned
    p = base + 4 * off
    return cu.lib.b200rl_ln_act_route(C, ld, ld, ld, p, p, p, base, base)


@pytest.mark.parametrize("case", list(LN_CASES))
def test_ln_act_precision(cu, case):
    route, C, M, act, eps, fam, layout = LN_CASES[case]
    assert route_of(cu, torch.empty(M, C), layout) == route
    X, gamma, beta, dY = ln_inputs(M, C, fam, eps, act, seed=len(case), device="cuda")
    acc = layout == "accumulate"
    gen = torch.Generator(device="cuda").manual_seed(1)
    prior_g = math.sqrt(M) * torch.randn(C, generator=gen, device="cuda") if acc else torch.full((C,), float("nan"),
                                                                                              device="cuda")
    prior_b = math.sqrt(M) * torch.randn(C, generator=gen, device="cuda") if acc else prior_g.clone()
    first = run_ln(cu, X, gamma, beta, eps, act, dY, layout, prior_g, prior_b)
    again = run_ln(cu, X, gamma, beta, eps, act, dY, layout, prior_g, prior_b)
    assert torch.equal(first[0], again[0]) and torch.equal(first[1], again[1]), "rerun is not bit-identical"
    worst = {}
    for run in (first, again):
        m = margins(X, gamma, beta, eps, act, dY, *run, prior_g=prior_g if acc else None,
                    prior_b=prior_b if acc else None)
        worst = {k: max(v, worst.get(k, 0.0)) for k, v in m.items()}
    MARGINS[case] = worst
    assert max(worst.values()) <= 1.0, worst


def test_ln_act_precision_at_the_once_failed_shape(cu):
    """tanh, M = 1000, C = 32, eps 1e-5 with the inputs of test_ln_act_tanh_relu[2-1000-32]"""
    M, C, act, eps = FLAKE_SHAPE
    X, gamma, beta, dY = (t.cuda() for t in flake_inputs())
    first = run_ln(cu, X, gamma, beta, eps, act, dY, "plain", torch.full((C,), float("nan"), device="cuda"),
                   torch.full((C,), float("nan"), device="cuda"))
    MARGINS["flake_tanh_M1000_C32"] = m = margins(X, gamma, beta, eps, act, dY, *first)
    assert max(m.values()) <= 1.0, m


def test_every_route_is_exercised(cu):
    assert {v[0] for v in LN_CASES.values()} == {0, 1, 2}


def test_generic_backward_refuses_before_writing(cu):
    """C = 30000 is past the generic backward's shared accumulators: the call is refused, and dgamma, dbeta and dX keep
    what they held"""
    from sheeprl_b200.lib import B200RLError

    M, C = 4, 30000
    X, dY = torch.randn(M, C, device="cuda"), torch.randn(M, C, device="cuda")
    gamma, beta = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    dX, dg, db = (torch.full(s, float("nan"), device="cuda") for s in ((M, C), (C,), (C,)))
    assert route_of(cu, X, "plain") == 0
    with pytest.raises(B200RLError, match="bad argument"):
        cu.ln_act_bwd(X, gamma, beta, 1e-3, 0, dY, dX, dg, db)
    torch.cuda.synchronize()
    assert bool(dX.isnan().all()) and bool(dg.isnan().all()) and bool(db.isnan().all())


# ------------------------------------------------------------------------------------------------------------ col_sum
# M, C, ld (None: C), accumulate.  The flat float4 kernel takes contiguous, 16-byte aligned X with C <= 32 and
# M * C >= 65536; the tail of a total that is not a multiple of 4 is added by one thread.
COL_SUM_CASES = {
    "narrow_C1": (65537, 1, None, False), "narrow_C3": (21847, 3, None, True), "narrow_C7": (9363, 7, None, False),
    "narrow_C32": (2049, 32, None, True),
    "general_C5_strided": (1000, 5, 8, False), "general_C100_strided": (70001, 100, 103, True),
    "general_C1536_strided": (3000, 1536, 1537, False), "general_C33_M1": (1, 33, 40, True),
    "general_C32_small": (2047, 32, None, False),
}


@pytest.mark.parametrize("family", ["centred", "offset"])
@pytest.mark.parametrize("case", list(COL_SUM_CASES))
def test_col_sum_precision(cu, case, family):
    M, C, ld, acc = COL_SUM_CASES[case]
    narrow = C <= 32 and ld is None and M * C >= 1 << 16
    assert narrow == case.startswith("narrow")
    X = ln_inputs(M, C, family, 1e-3, 0, seed=3, device="cuda")[0]
    x = Guarded(M, C, ld or C, fill=X)
    prior = torch.randn(C, device="cuda") * math.sqrt(M) if acc else None
    outs = []
    for _ in range(2):
        out = Guarded(1, C, C, fill=prior if acc else torch.full((C,), float("nan"), device="cuda"))
        cu.col_sum(x.view, out.view[0], accumulate=acc)
        assert out.outside_untouched(), "write outside the output view"
        outs.append(out.view[0].clone())
    s, mag = ln_ref.col_sum64(X)
    if acc:
        s = s + prior.double()
    worst = max(ratio(o, s, ln_ref.param_bound(M, mag, prior=prior)) for o in outs)
    MARGINS[f"col_sum_{case}_{family}"] = {"col_sum": worst}
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------------------ onehot_linear_ln
@pytest.mark.parametrize("SK", [(32, 32), (64, 3), (1, 40)], ids=lambda s: f"S{s[0]}xK{s[1]}")
@pytest.mark.parametrize("N", [128, 256, 512, 1024])
def test_onehot_linear_ln_precision(cu, N, SK):
    """`pre` against the float64 gather-sum with tau1(S + A); the output against the float64 SiLU(LayerNorm) of the
    kernel's own `pre` with the forward bound (the LayerNorm isolated from its input); the same output without `pre`"""
    S, K = SK
    M, eps = 256, 1e-3
    worst = {"pre": 0.0, "out": 0.0}
    for A in (0, 1, 18, 32):
        g = torch.Generator(device="cuda").manual_seed(N + A)
        z = torch.nn.functional.one_hot(torch.randint(0, K, (M, S), generator=g, device="cuda"), K).float()
        z = z.reshape(M, S * K)
        act = torch.randn(M, A, generator=g, device="cuda")                        # A = 0: NULL, never read
        WT = 0.1 * torch.randn(S * K + A, N, generator=g, device="cuda")
        gamma = 1 + 0.3 * torch.randn(N, generator=g, device="cuda")
        beta = 0.2 * torch.randn(N, generator=g, device="cuda")
        assert cu.onehot_linear_supported(S, K, A, N)
        outs = []
        for keep in (True, False, True):
            out = Guarded(M, N, N + 8, fill=torch.full((M, N), float("nan"), device="cuda"))
            pre = Guarded(M, N, N, fill=torch.full((M, N), float("nan"), device="cuda")) if keep else None
            assert cu.onehot_linear_ln_supported(WT, out.view, None if pre is None else pre.view)
            cu.onehot_linear_ln(z, act, WT, gamma, beta, eps, out.view, S, K, pre=None if pre is None else pre.view)
            assert out.outside_untouched() and (pre is None or pre.outside_untouched())
            outs.append((out.view.clone(), None if pre is None else pre.view.clone()))
        assert all(torch.equal(o, outs[0][0]) for o, _ in outs) and torch.equal(outs[0][1], outs[2][1])
        y, p = outs[0]
        pre64, mag = ln_ref.gather64(z, act, WT, S, K)
        worst["pre"] = max(worst["pre"], ratio(p, pre64, tau1(S + A) * mag))
        y64 = ln_ref.ln_act_fwd64(p, gamma, beta, eps, 1)[0]
        worst["out"] = max(worst["out"], ratio(y, y64, ln_ref.ln_act_fwd_bound(p, gamma, beta, eps, 1, y64)))
    MARGINS[f"onehot_linear_ln_N{N}_S{S}xK{K}"] = worst
    assert max(worst.values()) <= 1.0, worst
