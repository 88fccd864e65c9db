"""Every tensor-core product route of csrc/gemm_tc.cu and csrc/conv.cu against a float64 reference (oracle/tc_ref.py),
in both matmul precisions.

Each case runs under "highest" (3xTF32), then "high" (one TF32 pass), then "highest" again, and checks:
  - the intended route is taken (the `_supported` / workspace entry points that pick it);
  - "highest" error <= tau3(K) = 2^-24 (TAU_CONST + TAU_SQRT sqrt(K)), K = the kernel's reduction length;
  - "high" error inside the TF32 band, and at least MIN_RATIO times the "highest" error on positive operands: the
    single-pass instantiation is a built-in kernel with lost TF32 passes, so the ratio shows that this case would catch
    a lost pass (a dropped cross term costs ~2^-11 relative, within 4x of a single pass) on its own route;
  - the second "highest" run reproduces the first bit for bit: split-K partials and persistent tiles are reduced in a
    fixed order, and leaving "high" restores the three-pass kernels;
  - nothing outside the output view is written (guard rows / columns / elements).

Two operand families:
  positive  U(0.5, 1) with full mantissas: truncating TF32 passes bias every product the same way, so errors cannot
            cancel.  Metric: max |C - C64| / C64.
  mixed     N(0, 1).  Metric: max |C - C64| / (sum_k |a||b| + |bias| + |C0|), per element, independent of the largest
            entry of the output.
"""
import ctypes
import math

import pytest
import torch

from oracle import tc_ref
from oracle.ln_ref import ln_bound

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
# 3xTF32, in units of u = 2^-24 relative to sum |a||b|: each product keeps hi*hi + hi*lo + lo*hi with both lo parts
# truncated to TF32 and lo*lo dropped (< 3 x 16 u); the tensor core accumulates a chunk of 128 k with truncation (up to
# ~96 u); the chunk sums add with round to nearest, which grows like sqrt(K / 128) u ~ 0.09 sqrt(K) u.  The bound
# takes that constant and 5x the sqrt(K) term.  On an H100 the worst "highest" errors were 3.3e-6 = 56 u (positive
# operands, every K) and 1.2e-6 (mixed signs); a dropped cross term cost 3.3e-4 .. 4.5e-4, 6x over tau3 at the largest
# K tested (2.3e6) and 25x over it at K <= 16384.
TAU_CONST, TAU_SQRT = 144.0, 0.5
# one TF32 pass truncates both operands to 10 mantissa bits: 2^-12 .. 2^-10 relative each on U(0.5, 1)
BAND = (2.0 ** -13, 2.0 ** -9)
MIN_RATIO = 50.0
FAMILIES = ("positive", "mixed")
EPS = 1e-3
GUARD = -7.0
MARGINS = {}          # case id -> measured errors and error / bound, kept for reporting


def tau3(K):
    return U * (TAU_CONST + TAU_SQRT * math.sqrt(K))


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    ops = CudaOps("cuda")
    assert ops.use_tc, "the tensor-core paths are disabled (B200RL_DISABLE_TC=1)"
    assert ops.matmul_precision() == "highest"
    return ops


def draw(shape, family, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if family == "positive":
        return torch.rand(shape, generator=g, device="cuda") * 0.5 + 0.5
    return torch.randn(shape, generator=g, device="cuda")


def padded(rows, cols, family, seed):
    """[rows][cols] view of a buffer whose row stride is rounded up to 16 bytes (the tensor-core operand rule); the
    pad columns hold 1e6, which must never be read"""
    buf = torch.full((rows, (cols + 3) // 4 * 4), 1e6, device="cuda")
    buf[:, :cols] = draw((rows, cols), family, seed)
    return buf[:, :cols]


def guarded(shape, pad=32):
    """contiguous output of `shape` inside a buffer of GUARD values; returns (buffer, view)"""
    n = math.prod(shape)
    buf = torch.full((n + 2 * pad,), GUARD, device="cuda")
    return buf, buf[pad:pad + n].view(shape)


def assert_guards(buf, view_slice):
    rest = buf.clone()
    rest[view_slice] = GUARD
    assert bool((rest == GUARD).all()), "write outside the output view"


def precisions(cu, run):
    """`run()` launches the op on fresh outputs and returns them.  Returns (outputs at "highest", outputs at "high")."""
    first = run()
    try:
        cu.set_matmul_precision("high")
        single = run()
    finally:
        cu.set_matmul_precision("highest")
    again = run()
    for a, b in zip(first, again):
        assert torch.equal(a, b), "rerun at \"highest\" is not bit-identical"
    return first, single


def rel_err(got, ref, mag, family):
    d = (got.double() - ref).abs()
    if family == "positive":
        assert bool((ref > 0).all())
        return float((d / ref).max())
    return float((d / mag).max())


def assess(case, K, errs, extra=None):
    """errs[family] = (error at "highest", error at "high")"""
    tau = tau3(K)
    (p3, p1), (m3, m1) = errs["positive"], errs["mixed"]
    m = {"K": K, "positive": p3, "mixed": m3, "high": p1, "high_mixed": m1, "ratio": p1 / max(p3, 1e-30),
         "highest/tau3": max(p3, m3) / tau}
    m.update(extra or {})
    MARGINS[case] = m
    assert p3 <= tau and m3 <= tau, ("3xTF32 error over tau3", m)
    assert BAND[0] <= p1 <= BAND[1] and m1 <= BAND[1], ("single-pass error outside the TF32 band", m)
    assert p1 >= MIN_RATIO * p3, ("\"high\" / \"highest\" error ratio", m)


# ---------------------------------------------------------------------------------------------------------- GEMM
# M, N, K, transA, transB.  Tiles are 128 x BN (BN = 64 when N <= 64); gemm_tc_impl splits K when tiles < 2 * 132 and
# there are >= 8 k-blocks of 32, and runs a persistent grid when tiles x splits > 2 * 132.  Expected route per case:
GEMM_CASES = {
    "nt_bn64_split": (2048, 64, 1536, False, True),       # BN 64, 16 tiles, 8 splits
    "nt_bn64_direct": (1000, 48, 200, False, True),       # BN 64, 7 k-blocks: no split; ragged M, K
    "nt_bn64_persistent": (65536, 64, 256, False, True),  # BN 64, 512 tiles: persistent, no split
    "nt_direct": (4096, 256, 200, False, True),           # 64 tiles, 7 k-blocks: no split
    "nt_split": (1024, 512, 4096, False, True),           # 32 tiles, 4 splits
    "nt_persistent": (16384, 512, 1536, False, True),     # 512 tiles: persistent, no split
    "nt_m64": (64, 3072, 1280, False, True),              # one half-empty row tile, 24 tiles, 5 splits
    "nt_m40": (40, 512, 512, False, True),                # 4 tiles, 4 splits
    "nt_ragged": (257, 129, 100, False, True),            # ragged M, N, K: 6 tiles, no split
    "nt_ragged_k": (1000, 200, 1026, False, True),        # K = 1026 in rows of 1028: 16 tiles, 7 splits
    "nt_k16384": (256, 256, 16384, False, True),          # 4 tiles, 32 splits
    "nn_persistent": (16384, 1536, 512, False, False),    # MN-major B: 1536 tiles, persistent
    "nn_ragged": (300, 200, 68, False, False),            # 6 tiles, no split
    "nn_twohot": (1024, 512, 255, False, False),          # dX of the 255-bin heads: A rows of 256 floats, no split
    "tn_k16384": (512, 1536, 16384, True, False),         # MN-major A and B, 48 tiles x 8 splits: persistent
    "tn_twohot": (255, 512, 15360, True, False),          # dW of the 255-bin heads: A [15360][256], 16 splits
    "tn_ragged": (257, 129, 100, True, False),            # no split
    "tt_ragged": (129, 52, 36, True, True),               # MN-major A, K-major B, BN 64, no split
    "tt_split": (1024, 768, 2048, True, True),            # 48 tiles, 2 splits
}


def gemm_errors(cu, family, M, N, K, tA, tB, bias=False, acc=False, odd_ldc=False, seed=0):
    A = padded(*((K, M) if tA else (M, K)), family, seed)
    B = padded(*((N, K) if tB else (K, N)), family, seed + 1)
    b = draw((N,), family, seed + 2) if bias else None
    C0 = draw((M, N), family, seed + 3) if acc else None
    assert cu.lib.b200rl_gemm_tc_supported(ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(B.data_ptr()), M, N, K,
                                           A.stride(0), B.stride(0), int(tA), int(tB)) == 1
    # odd_ldc: a column slice of rows with an odd float stride (scalar store branch on every other row)
    ldc = (N + 3 if N % 2 == 0 else N + 2) if odd_ldc else N
    col0 = 1 if odd_ldc else 0
    view = (slice(1, M + 1), slice(col0, col0 + N))

    def run():
        Cbuf = torch.full((M + 2, ldc), GUARD, device="cuda")
        C = Cbuf[view]
        if C0 is not None:
            C.copy_(C0)
        cu.gemm(A, B, C, tA, tB, bias=b, accumulate=acc)
        return (Cbuf,)

    (c3,), (c1,) = precisions(cu, run)
    for c in (c3, c1):
        assert_guards(c, view)
    ref, mag = tc_ref.gemm64(A, B, tA, tB, bias=b, C0=C0)
    return rel_err(c3[view], ref, mag, family), rel_err(c1[view], ref, mag, family)


@pytest.mark.parametrize("case", list(GEMM_CASES))
def test_gemm_tc_precision(cu, case):
    M, N, K, tA, tB = GEMM_CASES[case]
    errs = {f: gemm_errors(cu, f, M, N, K, tA, tB, seed=10 * i) for i, f in enumerate(FAMILIES)}
    assess("gemm_" + case, K, errs)


# epilogue: bias / accumulate through the direct store (4096 x 256 x 200: no split) and through the split-K reduce
# (1024 x 512 x 4096: 4 splits), into contiguous rows and into rows with an odd stride
EPI_ROUTES = {"direct": (4096, 256, 200), "split": (1024, 512, 4096)}


@pytest.mark.parametrize("route", list(EPI_ROUTES))
@pytest.mark.parametrize("epi", ["bias", "acc", "bias_acc"])
@pytest.mark.parametrize("odd_ldc", [False, True], ids=["ldc_n", "ldc_odd"])
def test_gemm_tc_epilogue_precision(cu, route, epi, odd_ldc):
    M, N, K = EPI_ROUTES[route]
    errs = {f: gemm_errors(cu, f, M, N, K, False, True, bias="bias" in epi, acc="acc" in epi, odd_ldc=odd_ldc,
                           seed=10 * i + 100) for i, f in enumerate(FAMILIES)}
    assess(f"epilogue_{route}_{epi}_{'odd' if odd_ldc else 'n'}", K, errs)


# ------------------------------------------------------------------------------------ fused product + LayerNorm
def ln_params(N, seed):
    return 1.0 + 0.1 * draw((N,), "mixed", seed), 0.1 * draw((N,), "mixed", seed + 1)


@pytest.mark.parametrize("N", [96, 200, 512, 1000, 1536], ids=lambda n: f"N{n}")   # NV = 1, 2, 4, 8, 12
@pytest.mark.parametrize("act", [0, 1], ids=["identity", "silu"])
def test_gemm_ln_precision(cu, N, act):
    M, K = 1000, 512
    errs, out_margin = {}, {"highest": 0.0, "high": 0.0}
    for i, family in enumerate(FAMILIES):
        A, W = draw((M, K), family, 10 * i + 1), draw((N, K), family, 10 * i + 2)
        gamma, beta = ln_params(N, 10 * i + 3)
        assert cu.gemm_ln_supported(A, W, 0)

        def run():
            out, pre = torch.empty(M, N, device="cuda"), torch.empty(M, N, device="cuda")
            cu.gemm_ln_act(A, W, gamma, beta, EPS, act, out, pre)
            out2 = torch.empty(M, N, device="cuda")
            cu.gemm_ln_act(A, W, gamma, beta, EPS, act, out2, None)
            assert torch.equal(out, out2), "the optional `pre` save changed the output"
            return out, pre

        (o3, p3), (o1, p1) = precisions(cu, run)
        ref, mag, pre64 = tc_ref.gemm_ln64(A, W, gamma, beta, EPS, act)
        errs[family] = (rel_err(p3, pre64, mag, family), rel_err(p1, pre64, mag, family))
        # SiLU: |silu'| <= 1.1, plus 4 u |out| for expf and the division
        slope = 1.1 if act else 1.0
        for name, o, tau in (("highest", o3, tau3(K)), ("high", o1, BAND[1])):
            bound = slope * ln_bound(pre64, mag, gamma, beta, tau, EPS) + 4 * U * ref.abs()
            out_margin[name] = max(out_margin[name], float(((o.double() - ref).abs() / bound).max()))
    assess(f"gemm_ln_N{N}_act{act}", K, errs, {"out/bound": out_margin["highest"], "out_high/bound": out_margin["high"]})
    assert out_margin["highest"] <= 1.0 and out_margin["high"] <= 1.0, out_margin


@pytest.mark.parametrize("N", [384, 768, 1152, 1536], ids=lambda n: f"N{n}")      # NV = 3, 6, 9, 12
def test_gemm_ln_gru_precision(cu, N):
    M, R = 1000, N // 3
    K = R + 256
    errs, h_margin = {}, {"highest": 0.0, "high": 0.0}
    for i, family in enumerate(FAMILIES):
        A, W = draw((M, K), family, 10 * i + 1), draw((N, K), family, 10 * i + 2)
        gamma, beta = ln_params(N, 10 * i + 3)
        h_prev = 0.5 * draw((M, R), "mixed", 10 * i + 5)
        assert cu.gemm_ln_supported(A, W, 1)

        def run():
            h, pre, ln = (torch.empty(M, n, device="cuda") for n in (R, N, N))
            cu.gemm_ln_gru(A, W, gamma, beta, EPS, h_prev, h, g_pre=pre, g_ln=ln)
            return h, pre, ln

        (h3, p3, _), (h1, p1, _) = precisions(cu, run)
        h64, mag, pre64, ln64 = tc_ref.gemm_ln_gru64(A, W, gamma, beta, EPS, h_prev)
        errs[family] = (rel_err(p3, pre64, mag, family), rel_err(p1, pre64, mag, family))
        # first-order propagation of the LayerNorm bound through the gate, per third, plus 16 u for expf / tanhf
        gr, gc, gu = torch.chunk(ln64, 3, -1)
        r, u = torch.sigmoid(gr), torch.sigmoid(gu - 1.0)
        c = torch.tanh(r * gc)
        dr, dc, du = (u * (1 - c * c) * gc * r * (1 - r)).abs(), u * (1 - c * c) * r, ((c - h_prev.double()) * u * (1 - u)).abs()
        for name, h, tau in (("highest", h3, tau3(K)), ("high", h1, BAND[1])):
            br, bc, bu = torch.chunk(ln_bound(pre64, mag, gamma, beta, tau, EPS), 3, -1)
            bound = dr * br + dc * bc + du * bu + 16 * U * (1 + h_prev.double().abs())
            h_margin[name] = max(h_margin[name], float(((h.double() - h64).abs() / bound).max()))
    assess(f"gemm_ln_gru_N{N}", K, errs, {"h/bound": h_margin["highest"], "h_high/bound": h_margin["high"]})
    assert h_margin["highest"] <= 1.0 and h_margin["high"] <= 1.0, h_margin


# ------------------------------------------------------------------------------- implicit-GEMM convolutions
# kind, NB, h, w, Cs, Cb (Conv2d big Cb -> small Cs; ConvTranspose2d small Cs -> big Cb).  Output tiles are 128 pixels of
# the small grid x BN output channels (BN = 64 when Cout <= 64); a grid of more than 2 * 132 tiles (x 4 parities for
# "up") is persistent.
CONV_CASES = {
    "down_bn64_ragged": ("down", 8, 8, 8, 40, 32),        # Cout 40 of a 64-wide tile, 4 tiles
    "down_bn128_ragged": ("down", 4, 16, 16, 200, 64),    # Cout 200: second n tile 72 wide, 16 tiles
    "down_persistent": ("down", 64, 16, 16, 384, 32),     # 128 x 3 tiles: persistent
    "up_bn64_ragged": ("up", 8, 8, 8, 64, 48),            # Cout 48 of a 64-wide tile, 4 tiles x 4 parities
    "up_bn128_persistent": ("up", 32, 16, 16, 32, 132),   # Cout 132: 64 x 2 tiles x 4 parities, persistent
    "up4": ("up", 4, 16, 16, 64, 32),                     # Cout 32: the merged four-parity UP4 tile, 8 tiles
    "up4_persistent": ("up", 256, 16, 16, 32, 32),        # UP4, 512 tiles: persistent
}


CONV_PARAMS = [pytest.param(c, b, id=f"{c}-{'bias' if b else 'nobias'}") for c, v in CONV_CASES.items()
               for b in ((False, True) if v[0] == "up" else (False,))]      # the Conv2d forward has no bias


@pytest.mark.parametrize("case,bias", CONV_PARAMS)
def test_conv_tc_precision(cu, case, bias):
    kind, NB, h, w, Cs, Cb = CONV_CASES[case]
    up = kind == "up"
    assert cu.lib.b200rl_conv_tc_supported(int(up), NB, h, w, Cs, Cb) == 1
    merged = int(cu.lib.b200rl_conv_pack_floats(int(up), Cs, Cb)) == 36 * Cs * Cb
    assert merged == case.startswith("up4")
    K = 16 * Cb if not up else (9 * Cs if merged else 4 * Cs)      # the kernel's reduction length
    errs = {}
    for i, family in enumerate(FAMILIES):
        big, small = draw((NB, 2 * h, 2 * w, Cb), family, 10 * i + 1), draw((NB, h, w, Cs), family, 10 * i + 2)
        W, b = draw((Cs, Cb, 4, 4), family, 10 * i + 3), (draw((Cb,), family, 10 * i + 4) if bias else None)
        shape = (NB, 2 * h, 2 * w, Cb) if up else (NB, h, w, Cs)

        def run():
            buf, out = guarded(shape)
            if up:
                cu.conv_up(small, W, out, b)
            else:
                cu.conv_down(big, W, out)
            return (buf,)

        (o3,), (o1,) = precisions(cu, run)
        view = slice(32, 32 + math.prod(shape))
        for o in (o3, o1):
            assert_guards(o, view)
        ref, mag = tc_ref.conv_up64(small, W, b) if up else tc_ref.conv_down64(big, W)
        errs[family] = tuple(rel_err(o[view].view(shape), ref, mag, family) for o in (o3, o1))
    assess(f"conv_{case}_{'bias' if bias else 'nobias'}", K, errs)


# --------------------------------------------------------------------------------------- conv weight gradient
# NB, h, w, Cs, Cb.  "mn": both operands read in place (b200rl_conv_wgrad_mn: power-of-two grids, Cb % 32 == 0); the
# 32 pixels of a k-block are part of a row, whole rows or whole images.  "fb": the im2col_t + transpose2d + gemm_tc
# fallback, K padded to Pp = P rounded up to 4.
WGRAD_CASES = {
    "mn_row_part": (1, 64, 64, 48, 32),        # k-block = 32 of a 64-pixel row; 4 tiles, 66 splits
    "mn_rows": (16, 8, 8, 128, 64),            # k-block = 4 rows of 8
    "mn_images": (64, 4, 4, 256, 128),         # k-block = 2 whole 4 x 4 images
    "mn_direct": (16, 8, 8, 1152, 256),        # 32 x 9 = 288 tiles: one split, direct store
    "mn_k65536": (64, 32, 32, 64, 32),         # P = 65536, 4 tiles x 66 splits
    "fb_cb8": (4, 16, 16, 48, 8),              # Cb % 32 != 0 (one 128-row tile)
    "fb_cb12": (8, 16, 16, 64, 12),            # frame-stacked RGB: 192 rows
    "fb_h24": (2, 24, 24, 64, 32),             # 96 x 96 image, 24 x 24 grid: not a power of two
    "fb_h15_pp": (5, 15, 15, 48, 16),          # P = 1125: Pp = 1128 != P
    "fb_w40": (4, 8, 40, 96, 32),              # w = 40
    "fb_chunked": (1457, 40, 40, 48, 8),       # P = 2331200 > 32 * 65535: transpose2d runs in two launches
}


@pytest.mark.parametrize("acc", [False, True], ids=["store", "accumulate"])
@pytest.mark.parametrize("case", list(WGRAD_CASES))
def test_conv_wgrad_tc_precision(cu, case, acc):
    NB, h, w, Cs, Cb = WGRAD_CASES[case]
    P = NB * h * w
    Pp = (P + 3) // 4 * 4
    mn = case.startswith("mn")
    assert P >= 1024 and Cs >= 48 and Cb >= 8        # CudaOps.conv_wgrad takes the tensor-core route
    assert cu.lib.b200rl_conv_wgrad_mn_supported(NB, h, w, Cs, Cb) == int(mn)
    ws = int(cu.lib.b200rl_conv_wgrad_tc_workspace(NB, h, w, Cs, Cb))
    assert ws == (16 * Cs * Cb if mn else (Cs + 16 * Cb) * Pp + 16 * Cs * Cb)
    assert (P > 32 * 65535) == (case == "fb_chunked")
    shape = (Cs, Cb, 4, 4)
    errs = {}
    for i, family in enumerate(FAMILIES):
        small, big = draw((NB, h, w, Cs), family, 10 * i + 1), draw((NB, 2 * h, 2 * w, Cb), family, 10 * i + 2)
        dW0 = draw(shape, family, 10 * i + 3) if acc else None

        def run():
            buf, dW = guarded(shape)
            if acc:
                dW.copy_(dW0)
            cu.conv_wgrad(small, big, dW, accumulate=acc)
            return (buf,)

        (o3,), (o1,) = precisions(cu, run)
        view = slice(32, 32 + math.prod(shape))
        for o in (o3, o1):
            assert_guards(o, view)
        ref, mag = tc_ref.conv_wgrad64(small, big, dW0)
        errs[family] = tuple(rel_err(o[view].view(shape), ref, mag, family) for o in (o3, o1))
        del small, big, ref, mag
    assess(f"wgrad_{case}_{'acc' if acc else 'store'}", P, errs)
