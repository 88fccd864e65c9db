"""Every CUDA-core (FFMA) product route against a float64 reference: the SIMT GEMM and rank-K kernels of csrc/gemm.cu,
the batched MLP product of csrc/mlp.cu, the implicit-GEMM and weight-gradient convolutions of csrc/conv.cu, the
thin-channel convolutions of csrc/conv_thin.cu and the LSTM recurrence of csrc/lstm.cu (oracle/tc_ref.py,
oracle/simt_ref.py).

Each case runs under "highest", then "high", then "highest" again, and checks:
  - the intended route: the library's tensor-core and thin-channel predicates, and for the weight gradient the
    condition under which CudaOps.conv_wgrad takes the tensor-core route;
  - error <= tau1(K) = 2^-24 (16 + 2 sqrt(K)), K = the kernel's reduction length, plus the propagated term of an
    elementwise epilogue;
  - routes without atomics give bit-identical results in all three runs (FFMA does not depend on the matmul precision,
    and a fixed summation order reproduces).  Atomic routes (split-K sgemm / bgemm, every conv weight gradient) are NOT
    bit-reproducible: their partial sums land in any order, so every run is held to the bound instead.  One TF32 pass
    costs ~7e-4, far over tau1, so the "high" run also shows that no case took a tensor-core route;
  - nothing outside the output view is written.

Operand families and metrics as tests/test_gpu_tc_precision.py: positive U(0.5, 1) (rounding cannot cancel, a lost
product is a pure bias; max |C - C64| / C64) and mixed N(0, 1) (max |C - C64| / sum_k |a||b|).  A sequential fp32 FMA chain
of length K reaches ~1.0 sqrt(K) u on positive operands and a few u on mixed ones, so tau1 leaves ~2x headroom on
positive operands and rejects one dropped 16-wide k-step at every K up to 65536.
"""
import ctypes
import math

import pytest
import torch

from oracle import simt_ref, tc_ref
from oracle.simt_ref import U, tau1
from tests.test_gpu_tc_precision import FAMILIES, GUARD, assert_guards, draw, guarded, padded, rel_err

pytestmark = pytest.mark.gpu

MARGINS = {}          # case id -> measured errors and error / bound, kept for reporting


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    ops = CudaOps("cuda")
    assert ops.matmul_precision() == "highest"
    return ops


def runs(cu, run, atomic):
    """`run()` launches the op on fresh outputs and returns them.  Returns the outputs at "highest", "high" and
    "highest" again; without atomics the three must be bit-identical."""
    first = run()
    try:
        cu.set_matmul_precision("high")
        high = run()
    finally:
        cu.set_matmul_precision("highest")
    again = run()
    if not atomic:
        for a, b, c in zip(first, high, again):
            assert torch.equal(a, b), "FFMA route changed under matmul precision \"high\""
            assert torch.equal(a, c), "rerun is not bit-identical"
    return first, high, again


def ratio(got, ref, bound):
    """max |got - ref| / bound; an element whose bound is 0 must be exact"""
    d = (got.double() - ref).abs()
    return float(torch.where(d == 0, torch.zeros_like(d), d / bound).max())


def assess(case, K, errs, extra=None):
    """errs[family] = (error, error / bound) over every run of the case"""
    (p, pr), (m, mr) = errs["positive"], errs["mixed"]
    MARGINS[case] = {"K": K, "positive": p, "mixed": m, "err/bound": max(pr, mr), **(extra or {})}
    assert pr <= 1.0 and mr <= 1.0, ("error over tau1", MARGINS[case])


def product_errors(outs, view, ref, mag, family, K, shape=None):
    """(error, error / tau1(K)) of a plain product over all runs, with the guards of each run checked"""
    err = 0.0
    for (buf,) in outs:
        assert_guards(buf, view)
        got = buf[view] if shape is None else buf[view].view(shape)
        err = max(err, rel_err(got, ref, mag, family))
    return err, err / tau1(K)


# ---------------------------------------------------------------------------------------------------------- GEMM
# M, N, K, transA, transB, splits, lda (None: rows padded to 16 bytes).  b200rl_gemm_f32 tiles: 16x64 (BK 32) for
# M <= 32, else 128x32 for N <= 32, else 64x64 when M or N <= 64, else 128x128 (BK 16); split-K (fp32 atomics into C
# initialised by init2d / addbias2d) when tiles < 132 and K >= 8 BK, into min(ceil(264 / tiles), K / 4BK) slices rounded
# to whole k-steps.  Expected route per case:
GEMM_CASES = {
    "m16_nt_split8": (16, 1536, 1024, False, True, 8, None),   # 16x64, 24 tiles, 8 splits of 128
    "m16_nn_split4": (16, 1024, 512, False, False, 4, None),   # 16x64, 16 tiles, 4 splits of 128
    "m16_k24": (16, 256, 24, False, True, 1, None),            # 16x64, 4 tiles, K < 8 BK: direct
    "n32_nt_split32": (1000, 32, 2048, False, True, 32, None), # 128x32, 8 tiles, 32 splits of 64
    "n24_tn_wgrad": (256, 24, 4096, True, False, 64, None),    # dW = dY^T X: 128x32, 2 tiles, 64 splits of 64
    "n40_split3": (300, 40, 200, False, True, 3, None),        # 64x64, 5 tiles, 3 splits of 80
    "lda513_split7": (200, 300, 500, False, True, 7, 513),     # unaligned A rows: 128x128, 6 tiles, 7 splits of 80
    "k31_direct": (2048, 2048, 31, False, True, 1, None),      # K < 32: 128x128, 256 tiles, direct
    "tt": (129, 40, 36, True, True, 1, None),                  # 64x64, 3 tiles, K < 8 BK: direct
    # rank_k_nn_kernel: NN, K <= 8, M >= 1024, N, ldb, ldc multiples of 4 and 16-byte aligned B, C, bias
    "rank_k1": (2048, 256, 1, False, False, 1, None),
    "rank_k2": (2048, 256, 2, False, False, 1, None),
    "rank_k8": (1024, 64, 8, False, False, 1, None),
    "rank_k8_m1000": (1000, 256, 8, False, False, 1, None),    # M < 1024: 128x128, 16 tiles, direct
}


def gemm_errors(cu, family, M, N, K, tA, tB, splits, lda, bias=False, acc=False, seed=0):
    if lda is None:
        A = padded(*((K, M) if tA else (M, K)), family, seed)
    else:
        rows, cols = (K, M) if tA else (M, K)
        buf = torch.full((rows, lda), 1e6, device="cuda")
        buf[:, :cols] = draw((rows, cols), family, seed)
        A = buf[:, :cols]
    B = padded(*((N, K) if tB else (K, N)), family, seed + 1)
    b = draw((N,), family, seed + 2) if bias else None
    C0 = draw((M, N), family, seed + 3) if acc else None
    assert cu.lib.b200rl_gemm_tc_supported(ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(B.data_ptr()), M, N, K,
                                           A.stride(0), B.stride(0), int(tA), int(tB)) == 0
    ldc = (N + 7) // 4 * 4                                   # guard columns; rows stay 16-byte aligned (rank-K)
    view = (slice(1, M + 1), slice(0, N))

    def run():
        Cbuf = torch.full((M + 2, ldc), GUARD, device="cuda")
        if C0 is not None:
            Cbuf[view].copy_(C0)
        cu.gemm(A, B, Cbuf[view], tA, tB, bias=b, accumulate=acc)
        return (Cbuf,)

    outs = runs(cu, run, atomic=splits > 1)
    ref, mag = tc_ref.gemm64(A, B, tA, tB, bias=b, C0=C0)
    return product_errors(outs, view, ref, mag, family, K)


@pytest.mark.parametrize("case", list(GEMM_CASES))
def test_gemm_simt_precision(cu, case):
    M, N, K, tA, tB, splits, lda = GEMM_CASES[case]
    errs = {f: gemm_errors(cu, f, M, N, K, tA, tB, splits, lda, seed=10 * i) for i, f in enumerate(FAMILIES)}
    assess("gemm_" + case, K, errs, {"splits": splits})


# bias / accumulate through the split-K initialisation (init2d: C = bias; addbias2d: C += bias; accumulate alone keeps
# C) and through the direct store; and through the rank-K kernel
EPI_ROUTES = {"split": "m16_nt_split8", "direct": "m16_k24", "rank_k": "rank_k2", "tiles_128x32": "n32_nt_split32"}


@pytest.mark.parametrize("route", list(EPI_ROUTES))
@pytest.mark.parametrize("epi", ["bias", "acc", "bias_acc"])
def test_gemm_simt_epilogue_precision(cu, route, epi):
    M, N, K, tA, tB, splits, lda = GEMM_CASES[EPI_ROUTES[route]]
    errs = {f: gemm_errors(cu, f, M, N, K, tA, tB, splits, lda, bias="bias" in epi, acc="acc" in epi, seed=10 * i + 100)
            for i, f in enumerate(FAMILIES)}
    assess(f"gemm_epilogue_{route}_{epi}", K, errs, {"splits": splits})


@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("acc", [False, True], ids=["store", "accumulate"])
def test_gemm_k0(cu, bias, acc):
    """an empty product: C = bias (or 0), or C += bias when accumulating (C unchanged without a bias)"""
    M, N = 37, 50
    A, B = torch.ones(M, 4, device="cuda"), torch.ones(4, N, device="cuda")   # real buffers: the entry point refuses NULL
    b = draw((N,), "mixed", 1) if bias else None
    C0 = draw((M, N), "mixed", 2)
    buf, view = torch.full((M + 2, N + 3), GUARD, device="cuda"), (slice(1, M + 1), slice(1, N + 1))
    buf[view].copy_(C0)
    p = lambda t: ctypes.c_void_p(0 if t is None else t.data_ptr())      # noqa: E731
    cu._ck(cu.lib.b200rl_gemm_f32(p(A), p(B), p(buf[view]), p(b), M, N, 0, 4, N, N + 3, 0, 0, int(acc), cu._st()))
    want = (C0 if acc else torch.zeros_like(C0)) + (b if bias else 0.0)
    assert torch.equal(buf[view], want)
    assert_guards(buf, view)


# ---------------------------------------------------------------------------------------------------------- bgemm
# b200rl_bgemm tiles: 64x32 when N <= 32 and ceil(M / 64) x nets >= 132, else 64x64 when the 64x64 tiles (x nets) fill
# the 132 SMs, else 32x32.  Split-K only for plain products without bias (weight gradients) whose tiles do not fill the
# SMs and K >= 256: ceil(528 / tiles) slices, at most K / 64 and 128, of whole 32-deep k-steps; C (and rsum) are zeroed
# first unless accumulating, and partial tiles add with float2 atomics where the address allows, scalar ones elsewhere.
#
# layout: "nt" forward y = x W^T (A [n|1, M, K], W [n, N, K] read transposed), "nn" input gradient dY W (B [n, K, N]
# possibly a column slice), "tn" weight gradient dY^T X (A = dY [n, K, M] read transposed, B = X [1|n, K, N]).
# name: layout, nets, shared operand, M, N, K, epi, bias, accumulate, rsum, extra C / aux columns, splits
BGEMM_CASES = {}
for _cfg, (_nets, _M, _N, _K, _shared) in {"t32": (2, 200, 72, 96, False),      # 32x32, 7 x 3 x 2 = 42 tiles
                                           "t64": (2, 2048, 256, 64, True),      # 64x64, 32 x 4 x 2 = 256 tiles
                                           "t64x32": (2, 4300, 24, 64, True)}.items():   # 64x32, 68 x 2 = 136 tiles
    # forward, with bias: never split (on positive operands tanh saturates to 1; the mixed family carries that epilogue)
    for _epi in ("none", "relu", "tanh"):
        BGEMM_CASES[f"{_cfg}_{_epi}"] = ("nt", _nets, _shared, _M, _N, _K, _epi, True, False, False, 0, 1)
    for _epi in ("drelu", "dtanh"):                                               # input gradient, aux of the layer
        BGEMM_CASES[f"{_cfg}_{_epi}"] = ("nn", _nets, False, _M, _N, _K, _epi, False, False, False, 0, 1)
BGEMM_CASES.update({
    # PPO's second critic / actor input gradient adds into the first (accumulate), on a column slice of the features
    "ppo_dx_drelu_acc": ("nn", 1, False, 64, 40, 64, "drelu", False, True, False, 10, 1),   # 32x32, 4 tiles
    "split_zero": ("tn", 1, False, 64, 64, 4096, "none", False, False, False, 0, 64),       # 4 tiles, 64 splits of 64
    "split_acc": ("tn", 1, False, 64, 64, 4096, "none", False, True, False, 0, 64),
    "split_rsum": ("tn", 2, True, 64, 48, 2048, "none", False, False, True, 0, 32),         # 8 tiles, 32 splits of 64
    "split_rsum_acc": ("tn", 2, True, 64, 48, 2048, "none", False, True, True, 0, 32),
    "direct_rsum_acc": ("tn", 2, True, 64, 48, 128, "none", False, True, True, 0, 1),       # K < 256: no split
    "split_odd_ldc": ("tn", 1, False, 64, 64, 4096, "none", False, False, False, 1, 64),    # ldc 65: scalar atomics on odd rows
    # the engines' weight gradients (dY^T X with the bias gradient as rsum)
    "ppo_wgrad_64rows": ("tn", 1, False, 64, 17, 64, "none", False, False, True, 0, 1),     # 64-row minibatch: direct
    "rppo_dW_ih_1120": ("tn", 1, False, 256, 20, 1120, "none", False, False, True, 0, 12),  # 8 tiles, 12 splits of 96
    "rppo_dW_hh_1120": ("tn", 1, False, 256, 64, 1120, "none", False, False, False, 0, 12), # hbuf[:-1]: 16 tiles, 12 x 96
    "a2c_wgrad_k2048": ("tn", 1, False, 64, 64, 2048, "none", False, False, True, 0, 32),   # 4 tiles, 32 splits of 64
    "a2c_wgrad_k65536": ("tn", 1, False, 64, 64, 65536, "none", False, False, True, 0, 128),  # 128 splits of 512
})


def bgemm_operands(family, layout, nets, shared, M, N, K, seed, case):
    if layout == "nt":
        A = draw((1 if shared else nets, M, K), family, seed)
        B = draw((nets, N, K), family, seed + 1).transpose(1, 2)
    elif layout == "nn":
        A = draw((nets, M, K), family, seed)
        B = draw((nets, K, N + 7), family, seed + 1)[:, :, 5:5 + N]          # a column slice of W
    else:
        A = draw((nets, K, M), family, seed).transpose(1, 2)
        if case == "rppo_dW_hh_1120":                        # the recurrent PPO engine's shifted hidden-state rows
            T, Bs = 16, 70
            hbuf = torch.full((T + 1, Bs, N), 1e6, device="cuda")
            hbuf[:-1] = draw((T, Bs, N), family, seed + 1)
            B = hbuf[:-1].view(1, K, N)
        else:
            B = draw((1 if shared else nets, K, N), family, seed + 1)
    return A, B


EPI_SLOPE = {"none": 1.0, "relu": 1.0, "tanh": 1.0}        # |f'| <= 1


@pytest.mark.parametrize("case", list(BGEMM_CASES))
def test_bgemm_simt_precision(cu, case):
    layout, nets, shared, M, N, K, epi, has_bias, acc, has_rsum, extra, splits = BGEMM_CASES[case]
    atomic = splits > 1
    errs = {}
    for i, family in enumerate(FAMILIES):
        seed = 10 * i
        A, B = bgemm_operands(family, layout, nets, shared, M, N, K, seed, case)
        bias = draw((nets, N), family, seed + 2) if has_bias else None
        aux = None
        if epi in ("drelu", "dtanh"):
            aux = draw((nets, M, N + extra), family, seed + 3)
            aux = aux.clamp_min(0.0) if epi == "drelu" else torch.tanh(aux)
            if epi == "drelu":
                aux.view(-1)[::3] = 0.0                      # exact zeros: ReLU'(0) = 0
            aux = aux[:, :, extra:]
        C0 = draw((nets, M, N), family, seed + 4) if acc else None
        r0 = draw((nets, M), family, seed + 5) if (acc and has_rsum) else None
        W = N + extra

        def run():
            # C: rows of W = N + extra floats (a column slice when extra > 0) inside guard rows
            cbuf = torch.full((nets, M + 2, W), GUARD, device="cuda")
            C = cbuf[:, 1:M + 1, extra:]
            rbuf = torch.full((nets, M + 2), GUARD, device="cuda")
            rsum = rbuf[:, 1:M + 1] if has_rsum else None
            if C0 is not None:
                C.copy_(C0)
            if r0 is not None:
                rsum.copy_(r0)
            cu.bgemm(A, B, C, bias=bias, aux=aux, rsum=rsum, epi=epi, accumulate=acc)
            return cbuf, rbuf

        outs = runs(cu, run, atomic)
        ref, mag, rs = simt_ref.bgemm64(A, B, bias, aux, epi, C0)
        c0 = C0.double().abs() if C0 is not None else 0.0
        pre_mag = mag - c0
        if epi == "dtanh":
            y2 = aux.double() ** 2
            pre = simt_ref.bgemm64(A, B, bias)[0]
            # (1 - y^2) and the product round once each; y^2 itself is u y^2 of |pre|
            bound = tau1(K) * ((1.0 - y2) * pre_mag + c0) + U * y2 * pre.abs() + 4 * U * ref.abs()
        elif epi == "drelu":
            bound = tau1(K) * ((aux > 0).double() * pre_mag + c0)     # masked entries: exactly C0 (or 0)
        else:
            bound = tau1(K) * (EPI_SLOPE[epi] * pre_mag + c0) + (4 * U * ref.abs() if epi == "tanh" else 0.0)
        rs_ref = rs + (r0.double() if r0 is not None else 0.0)
        rs_bound = tau1(K) * (A.double().abs().sum(-1).expand(nets, -1) + (r0.double().abs() if r0 is not None else 0.0))
        err, r = 0.0, 0.0
        for cbuf, rbuf in outs:
            assert_guards(cbuf, (slice(None), slice(1, M + 1), slice(extra, None)))
            got = cbuf[:, 1:M + 1, extra:]
            err = max(err, float(((got.double() - ref).abs() / mag).max()))
            r = max(r, ratio(got, ref, bound))
            if has_rsum:
                assert_guards(rbuf, (slice(None), slice(1, M + 1)))
                r = max(r, ratio(rbuf[:, 1:M + 1], rs_ref, rs_bound))
            else:
                assert bool((rbuf == GUARD).all())
        errs[family] = (err, r)
    assess("bgemm_" + case, K, errs, {"splits": splits})


# ------------------------------------------------------------------------------------- SIMT convolutions
# kind, NB, h, w, Cs, Cb, thin (the thin-channel predicate of the direction).  None of these is a tensor-core shape
# (gathered channels not a multiple of 32, or a grid that does not tile by 128 pixels).  conv_igemm_kernel: 128 pixels x
# BN output channels, BN = 32 / 64 / 128 by Cout; the gather is 2 x float4 when Cin % 8 == 0, scalar otherwise.
CONV_CASES = {
    "down_bn32_fast": ("down", 4, 6, 10, 24, 16, False),        # Cin 16, K = 256
    "down_bn32_generic": ("down", 2, 5, 7, 20, 3, False),       # Cin 3, K = 48
    "down_bn64_fast": ("down", 2, 12, 12, 48, 40, False),       # Cin 40, K = 640
    "down_bn64_generic": ("down", 2, 9, 9, 64, 12, False),      # Cin 12, K = 192
    "down_bn128_fast": ("down", 1, 10, 10, 200, 200, False),    # Cout 200: 2 column tiles; K = 3200
    "down_bn128_generic": ("down", 2, 6, 6, 96, 20, False),     # Cin 20, K = 320
    "up_bn32_fast": ("up", 3, 5, 6, 24, 20, False),             # Cin 24, K = 96
    "up_bn32_generic": ("up", 2, 7, 5, 10, 3, False),           # Cin 10, K = 40
    "up_bn64_fast": ("up", 2, 12, 12, 64, 48, False),           # 12 x 12 grid, K = 256
    "up_bn64_generic": ("up", 2, 8, 8, 36, 64, False),          # Cin 36, K = 144
    "up_bn128_fast": ("up", 1, 10, 10, 800, 200, False),        # K = 3200
    "up_bn128_generic": ("up", 2, 6, 6, 20, 130, False),        # Cin 20, K = 80
    # conv_down_thin_kernel<CS>: 3-channel 64-wide images, two output rows per warp (h = 1 and odd h: a lone last row)
    "down_thin_cs32_h1": ("down", 3, 1, 32, 32, 3, True),
    "down_thin_cs64_h5": ("down", 2, 5, 32, 64, 3, True),
    "down_thin_cs96_h7": ("down", 2, 7, 32, 96, 3, True),
    # conv_up_thin_kernel<3, CS>: w != 32
    "up_thin_cs32_w16": ("up", 2, 6, 16, 32, 3, True),
    "up_thin_cs48_w20": ("up", 2, 5, 20, 48, 3, True),
    "up_thin_cs64_w16": ("up", 1, 4, 16, 64, 3, True),
    "up_thin_cs96_w20": ("up", 1, 3, 20, 96, 3, True),
    # conv_up_thin2_kernel<CS>: w = 32, 8-row CTA units with a partial last unit
    "up_thin2_cs32_h5": ("up", 2, 5, 32, 32, 3, True),
    "up_thin2_cs64_h11": ("up", 1, 11, 32, 64, 3, True),
    "up_thin2_cs96_h13": ("up", 1, 13, 32, 96, 3, True),
    # Dreamer-V3's RGB layers at batch 1024 on 64 x 64 images
    "down_thin_rgb_nb1024": ("down", 1024, 32, 32, 32, 3, True),
    "up_thin2_rgb_nb1024": ("up", 1024, 32, 32, 32, 3, True),
}
CONV_PARAMS = [pytest.param(c, b, id=f"{c}-{'bias' if b else 'nobias'}") for c, v in CONV_CASES.items()
               for b in ((False, True) if v[0] == "up" else (False,))]      # the Conv2d forward has no bias


@pytest.mark.parametrize("case,bias", CONV_PARAMS)
def test_conv_simt_precision(cu, case, bias):
    kind, NB, h, w, Cs, Cb, thin = CONV_CASES[case]
    up = kind == "up"
    assert cu.lib.b200rl_conv_tc_supported(int(up), NB, h, w, Cs, Cb) == 0
    assert (cu.lib.b200rl_thin_up_supported(Cs, Cb) if up else cu.lib.b200rl_thin_down_supported(w, Cs, Cb)) == int(thin)
    K = 4 * Cs if up else 16 * Cb
    shape = (NB, 2 * h, 2 * w, Cb) if up else (NB, h, w, Cs)
    view = slice(32, 32 + math.prod(shape))
    errs = {}
    for i, family in enumerate(FAMILIES):
        big, small = draw((NB, 2 * h, 2 * w, Cb), family, 10 * i + 1), draw((NB, h, w, Cs), family, 10 * i + 2)
        W, b = draw((Cs, Cb, 4, 4), family, 10 * i + 3), (draw((Cb,), family, 10 * i + 4) if bias else None)

        def run():
            buf, out = guarded(shape)
            if up:
                cu.conv_up(small, W, out, b)
            else:
                cu.conv_down(big, W, out)
            return (buf,)

        outs = runs(cu, run, atomic=False)
        ref, mag = tc_ref.conv_up64(small, W, b) if up else tc_ref.conv_down64(big, W)
        errs[family] = product_errors(outs, view, ref, mag, family, K, shape)
        del big, small, ref, mag, outs
    assess(f"conv_{case}_{'bias' if bias else 'nobias'}", K, errs)


# --------------------------------------------------------------------------------------- conv weight gradient
# NB, h, w, Cs, Cb.  All outside CudaOps.conv_wgrad's tensor-core condition (P >= 1024, Cs >= 48, Cb >= 8).  Every route
# adds per-CTA partial sums with fp32 atomics into dW (zeroed first unless accumulating).  b200rl_conv_wgrad takes
# conv_wgrad_thin (Cb <= 4, Cs % 32 == 0, Cs <= 128; conv_wgrad_thin2 when also Cb = 3 and w = 32), else
# conv_wgrad_smallcb<Cb> (Cb <= 4, 16 Cs Cb <= 6144), else conv_wgrad_kernel: 64 x 64 (cs, cb) tiles x 16 taps x pixel
# splits, max(1, min(ceil(528 / tiles), P / 256)) of them.
WGRAD_CASES = {
    "igemm_1split": (2, 10, 10, 40, 24, False),          # P = 200: one split
    "igemm_8splits": (8, 16, 16, 100, 6, False),         # 2 x 1 tiles, P = 2048: 8 splits of 256
    "igemm_p65536": (64, 32, 32, 32, 16, False),         # 1 tile, P = 65536: 33 splits of 2000
    "smallcb1_cs40": (4, 12, 12, 40, 1, False),
    "smallcb2_cs130": (4, 12, 12, 130, 2, False),
    "smallcb3_cs40": (4, 12, 12, 40, 3, False),
    "smallcb4_cs40": (4, 12, 12, 40, 4, False),
    "thin1_w40": (2, 3, 40, 32, 1, True),                # 40-wide rows: a partial 32-pixel tile
    "thin2_w40": (2, 3, 40, 64, 2, True),
    "thin3_w40": (1, 4, 40, 96, 3, True),
    "thin4_w40": (1, 3, 40, 128, 4, True),
    "thin2x_cs32": (2, 6, 32, 32, 3, True),              # conv_wgrad_thin2
    "thin2x_cs64": (1, 8, 32, 64, 3, True),
    "thin2x_cs96": (1, 5, 32, 96, 3, True),
    "thin2x_cs128": (1, 4, 32, 128, 3, True),
    "thin2x_rgb_nb1024": (1024, 32, 32, 32, 3, True),    # Dreamer-V3's RGB layer at batch 1024: K = 1048576 pixels
}


@pytest.mark.parametrize("acc", [False, True], ids=["store", "accumulate"])
@pytest.mark.parametrize("case", list(WGRAD_CASES))
def test_conv_wgrad_simt_precision(cu, case, acc):
    NB, h, w, Cs, Cb, thin = WGRAD_CASES[case]
    P = NB * h * w
    assert not (P >= 1024 and Cs >= 48 and Cb >= 8)         # CudaOps.conv_wgrad keeps these off the tensor cores
    assert cu.lib.b200rl_thin_wgrad_supported(Cs, Cb) == int(thin)
    shape = (Cs, Cb, 4, 4)
    view = slice(32, 32 + math.prod(shape))
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

        outs = runs(cu, run, atomic=True)
        ref, mag = tc_ref.conv_wgrad64(small, big, dW0)
        errs[family] = product_errors(outs, view, ref, mag, family, P, shape)
        del small, big, ref, mag, outs
    assess(f"wgrad_{case}_{'acc' if acc else 'store'}", P, errs)


# ---------------------------------------------------------------------------------------------------------- LSTM
# T, B, H.  pick_sb: sequences per CTA double (up to 8) while B > 2 x 132 x SB and the doubled state fits 160 KB;
# dynamic shared memory SB x 24 H bytes, opted in above 48 KB.
LSTM_CASES = {
    "sb1": (16, 70, 64),
    "sb2_h100": (2, 300, 100),             # H not a multiple of 32
    "sb4": (32, 530, 256),
    "sb8_last_cta_1seq": (8, 1057, 64),    # 133 CTAs, the last one with one sequence
    "sb8_smem61440": (4, 1200, 320),       # 61440 B of shared memory
    "sb1_smem50400": (1, 16, 2100),        # 50400 B, 8400 gate rows per step
}
LSTM_PARAMS = [pytest.param(c, m, id=f"{c}-{m}") for c, v in LSTM_CASES.items()
               for m in (("all_T",) if v[0] == 1 else ("all_1", "all_T", "mixed"))]


def lstm_inputs(family, T, B, H, mode, seed):
    if mode == "all_1":
        lengths = torch.ones(B, dtype=torch.int32)
    elif mode == "all_T":
        lengths = torch.full((B,), T, dtype=torch.int32)
    else:
        lengths = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(seed), dtype=torch.int32)
        lengths[0], lengths[-1] = 1, T
    # W scaled by 1 / H: the absolute bound of the backward is propagated through |W|^T, which stays contractive
    return (draw((T, B, 4 * H), family, seed + 1), draw((4 * H, H), family, seed + 2) / H,
            0.5 * draw((B, H), family, seed + 3), 0.5 * draw((B, H), family, seed + 4), lengths.cuda(),
            draw((T, B, H), family, seed + 5))


def lstm_fwd_bounds(xw, W, h0, c0, out, cs):
    """Teacher-forced float64 step from the kernel's own previous state, and a first-order bound on each output.

    Gates: |act'(z)| tau1(H) (|xw| + sum |W||h|) for the product, plus 8u |gate| for expf / tanhf (2 ulp = 4u) and the
    sigmoid's add and division.  c = f c' + i g and h = o tanh(c) propagate those, plus their own roundings."""
    T, B, H = out.shape
    hp = torch.cat((h0.unsqueeze(0), out[:-1]))
    cp = torch.cat((c0.unsqueeze(0), cs[:-1]))
    gates, c, h, mag = simt_ref.lstm_step64(xw, W, hp, cp)
    i, f, g, o = torch.split(gates, H, -1)
    slope = torch.cat((i * (1 - i), f * (1 - f), 1 - g * g, o * (1 - o)), -1)
    e_gate = slope * tau1(H) * mag + 8 * U * gates.abs()
    e_i, e_f, e_g, e_o = torch.split(e_gate, H, -1)
    cpd = cp.double()
    e_c = cpd.abs() * e_f + g.abs() * e_i + i.abs() * e_g + 3 * U * ((f * cpd).abs() + (i * g).abs())
    tc = torch.tanh(c)
    e_h = tc.abs() * e_o + o.abs() * (1 - tc * tc) * e_c + 5 * U * (o * tc).abs()
    return (gates, c, h), (e_gate, e_c, e_h)


@pytest.mark.parametrize("case,mode", LSTM_PARAMS)
def test_lstm_simt_precision(cu, case, mode):
    T, B, H = LSTM_CASES[case]
    G = 4 * H
    shapes = ((T, B, H), (T, B, G), (T, B, H), (B, H), (B, H), (T, B, G))      # out, gates, cs, hT, cT, d_gates
    margins, errs = {"fwd/bound": 0.0, "bwd/bound": 0.0, "bwd bound / max|dg|": 0.0}, {}
    for k, family in enumerate(FAMILIES):
        xw, W, h0, c0, lengths, d_out = lstm_inputs(family, T, B, H, mode, seed=100 * k + T + B)

        def run():
            bufs = [guarded(s) for s in shapes]
            out, gates, cs, hT, cT, dg = (v for _, v in bufs)
            cu.lstm_seq_fwd(xw, W, h0, c0, lengths, out, gates, cs, hT, cT)
            cu.lstm_seq_bwd(d_out, W, gates, cs, c0, lengths, dg)
            return tuple(b for b, _ in bufs)

        first, _, _ = runs(cu, run, atomic=False)
        views = []
        for buf, s in zip(first, shapes):
            v = slice(32, 32 + math.prod(s))
            assert_guards(buf, v)
            views.append(buf[v].view(s))
        out, gates, cs, hT, cT, dg = views
        valid = (torch.arange(T, device="cuda").unsqueeze(1) < lengths.long().unsqueeze(0)).unsqueeze(-1)
        # padded steps are exactly zero; (hT, cT) is the state after each sequence's last valid step
        for t_ in (out, gates, cs, dg):
            assert bool((t_.masked_select(~valid) == 0).all()), "padded step not zero"
        last = (lengths.long() - 1).view(1, B, 1)
        assert torch.equal(hT, out.gather(0, last.expand(1, B, H))[0])
        assert torch.equal(cT, cs.gather(0, last.expand(1, B, H))[0])
        # forward, teacher-forced
        (g64, c64, h64), (eg, ec, eh) = lstm_fwd_bounds(xw, W, h0, c0, out, cs)
        v = valid.double()
        fr = max(ratio(gates * v, g64 * v, eg), ratio(cs * v, c64 * v, ec), ratio(out * v, h64 * v, eh))
        # backward on the kernel's own saved forward
        dg64, bound = simt_ref.lstm_bwd64(d_out, W, gates, cs, c0, lengths)
        br = ratio(dg, dg64, bound)
        margins["fwd/bound"] = max(margins["fwd/bound"], fr)
        margins["bwd/bound"] = max(margins["bwd/bound"], br)
        margins["bwd bound / max|dg|"] = max(margins["bwd bound / max|dg|"], float(bound.max() / dg64.abs().max()))
        errs[family] = (float((dg.double() - dg64).abs().max()), max(fr, br))
    assess(f"lstm_{case}_{mode}", 4 * H, errs, margins)
