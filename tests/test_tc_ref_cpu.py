"""The float64 reference of the tensor-core products (oracle/tc_ref.py) against the fp32 op emulator
(oracle/ops_emul.py) on small shapes, so that a layout mistake in the reference fails without a GPU.  The GPU
precision tests (tests/test_gpu_tc_precision.py) hold the kernels to this reference."""
import pytest
import torch

from oracle import tc_ref
from oracle.ops_emul import EmulOps

em = EmulOps()


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def check(ref64, mag, got32, what):
    """fp32 agreement, per element, against the magnitude the reference reports"""
    assert ref64.dtype == torch.float64 and mag.shape == ref64.shape, what
    assert bool((mag >= ref64.abs() * (1 - 1e-12)).all()), what            # |sum| <= sum |.|
    err = (got32.double() - ref64).abs() / (mag + 1e-30)
    assert float(err.max()) < 1e-6, (what, float(err.max()))


@pytest.mark.parametrize("transA", [False, True])
@pytest.mark.parametrize("transB", [False, True])
@pytest.mark.parametrize("epi", ["plain", "bias", "acc", "bias_acc"])
def test_gemm64(transA, transB, epi):
    M, N, K = 13, 7, 29
    A = rnd(*((K, M) if transA else (M, K)), seed=1)
    B = rnd(*((N, K) if transB else (K, N)), seed=2)
    bias = rnd(N, seed=3) if "bias" in epi else None
    C0 = rnd(M, N, seed=4) if "acc" in epi else None
    C = C0.clone() if C0 is not None else torch.empty(M, N)
    em.gemm(A, B, C, transA, transB, bias=bias, accumulate=C0 is not None)
    ref, mag = tc_ref.gemm64(A, B, transA, transB, bias=bias, C0=C0)
    check(ref, mag, C, "gemm")
    # the magnitude is the product of the absolute operands (+ |bias| + |C0|)
    a, b = (A.t() if transA else A).double().abs(), (B.t() if transB else B).double().abs()
    want = a @ b + (bias.double().abs() if bias is not None else 0) + (C0.double().abs() if C0 is not None else 0)
    assert torch.allclose(mag, want, rtol=1e-12, atol=0)


@pytest.mark.parametrize("NB,h,w,Cs,Cb", [(2, 3, 5, 6, 4), (1, 4, 4, 3, 7), (3, 1, 2, 5, 2)])
def test_conv64(NB, h, w, Cs, Cb):
    big, small = rnd(NB, 2 * h, 2 * w, Cb, seed=1), rnd(NB, h, w, Cs, seed=2)
    W, bs, bb = rnd(Cs, Cb, 4, 4, seed=3), rnd(Cs, seed=4), rnd(Cb, seed=5)
    for bias in (None, bs):
        out = torch.empty(NB, h, w, Cs)
        em.conv_down(big, W, out)
        if bias is not None:
            out += bias
        ref, mag = tc_ref.conv_down64(big, W, bias)
        check(ref, mag, out, "conv_down")
    for bias in (None, bb):
        out = torch.empty(NB, 2 * h, 2 * w, Cb)
        em.conv_up(small, W, out, bias)
        ref, mag = tc_ref.conv_up64(small, W, bias)
        check(ref, mag, out, "conv_up")
    dW0 = rnd(Cs, Cb, 4, 4, seed=6)
    for acc in (False, True):
        out = dW0.clone() if acc else torch.empty(Cs, Cb, 4, 4)
        em.conv_wgrad(small, big, out, accumulate=acc)
        ref, mag = tc_ref.conv_wgrad64(small, big, dW0 if acc else None)
        check(ref, mag, out, "conv_wgrad")
    # the magnitude of a conv is the conv of the absolute operands: one tap of one output element by hand
    _, mag = tc_ref.conv_down64(big, W)
    y, x = h - 1, 0                                        # a border pixel: taps with ky = 0 or kx = 0 fall off the image
    want = sum(float(big[0, 2 * y - 1 + ky, 2 * x - 1 + kx].double().abs() @ W[0, :, ky, kx].double().abs())
               for ky in range(4) for kx in range(4) if 0 <= 2 * y - 1 + ky < 2 * h and 0 <= 2 * x - 1 + kx < 2 * w)
    assert abs(float(mag[0, y, x, 0]) - want) <= 1e-12 * want


@pytest.mark.parametrize("act", [0, 1])
def test_gemm_ln64(act):
    M, N, K = 9, 24, 17
    A, W = rnd(M, K, seed=1), rnd(N, K, seed=2)
    gamma, beta = rnd(N, seed=3) + 1.0, rnd(N, seed=4)
    pre = torch.empty(M, N)
    em.gemm(A, W, pre, False, True)
    out = torch.empty(M, N)
    em.ln_act_fwd(pre, gamma, beta, 1e-3, act, out)
    ref, mag, pre64 = tc_ref.gemm_ln64(A, W, gamma, beta, 1e-3, act)
    check(pre64, mag, pre, "gemm_ln pre")
    assert float((out.double() - ref).abs().max()) < 1e-5


def test_gemm_ln_gru64():
    M, R, K = 9, 8, 21
    A, W = rnd(M, K, seed=1), rnd(3 * R, K, seed=2)
    gamma, beta, h_prev = rnd(3 * R, seed=3) + 1.0, rnd(3 * R, seed=4), rnd(M, R, seed=5)
    pre, ln, h = torch.empty(M, 3 * R), torch.empty(M, 3 * R), torch.empty(M, R)
    em.gemm(A, W, pre, False, True)
    em.ln_act_fwd(pre, gamma, beta, 1e-3, 0, ln)
    em.gru_gate_fwd(ln, h_prev, h)
    h64, mag, pre64, ln64 = tc_ref.gemm_ln_gru64(A, W, gamma, beta, 1e-3, h_prev)
    check(pre64, mag, pre, "gemm_ln_gru pre")
    assert float((ln.double() - ln64).abs().max()) < 1e-5
    assert float((h.double() - h64).abs().max()) < 1e-5
