"""Pre-split weight operands of the tensor-core GEMM (csrc/gemm_tc.cu): B given as its TF32 hi / lo planes, loaded by TMA
straight into the wgmma operand stages, must give exactly the bits of the raw-B kernel that splits B per tile.

Every route runs in both matmul precisions on the same inputs through both paths and is compared with torch.equal:
NT products (BN 64 and 128, split-K, ragged M and N, M < 128, bias, accumulate, a persistent walk over the deeper
pre-split ring), the input-gradient product on a transposed plane, gemm_ln modes 0 and 1, and conv down / up / UP4.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

PRECISIONS = ("highest", "high")
EPS = 1e-3


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    ops = CudaOps("cuda")
    assert ops.use_tc, "the tensor-core paths are disabled (B200RL_DISABLE_TC=1)"
    yield ops
    ops.set_matmul_precision("highest")


@pytest.fixture(params=PRECISIONS)
def precision(cu, request):
    cu.set_matmul_precision(request.param)
    yield request.param
    cu.set_matmul_precision("highest")


def draw(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda")


def p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ck(cu, rc):
    assert rc == 0, cu.lib.b200rl_last_error().decode()


def split(cu, X):
    hi, lo = torch.empty_like(X), torch.empty_like(X)
    ck(cu, cu.lib.b200rl_tf32_split(p(X), p(hi), p(lo), X.numel(), st()))
    return hi, lo


def split_t(cu, W):
    """hi^T, lo^T [Kin][ldt] of W [Nout][Kin], ldt = Nout rounded up to a multiple of 4"""
    rows, cols = W.shape
    ldt = (rows + 3) // 4 * 4
    hi, lo = (torch.full((cols, ldt), float("nan"), device="cuda") for _ in range(2))
    ck(cu, cu.lib.b200rl_tf32_split_t(p(W), p(hi), p(lo), rows, cols, W.stride(0), ldt, st()))
    return hi, lo


# ------------------------------------------------------------------------------------------------ the split kernels
@pytest.mark.parametrize("n", [1, 7, 4096, 1000003])
def test_tf32_split_is_the_bit_mask(cu, n):
    X = draw((n,), 1) * 37.0
    hi, lo = split(cu, X)
    want = (X.view(torch.int32) & -8192).view(torch.float32)
    assert torch.equal(hi, want)
    assert torch.equal(lo, X - want)
    assert torch.equal(hi + lo, X)


@pytest.mark.parametrize("rows,cols", [(255, 512), (512, 1536), (33, 70)])
def test_tf32_split_t_transposes_and_zeroes_the_padding(cu, rows, cols):
    W = draw((rows, cols + 5), 2)[:, :cols]           # a strided view: ldw > cols
    hi, lo = split_t(cu, W)
    want_hi, want_lo = split(cu, W.contiguous())
    assert torch.equal(hi[:, :rows], want_hi.t()) and torch.equal(lo[:, :rows], want_lo.t())
    assert not hi[:, rows:].any() and not lo[:, rows:].any()


# ------------------------------------------------------------------------------------------------------- NT products
# (M, N, K): BN 64 and 128; split-K (tiles < 264 and >= 8 k-blocks); ragged M and N; M < 128; K not a multiple of 32;
# 300 row tiles walk a persistent grid through the ring at every stage / phase offset
NT_CASES = [(256, 64, 512), (256, 256, 512), (1024, 512, 4096), (1000, 200, 1536), (64, 3072, 1280), (300, 130, 100),
            (128 * 300, 64, 160), (128 * 300, 256, 128), (128 * 300, 256, 4128)]


@pytest.mark.parametrize("M,N,K", NT_CASES, ids=[f"M{m}-N{n}-K{k}" for m, n, k in NT_CASES])
@pytest.mark.parametrize("epi", ["plain", "bias", "accumulate"])
def test_gemm_nt_presplit_matches_raw(cu, precision, M, N, K, epi):
    A, B = draw((M, K), 3), draw((N, K), 4)
    bias = draw((N,), 5) if epi == "bias" else None
    C0 = draw((M, N), 6) if epi == "accumulate" else torch.zeros(M, N, device="cuda")
    acc = int(epi == "accumulate")
    hi, lo = split(cu, B)
    assert cu.lib.b200rl_gemm_tc_presplit_supported(p(A), p(hi), p(lo), M, N, K, K, K) == 1
    raw, pre = C0.clone(), C0.clone()
    ck(cu, cu.lib.b200rl_gemm_tc(p(A), p(B), p(raw), p(bias), M, N, K, K, K, N, 0, 1, acc, st()))
    ck(cu, cu.lib.b200rl_gemm_tc_presplit(p(A), p(hi), p(lo), p(pre), p(bias), M, N, K, K, K, N, acc, st()))
    assert torch.equal(raw, pre)


# input gradient dX = dY W on the transposed plane of W [Nout][Kin]; Nout = 255 pads the plane's rows to 256 floats
NN_CASES = [(15360, 1536, 512), (1024, 512, 255), (200, 1024, 1536), (64, 96, 64)]


@pytest.mark.parametrize("M,Kin,Nout", NN_CASES, ids=[f"M{m}-Kin{k}-Nout{n}" for m, k, n in NN_CASES])
def test_gemm_nn_transposed_plane_matches_raw(cu, precision, M, Kin, Nout):
    lda = (Nout + 3) // 4 * 4
    dY, W = draw((M, lda), 7)[:, :Nout], draw((Nout, Kin), 8)
    hi, lo = split_t(cu, W)
    raw, pre = torch.zeros(M, Kin, device="cuda"), torch.zeros(M, Kin, device="cuda")
    ck(cu, cu.lib.b200rl_gemm_tc(p(dY), p(W), p(raw), None, M, Kin, Nout, lda, Kin, Kin, 0, 0, 0, st()))
    ld = hi.stride(0)
    assert cu.lib.b200rl_gemm_tc_presplit_supported(p(dY), p(hi), p(lo), M, Kin, Nout, lda, ld) == 1
    ck(cu, cu.lib.b200rl_gemm_tc_presplit(p(dY), p(hi), p(lo), p(pre), None, M, Kin, Nout, lda, ld, Kin, 0, st()))
    assert torch.equal(raw, pre)


# CudaOps.gemm hands products of PRESPLIT_MIN_ROWS rows and more a pre-split B; the step's shapes, B a column slice of a
# wider weight (the split runs over the strided span), and the 255-wide heads (a ragged N, and a K padded to 256)
OPS_CASES = [(16384, 512, 1536, True, 0), (15360, 512, 512, False, 0), (16384, 255, 512, True, 0),
             (15360, 512, 255, False, 0), (4096, 384, 256, True, 128), (4096, 200, 300, False, 36)]


@pytest.mark.parametrize("M,N,K,transB,extra", OPS_CASES,
                         ids=[f"M{m}-N{n}-K{k}-{'NT' if t else 'NN'}-pad{e}" for m, n, k, t, e in OPS_CASES])
def test_ops_gemm_presplit_route_matches_raw(cu, precision, M, N, K, transB, extra):
    from sheeprl_b200.lib import PRESPLIT_MIN_ROWS

    assert M >= PRESPLIT_MIN_ROWS
    lda = (K + 3) // 4 * 4
    A = draw((M, lda), 18)[:, :K]
    Bfull = draw((N, K + extra) if transB else (K, N + extra), 19)
    B = Bfull[:, :K] if transB else Bfull[:, :N]
    bias = draw((N,), 20)
    raw, got = torch.empty(M, N, device="cuda"), torch.empty(M, N, device="cuda")
    ck(cu, cu.lib.b200rl_gemm_tc(p(A), p(B), p(raw), p(bias), M, N, K, lda, B.stride(0), N, 0, int(transB), 0, st()))
    cu.gemm(A, B, got, False, transB, bias=bias)
    assert torch.equal(raw, got)


# ------------------------------------------------------------------------------------------------------- gemm_ln tails
def gemm_ln(cu, A, W, planes, gamma, beta, mode, h_prev=None):
    M, K = A.shape
    N = W.shape[0]
    pre, out = torch.empty(M, N, device="cuda"), torch.empty(M, N, device="cuda")
    h = torch.empty(M, N // 3, device="cuda") if mode == 1 else None
    act = 1 if mode == 0 else 0
    tail = (p(gamma), p(beta), EPS, act, p(pre), N, p(out), N, mode, p(h_prev), 0 if h_prev is None else h_prev.stride(0),
            p(h), 0 if h is None else N // 3, None, 0, st())
    if planes is None:
        ck(cu, cu.lib.b200rl_gemm_ln(p(A), p(W), M, N, K, K, K, *tail))
    else:
        assert cu.lib.b200rl_gemm_ln_presplit_supported(p(A), p(planes[0]), p(planes[1]), M, N, K, K, K, mode) == 1
        ck(cu, cu.lib.b200rl_gemm_ln_presplit(p(A), p(planes[0]), p(planes[1]), M, N, K, K, K, *tail))
    return [t for t in (pre, out, h) if t is not None]


@pytest.mark.parametrize("mode,M,N,K", [(0, 1024, 512, 1536), (0, 100, 64, 256), (1, 1024, 1536, 1536), (1, 64, 384, 96)])
def test_gemm_ln_presplit_matches_raw(cu, precision, mode, M, N, K):
    A, W = draw((M, K), 9), draw((N, K), 10)
    gamma, beta = 1.0 + 0.1 * draw((N,), 11), 0.1 * draw((N,), 12)
    h_prev = 0.5 * draw((M, N // 3), 13) if mode == 1 else None
    raw = gemm_ln(cu, A, W, None, gamma, beta, mode, h_prev)
    pre = gemm_ln(cu, A, W, split(cu, W), gamma, beta, mode, h_prev)
    for a, b in zip(raw, pre):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------- convolutions
# the S encoder / decoder layers (h, Cs, Cb); Cb = 32 is the merged four-parity ConvTranspose2d tile (UP4)
CONV_LAYERS = ((16, 64, 32), (8, 128, 64), (4, 256, 128))


@pytest.mark.parametrize("NB", [64, 1024])
@pytest.mark.parametrize("kind", ["down", "up"])
@pytest.mark.parametrize("h,Cs,Cb", CONV_LAYERS, ids=[f"h{h}-Cs{cs}-Cb{cb}" for h, cs, cb in CONV_LAYERS])
def test_conv_presplit_matches_raw(cu, precision, kind, h, Cs, Cb, NB):
    up = int(kind == "up")
    big, small = draw((NB, 2 * h, 2 * h, Cb), 14), draw((NB, h, h, Cs), 15)
    W, bias = 0.05 * draw((Cs, Cb, 4, 4), 16), draw((Cb,), 17)
    assert cu.lib.b200rl_conv_tc_supported(up, NB, h, h, Cs, Cb) == 1
    n = int(cu.lib.b200rl_conv_pack_floats(up, Cs, Cb))
    packed, hi, lo = (torch.empty(n, device="cuda") for _ in range(3))
    ck(cu, cu.lib.b200rl_conv_pack(p(W), p(packed), up, Cs, Cb, st()))
    ck(cu, cu.lib.b200rl_conv_pack_split(p(W), p(hi), p(lo), up, Cs, Cb, st()))
    assert torch.equal(hi + lo, packed)
    out = (torch.empty(NB, h, h, Cs, device="cuda") if kind == "down" else torch.empty(NB, 2 * h, 2 * h, Cb, device="cuda"))
    raw, pre, via_ops = out, torch.empty_like(out), torch.empty_like(out)
    if kind == "down":
        ck(cu, cu.lib.b200rl_conv_down_tc(p(big), p(packed), p(raw), NB, h, h, Cs, Cb, st()))
        ck(cu, cu.lib.b200rl_conv_down_tc_presplit(p(big), p(hi), p(lo), p(pre), NB, h, h, Cs, Cb, st()))
        cu.conv_down(big, W, via_ops)
    else:
        ck(cu, cu.lib.b200rl_conv_up_tc(p(small), p(packed), p(raw), p(bias), NB, h, h, Cs, Cb, st()))
        ck(cu, cu.lib.b200rl_conv_up_tc_presplit(p(small), p(hi), p(lo), p(pre), p(bias), NB, h, h, Cs, Cb, st()))
        cu.conv_up(small, W, via_ops, bias)
    assert torch.equal(raw, pre)
    assert torch.equal(raw, via_ops)
