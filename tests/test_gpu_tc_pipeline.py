"""Exact-equality checks of the tensor-core GEMM's operand pipeline (csrc/gemm_tc.cu), in both matmul precisions.

The operand stages rotate through shared memory across k-blocks and across the tiles of the persistent walk; the B
splitters rewrite a stage's hi / lo halves as soon as the consumers arrive on its `empty` barrier, and the consumers read
their A fragments into registers that in-flight wgmma groups also read.  A hazard there (a stage handed back before the
last group that reads it has retired, a fragment register rewritten under a running group) changes bits without faulting,
so every check here is bitwise:
  - the same output rows computed at different ring phases (more row tiles, a persistent walk) are equal;
  - split-K products, the fused LayerNorm / GRU tails and the convolution modes reproduce themselves run after run;
  - a convolution over the first 64 images of a 1024-image batch equals the same convolution over those 64 alone.
"""
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


def draw(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda")


def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ------------------------------------------------------------------------------------------- ring wrap across tiles
# K = 32, 96, 128, 160: one k-block, fewer k-blocks than stages, exactly one chunk (4 k-blocks), a chunk plus one.  None
# of them is split (split-K needs >= 8 k-blocks).  300 row tiles are more than 2 x 132 tiles, so the grid is persistent
# and each CTA walks several tiles, entering each at a different stage / slot phase.
# K = 4128 (129 k-blocks) is split when there are fewer than 264 tiles, and a split moves the chunk boundaries; its
# reference is therefore the smallest tile count that runs unsplit and one tile per CTA (264 tiles).
SHORT_K = (32, 96, 128, 160)
LONG_K = 4128
ROW_TILES = (2, 5, 300)


def ring_cases():
    for bn, N in ((64, 64), (128, 256)):
        for K in SHORT_K + (LONG_K,):
            yield pytest.param(N, K, id=f"bn{bn}-K{K}")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("N,K", list(ring_cases()))
def test_ring_wrap_across_tiles(cu, precision, N, K):
    ntiles = (N + 127) // 128
    ref_tiles = 1 if K in SHORT_K else 264 // ntiles
    tiles = ROW_TILES if K in SHORT_K else (300,)
    A = draw((128 * max(tiles + (ref_tiles,)), K), 1)
    B = draw((N, K), 2)
    cu.set_matmul_precision(precision)
    try:
        def rows(t):
            C = torch.empty(128 * t, N, device="cuda")
            cu.gemm(A[: 128 * t], B, C, False, True)
            return C

        ref = rows(ref_tiles)
        for t in tiles:
            assert same_bits(rows(t)[: 128 * ref_tiles], ref), f"{t} row tiles differ from {ref_tiles} on the shared rows"
    finally:
        cu.set_matmul_precision("highest")


# ---------------------------------------------------------------------------------- split-K and the fused tails
RUNS = 3


def reproduces(run):
    first = run()
    for _ in range(RUNS - 1):
        again = run()
        for a, b in zip(first, again):
            assert same_bits(a, b), "a rerun is not bit-identical"


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("M,N,K", [(1024, 512, 4096), (1024, 1536, 1024), (64, 3072, 1280), (256, 64, 16384)])
def test_split_k_reproduces(cu, precision, M, N, K):
    A, B = draw((M, K), 3), draw((N, K), 4)
    cu.set_matmul_precision(precision)
    try:
        def run():
            C = torch.empty(M, N, device="cuda")
            cu.gemm(A, B, C, False, True)
            return (C,)

        reproduces(run)
    finally:
        cu.set_matmul_precision("highest")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_gemm_ln_act_reproduces(cu, precision):
    M, N, K = 1024, 512, 1536
    A, W = draw((M, K), 5), draw((N, K), 6)
    gamma, beta = 1.0 + 0.1 * draw((N,), 7), 0.1 * draw((N,), 8)
    assert cu.gemm_ln_supported(A, W, 0)
    cu.set_matmul_precision(precision)
    try:
        def run():
            out, pre = torch.empty(M, N, device="cuda"), torch.empty(M, N, device="cuda")
            cu.gemm_ln_act(A, W, gamma, beta, EPS, 1, out, pre)
            return out, pre

        reproduces(run)
    finally:
        cu.set_matmul_precision("highest")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_gemm_ln_gru_reproduces(cu, precision):
    M, R = 1024, 512
    N, K = 3 * R, R + 1024
    A, W = draw((M, K), 9), draw((N, K), 10)
    gamma, beta = 1.0 + 0.1 * draw((N,), 11), 0.1 * draw((N,), 12)
    h_prev = 0.5 * draw((M, R), 13)
    assert cu.gemm_ln_supported(A, W, 1)
    cu.set_matmul_precision(precision)
    try:
        def run():
            h, pre, ln = (torch.empty(M, n, device="cuda") for n in (R, N, N))
            cu.gemm_ln_gru(A, W, gamma, beta, EPS, h_prev, h, g_pre=pre, g_ln=ln)
            return h, pre, ln

        reproduces(run)
    finally:
        cu.set_matmul_precision("highest")


# ------------------------------------------------------------------------------------------------ convolutions
# the S encoder / decoder layers that run on the tensor cores: (h, Cs, Cb) of small [NB][h][h][Cs] <-> big
# [NB][2h][2h][Cb].  Cb = 32 is the merged four-parity ConvTranspose2d tile (UP4), the others the per-parity one (UP).
# 1024 images make a persistent grid; 64 images do not.
CONV_LAYERS = ((16, 64, 32), (8, 128, 64), (4, 256, 128))


def conv_params():
    for h, Cs, Cb in CONV_LAYERS:
        for kind in ("down", "up", "wgrad"):
            yield pytest.param(kind, h, Cs, Cb, id=f"{kind}-h{h}-Cs{Cs}-Cb{Cb}")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("kind,h,Cs,Cb", list(conv_params()))
def test_conv_modes_reproduce(cu, precision, kind, h, Cs, Cb):
    NB = 1024
    big, small = draw((NB, 2 * h, 2 * h, Cb), 14), draw((NB, h, h, Cs), 15)
    W, bias = 0.05 * draw((Cs, Cb, 4, 4), 16), draw((Cb,), 17)
    if kind == "wgrad":
        assert cu.lib.b200rl_conv_wgrad_mn_supported(NB, h, h, Cs, Cb) == 1
    else:
        assert cu.lib.b200rl_conv_tc_supported(int(kind == "up"), NB, h, h, Cs, Cb) == 1
    cu.set_matmul_precision(precision)
    try:
        def run(nb):
            if kind == "down":
                out = torch.empty(nb, h, h, Cs, device="cuda")
                cu.conv_down(big[:nb], W, out)
            elif kind == "up":
                out = torch.empty(nb, 2 * h, 2 * h, Cb, device="cuda")
                cu.conv_up(small[:nb], W, out, bias)
            else:
                out = torch.empty(Cs, Cb, 4, 4, device="cuda")
                cu.conv_wgrad(small[:nb], big[:nb], out)
            return out

        full = run(NB)
        assert same_bits(run(NB), full), "a rerun is not bit-identical"
        if kind != "wgrad":      # the weight gradient sums over every image, so only the rerun applies to it
            assert same_bits(run(64), full[:64]), "64 images differ from the first 64 of 1024"
    finally:
        cu.set_matmul_precision("highest")
