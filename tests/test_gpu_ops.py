"""Per-kernel parity: every C-ABI op (called through ctypes) against its executable specification
(oracle/ops_emul.py, fp32 torch on CPU) on seeded inputs.  Tolerances are fp32 round-off scaled by the
reduction length; integer / index outputs (samples, gathers) must be bit-exact."""
import numpy as np
import pytest
import torch

from oracle import ln_ref
from oracle.ops_emul import EmulOps
from tests.test_lib_cpu import HEAD_SAMPLE, ONEHOT_LINEAR, WGRAD_TC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from sheeprl_b200.lib import CudaOps

    return CudaOps("cuda"), EmulOps()


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def close(got, want, rtol=1e-5, atol=1e-6, what=""):
    got = got.detach().float().cpu()
    want = want.detach().float().cpu()
    err = (got - want).abs()
    bound = atol + rtol * want.abs().max()
    assert float(err.max()) <= float(bound), (what, float(err.max()), float(bound))


def run_both(ops, name, tensors, *scalars, outputs, **kw):
    """tensors: dict name -> CPU tensor (None allowed). Runs op `name` on both backends with the tensors
    passed positionally in dict order, returns {out_name: (cuda_result, cpu_result)}."""
    cu, em = ops
    cpu = {k: (v.clone() if v is not None else None) for k, v in tensors.items()}
    gpu = {k: (v.clone().cuda() if v is not None else None) for k, v in tensors.items()}
    return cu, em, cpu, gpu


def ln_close(X, gam, bet, eps, act, dY, got, want):
    """LayerNorm kernel vs emulator: |kernel - emulator| <= the sum of both float64 error bounds (oracle/ln_ref.py),
    element by element for y and dX, column by column for dgamma / dbeta.  got / want: (y, dX, dgamma, dbeta).  A
    tolerance relative to the largest entry was marginal: the float64 reference puts the kernel at the once-failed shape
    (tanh, M = 1000, C = 32, eps 1e-5) at 0.28 of its bound and the emulator within half of it."""
    M = X.shape[0]
    y64 = ln_ref.ln_act_fwd64(X, gam, bet, eps, act)[0]
    b_dx, p_g, p_b = ln_ref.ln_act_bwd_bound(X, gam, bet, eps, act, dY)
    mag = ln_ref.ln_act_bwd64(X, gam, bet, eps, act, dY)[3]
    bounds = (ln_ref.ln_act_fwd_bound(X, gam, bet, eps, act, y64), b_dx, ln_ref.param_bound(M, mag["dgamma"], p_g),
              ln_ref.param_bound(M, mag["dbeta"], p_b))
    for name, g_, w_, b_ in zip(("ln fwd", "ln dX", "ln dgamma", "ln dbeta"), got, want, bounds):
        err = (g_.detach().cpu().double() - w_.double()).abs()
        assert bool((err <= 2 * b_).all()), (name, float((err / b_).max()))


GEMM_SHAPES = [
    (16, 512, 1026, False, True), (16, 1536, 1024, False, True), (16, 1024, 512, False, False),
    (1024, 512, 1536, False, True), (1024, 1536, 255, False, False), (255, 512, 1024, True, False),
    (300, 70, 33, False, True), (7, 3, 5, False, True), (5, 1, 129, False, True), (1000, 2, 512, False, True),
    (2, 512, 1000, True, False), (130, 130, 70, True, True), (64, 4096, 200, False, True),
    # tensor-core (wgmma 3xTF32) eligible: NT, M >= 256, N >= 48, 16-byte aligned rows
    (16384, 512, 1536, False, True), (1024, 255, 512, False, True), (15360, 512, 512, False, True),
    (1000, 72, 40, False, True), (257, 129, 36, False, True), (1024, 4096, 1536, False, True),
    # transposed operands are read in place as MN-major tiles: input gradients (NN), weight gradients (TN)
    (16384, 1536, 512, False, False), (1024, 512, 255, False, False), (512, 1536, 16384, True, False),
    (255, 512, 15360, True, False), (4096, 1536, 1024, True, False), (1024, 4608, 512, False, False),
    # MN-major operands with ragged tiles in every dimension (TMA zero fill on both box axes)
    (257, 129, 100, True, False), (300, 200, 68, False, False), (129, 52, 36, True, True), (1024, 1024, 1026, True, False),
    # fewer rows than one 128-row tile (the 64-row products of the per-step scan at the XL width): forward, dX, dW
    (64, 3072, 1280, False, True), (64, 1280, 3072, False, False), (3072, 1280, 64, True, False), (40, 512, 512, False, True),
    # tiny K, many rows, NN (input gradient of a policy head): rank-K kernel
    (15360, 512, 2, False, False), (2048, 64, 7, False, False), (1024, 128, 8, False, False),
]


def test_gemm_tensor_core_path_is_taken_and_exact_enough(ops):
    """The tensor-core path must (a) be selected for the big NT products, (b) keep fp32-level accuracy (3xTF32)."""
    import ctypes

    cu, em = ops
    M, N, K = 2048, 512, 1536
    A, B = rnd(M, K, seed=11), rnd(N, K, seed=12)
    Ag, Bg = A.cuda(), B.cuda()
    assert cu.lib.b200rl_gemm_tc_supported(ctypes.c_void_p(Ag.data_ptr()), ctypes.c_void_p(Bg.data_ptr()), M, N, K, K, K, 0, 1) == 1
    Cg = torch.empty(M, N, device="cuda")
    cu.gemm(Ag, Bg, Cg, False, True)
    ref = (A.double() @ B.double().t())
    err = float((Cg.cpu().double() - ref).abs().max() / ref.abs().max())
    assert err < 3e-6, err          # plain TF32 would give ~1e-3 here
    # view with a 16-byte aligned column offset and a wider leading dimension
    Aw, Bw, Cw = rnd(M, K + 8, seed=13).cuda(), rnd(N, K + 8, seed=14).cuda(), torch.zeros(M, N + 8, device="cuda")
    cu.gemm(Aw[:, 4:4 + K], Bw[:, 4:4 + K], Cw[:, 4:4 + N], False, True)
    ref = Aw[:, 4:4 + K].cpu().double() @ Bw[:, 4:4 + K].cpu().double().t()
    assert float((Cw[:, 4:4 + N].cpu().double() - ref).abs().max() / ref.abs().max()) < 3e-6
    assert float(Cw[:, :4].abs().sum()) == 0 and float(Cw[:, 4 + N:].abs().sum()) == 0


def test_matmul_precision_knob_single_tf32_pass(ops):
    """`float32_matmul_precision: high` (the reference's GPU default, configs/config.yaml:18): one TF32 product per k-step —
    TF32-level error (~1e-3 of the largest entry), clearly distinct from the fp32-accurate default, and switching back
    restores it.  Also covers the split-K path (M = 1024) in both modes."""
    cu, em = ops
    for M, N, K in ((2048, 512, 1536), (1024, 1536, 1024)):
        A, B = rnd(M, K, seed=21), rnd(N, K, seed=22)
        Ag, Bg, Cg = A.cuda(), B.cuda(), torch.empty(M, N, device="cuda")
        ref = A.double() @ B.double().t()
        try:
            cu.set_matmul_precision("high")
            assert cu.matmul_precision() == "high"
            cu.gemm(Ag, Bg, Cg, False, True)
            err_hi = float((Cg.cpu().double() - ref).abs().max() / ref.abs().max())
        finally:
            cu.set_matmul_precision("highest")
        cu.gemm(Ag, Bg, Cg, False, True)
        err = float((Cg.cpu().double() - ref).abs().max() / ref.abs().max())
        assert err < 3e-6 and 2e-5 < err_hi < 5e-3, (M, N, K, err, err_hi)


def test_split_k_products_are_bit_reproducible(ops):
    """split-K partial tiles are summed in split order by the last CTA to arrive (no atomics on C): same bits every launch"""
    cu, em = ops
    M, N, K = 1024, 512, 4096
    A, B = rnd(M, K, seed=31).cuda(), rnd(N, K, seed=32).cuda()
    outs = []
    for _ in range(4):
        C = torch.empty(M, N, device="cuda")
        cu.gemm(A, B, C, False, True)
        outs.append(C.clone())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    # accumulate + bias through the split-K path
    bias = rnd(1, N, seed=33).cuda().reshape(N)
    C0 = rnd(M, N, seed=34).cuda()
    C1 = C0.clone()
    cu.gemm(A, B, C1, False, True, bias=bias, accumulate=True)
    ref = C0.cpu().double() + A.cpu().double() @ B.cpu().double().t() + bias.cpu().double()
    assert float((C1.cpu().double() - ref).abs().max() / ref.abs().max()) < 3e-6


@pytest.mark.parametrize("rows", [1024, 15360])
def test_gemm_twohot_gradient_operands_with_padded_rows(ops, rows):
    """the 255-bin logit gradients live in buffers with a 256-float row stride so that dX = dlogits W (K = 255) and
    dW = dlogits^T act (M = 255, MN-major A) are tensor-core eligible (16-byte TMA row stride, ragged last box)"""
    cu, em = ops
    nb, D = 255, 512
    dl_w = rnd(rows, 256, seed=1)
    dl_w[:, 255] = 1e6                                           # the pad column must never be read as data
    W, act = rnd(nb, D, seed=2), rnd(rows, D, seed=3)
    dl_g, Wg, actg = dl_w.cuda(), W.cuda(), act.cuda()
    import ctypes

    assert cu.lib.b200rl_gemm_tc_supported(ctypes.c_void_p(dl_g.data_ptr()), ctypes.c_void_p(Wg.data_ptr()), rows, D, nb,
                                           256, D, 0, 0) == 1
    dx_w, dx_g = torch.empty(rows, D), torch.empty(rows, D, device="cuda")
    em.gemm(dl_w[:, :nb], W, dx_w, False, False)
    cu.gemm(dl_g[:, :nb], Wg, dx_g, False, False)
    close(dx_g, dx_w, rtol=2e-6 * nb ** 0.5, what="dX")
    dw_w, dw_g = torch.empty(nb, D), torch.empty(nb, D, device="cuda")
    em.gemm(dl_w[:, :nb], act, dw_w, True, False)
    cu.gemm(dl_g[:, :nb], actg, dw_g, True, False)
    close(dw_g, dw_w, rtol=2e-6 * rows ** 0.5, what="dW")


@pytest.mark.parametrize("M,N,K,tA,tB", GEMM_SHAPES)
@pytest.mark.parametrize("mode", ["plain", "bias", "acc", "strided"])
def test_gemm(ops, M, N, K, tA, tB, mode):
    cu, em = ops
    A = rnd(*((K, M) if tA else (M, K)), seed=1)
    B = rnd(*((N, K) if tB else (K, N)), seed=2)
    C0 = rnd(M, N, seed=3)
    bias = rnd(N, seed=4) if mode == "bias" else None
    acc = mode == "acc"
    if mode == "strided":
        # operands are column slices of wider buffers (leading dimension > width)
        Aw = rnd(A.shape[0], A.shape[1] + 5, seed=5)
        Bw = rnd(B.shape[0], B.shape[1] + 3, seed=6)
        Cw = rnd(M, N + 7, seed=7)
        Ac, Bc, Cc = Aw[:, 2:2 + A.shape[1]], Bw[:, 1:1 + B.shape[1]], Cw.clone()[:, 4:4 + N]
        Awg, Bwg, Cwg = Aw.cuda(), Bw.cuda(), Cw.cuda()
        Ag, Bg, Cg = Awg[:, 2:2 + A.shape[1]], Bwg[:, 1:1 + B.shape[1]], Cwg[:, 4:4 + N]
        em.gemm(Ac, Bc, Cc, tA, tB)
        cu.gemm(Ag, Bg, Cg, tA, tB)
        close(Cg, Cc, rtol=2e-6 * max(K, 8) ** 0.5, what="gemm strided")
        assert torch.equal(Cwg[:, :4].cpu(), Cw[:, :4]) and torch.equal(Cwg[:, 4 + N:].cpu(), Cw[:, 4 + N:])
        return
    Cc, Cg = C0.clone(), C0.clone().cuda()
    em.gemm(A, B, Cc, tA, tB, bias=bias, accumulate=acc)
    cu.gemm(A.cuda(), B.cuda(), Cg, tA, tB, bias=None if bias is None else bias.cuda(), accumulate=acc)
    close(Cg, Cc, rtol=2e-6 * max(K, 8) ** 0.5, what="gemm")


@pytest.mark.parametrize("M,C", [(1024, 512), (1000, 32), (16, 1536), (37, 72), (5, 4), (4096, 255), (64, 3),
                                 # widths of the M / L / XL models (register-resident rows) and the XL GRU's 3 x 4096
                                 # joint LayerNorm (one CTA per row)
                                 (1000, 96), (500, 192), (300, 384), (100, 768), (64, 640), (128, 48), (64, 12288),
                                 (300, 3072), (3, 16384)])
@pytest.mark.parametrize("act", [0, 1])
def test_ln_act(ops, M, C, act):
    cu, em = ops
    X, gam, bet, dY = rnd(M, C, seed=1, scale=2.0), rnd(C, seed=2) + 1.0, rnd(C, seed=3), rnd(M, C, seed=4)
    Yc = torch.empty(M, C)
    Yg = torch.empty(M, C, device="cuda")
    em.ln_act_fwd(X, gam, bet, 1e-3, act, Yc)
    cu.ln_act_fwd(X.cuda(), gam.cuda(), bet.cuda(), 1e-3, act, Yg)
    dXc, dgc, dbc = torch.empty(M, C), torch.empty(C), torch.empty(C)
    dXg, dgg, dbg = torch.empty(M, C, device="cuda"), torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    em.ln_act_bwd(X, gam, bet, 1e-3, act, dY, dXc, dgc, dbc)
    cu.ln_act_bwd(X.cuda(), gam.cuda(), bet.cuda(), 1e-3, act, dY.cuda(), dXg, dgg, dbg)
    ln_close(X, gam, bet, 1e-3, act, dY, (Yg, dXg, dgg, dbg), (Yc, dXc, dgc, dbc))
    # in-place (dX aliases dY), no parameter grads
    dYg = dY.cuda()
    cu.ln_act_bwd(X.cuda(), gam.cuda(), bet.cuda(), 1e-3, act, dYg, dYg, None, None)
    ln_close(X, gam, bet, 1e-3, act, dY, (Yg, dYg, dgg, dbg), (Yc, dXc, dgc, dbc))


@pytest.mark.parametrize("M,C", [(1000, 32), (37, 72), (64, 64), (16, 1536), (256, 24)])
@pytest.mark.parametrize("act", [2, 3])
def test_ln_act_tanh_relu(ops, M, C, act):
    """LayerNorm + tanh / ReLU (PPO MLPs with layer_norm=True, eps 1e-5).  ReLU'(0) is a jump: the inputs are re-drawn
    until no LayerNorm output sits within 1e-5 of it, so a 1-ulp difference cannot flip a mask bit."""
    cu, em = ops
    for seed in range(1, 40):
        X, gam, bet, dY = rnd(M, C, seed=seed, scale=2.0), rnd(C, seed=seed + 100) + 1.0, rnd(C, seed=seed + 200), rnd(M, C, seed=seed + 300)
        ln = torch.nn.functional.layer_norm(X, (C,), gam, bet, 1e-5)
        if act != 3 or float(ln.abs().min()) > 1e-5:
            break
    Yc, Yg = torch.empty(M, C), torch.empty(M, C, device="cuda")
    em.ln_act_fwd(X, gam, bet, 1e-5, act, Yc)
    cu.ln_act_fwd(X.cuda(), gam.cuda(), bet.cuda(), 1e-5, act, Yg)
    dXc, dgc, dbc = torch.empty(M, C), torch.empty(C), torch.empty(C)
    dXg, dgg, dbg = torch.empty(M, C, device="cuda"), torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    em.ln_act_bwd(X, gam, bet, 1e-5, act, dY, dXc, dgc, dbc)
    cu.ln_act_bwd(X.cuda(), gam.cuda(), bet.cuda(), 1e-5, act, dY.cuda(), dXg, dgg, dbg)
    ln_close(X, gam, bet, 1e-5, act, dY, (Yg, dXg, dgg, dbg), (Yc, dXc, dgc, dbc))


@pytest.mark.parametrize("M,C", [(1024, 255), (1048576 // 64, 3), (17, 4096), (3, 1),
                                 # narrow contiguous matrices take the flat float4 kernel (tail of 2 elements in the second)
                                 (262144, 3), (21846, 3), (100000, 7), (70000, 32), (65536, 1)])
def test_col_sum(ops, M, C):
    cu, em = ops
    X = rnd(M, C, seed=1)
    oc, og = torch.zeros(C), torch.full((C,), 5.0, device="cuda")
    em.col_sum(X, oc)
    cu.col_sum(X.cuda(), og)
    close(og, oc, rtol=1e-5 * max(M, 16) ** 0.5, what="col_sum")


CONV_SHAPES = [(3, 8, 8, 16, 8), (2, 4, 4, 32, 16), (5, 16, 16, 4, 3), (2, 32, 32, 32, 3), (3, 2, 2, 40, 24),
               (2, 4, 4, 130, 72), (1, 8, 8, 8, 2),
               # thin big-image side (conv_thin.cu): partial / multiple 32-pixel row tiles, every channel-group count
               (3, 16, 16, 64, 3), (2, 40, 40, 96, 3), (1, 32, 32, 48, 3), (2, 8, 8, 32, 1), (2, 8, 8, 64, 4),
               # 32-wide small grids take the packed-FMA kernels: odd / non-multiple-of-8 heights, every channel count
               (3, 32, 32, 64, 3), (2, 32, 32, 96, 3), (2, 5, 32, 32, 3), (1, 12, 32, 64, 3), (5, 1, 32, 96, 3),
               # tensor-core implicit-GEMM eligible (gathered image has a multiple of 32 channels, grid tiles by 128 px)
               (8, 4, 4, 64, 32), (2, 32, 32, 32, 64), (4, 16, 16, 128, 64), (16, 8, 8, 256, 128), (24, 4, 4, 96, 32),
               # weight gradient with operands read in place (MN-major tiles): k-block = part of a row / rows / images
               (64, 4, 4, 256, 128), (2, 32, 32, 64, 32), (1, 64, 64, 48, 32), (32, 8, 8, 128, 64)]


@pytest.mark.parametrize("NB,h,w,Cs,Cb", CONV_SHAPES)
def test_conv_down_up_wgrad(ops, NB, h, w, Cs, Cb):
    cu, em = ops
    big, small = rnd(NB, 2 * h, 2 * w, Cb, seed=1), rnd(NB, h, w, Cs, seed=2)
    W, bias = rnd(Cs, Cb, 4, 4, seed=3, scale=0.2), rnd(Cb, seed=4)
    oc, og = torch.empty_like(small), torch.empty_like(small).cuda()
    em.conv_down(big, W, oc)
    cu.conv_down(big.cuda(), W.cuda(), og)
    close(og, oc, rtol=3e-6 * (16 * Cb) ** 0.5, what="conv_down")
    for b in (None, bias):
        oc, og = torch.empty_like(big), torch.empty_like(big).cuda()
        em.conv_up(small, W, oc, b)
        cu.conv_up(small.cuda(), W.cuda(), og, None if b is None else b.cuda())
        close(og, oc, rtol=3e-6 * (4 * Cs) ** 0.5, what="conv_up")
    oc, og = torch.empty_like(W), torch.full_like(W, 3.0).cuda()
    em.conv_wgrad(small, big, oc)
    cu.conv_wgrad(small.cuda(), big.cuda(), og)
    close(og, oc, rtol=3e-6 * (NB * h * w) ** 0.5, what="conv_wgrad")


def test_obs_prep_and_transpose(ops):
    cu, em = ops
    g = torch.Generator().manual_seed(0)
    # (6,3,16,16) / (2,12,84,84) / (3,1,8,8) / (2,4,20,20): the 4-pixel kernel; (2,5,6,6), (3,3,5,5): the generic one
    for shape in ((6, 3, 16, 16), (2, 12, 84, 84), (3, 1, 8, 8), (2, 4, 20, 20), (2, 5, 6, 6), (3, 3, 5, 5)):
        obs = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
        NB, C, H, W = shape
        for o in (obs, obs.float()):
            oc, og = torch.empty(NB, H, W, C), torch.empty(NB, H, W, C, device="cuda")
            em.obs_prep(o, oc)
            cu.obs_prep(o.cuda(), og)
            assert torch.equal(og.cpu(), oc), shape
    X = rnd(7, 16, 40, seed=1)
    Yc, Yg = torch.empty(7, 40, 16), torch.empty(7, 40, 16, device="cuda")
    em.transpose_batched(X, Yc)
    cu.transpose_batched(X.cuda(), Yg)
    assert torch.equal(Yg.cpu(), Yc)


def test_symlog_into_column_slices(ops):
    """vector observations are squashed straight into their column range of the encoder-input buffer"""
    cu, em = ops
    x = rnd(37, 5, seed=1, scale=30.0)
    x[0, :3] = torch.tensor([0.0, -0.0, 1e-9])
    wide_c, wide_g = torch.full((37, 11), 7.0), torch.full((37, 11), 7.0, device="cuda")
    em.symlog(x, wide_c[:, 4:9])
    cu.symlog(x.cuda(), wide_g[:, 4:9])
    close(wide_g, wide_c, rtol=1e-6, atol=1e-7, what="symlog")
    src_w = rnd(37, 9, seed=2, scale=5.0)                       # strided source as well
    em.symlog(src_w[:, 2:7], wide_c[:, 0:5])
    cu.symlog(src_w.cuda()[:, 2:7], wide_g[:, 0:5])
    close(wide_g, wide_c, rtol=1e-6, atol=1e-7, what="symlog strided")


@pytest.mark.parametrize("M,R", [(16, 512), (1024, 24), (3, 7)])
def test_gru_gate(ops, M, R):
    cu, em = ops
    G, Hin, dH = rnd(M, 3 * R, seed=1), rnd(M, R, seed=2), rnd(M, R, seed=3)
    oc, og = torch.empty(M, R), torch.empty(M, R, device="cuda")
    em.gru_gate_fwd(G, Hin, oc)
    cu.gru_gate_fwd(G.cuda(), Hin.cuda(), og)
    close(og, oc, what="gru fwd")
    dGc, dHc = torch.empty(M, 3 * R), torch.empty(M, R)
    dGg, dHg = torch.empty(M, 3 * R, device="cuda"), torch.empty(M, R, device="cuda")
    em.gru_gate_bwd(G, Hin, dH, dGc, dHc)
    cu.gru_gate_bwd(G.cuda(), Hin.cuda(), dH.cuda(), dGg, dHg)
    close(dGg, dGc, what="gru dG")
    close(dHg, dHc, what="gru dHin")


def test_masks(ops):
    cu, em = ops
    M, C = 16, 100
    prev, init, dIn = rnd(M, C, seed=1), rnd(1, C, seed=2), rnd(M, C, seed=3)
    first = (torch.rand(M, generator=torch.Generator().manual_seed(4)) < 0.3).float()
    oc, og = torch.empty(M, C), torch.empty(M, C, device="cuda")
    em.mask_mix(prev, init, first, oc)
    cu.mask_mix(prev.cuda(), init.cuda(), first.cuda(), og)
    close(og, oc, what="mask_mix")
    em.mask_rows(prev, first, oc)
    cu.mask_rows(prev.cuda(), first.cuda(), og)
    close(og, oc, what="mask_rows")
    dpc, dic = torch.empty(M, C), torch.ones(C)
    dpg, dig = torch.empty(M, C, device="cuda"), torch.ones(C, device="cuda")
    em.mask_bwd(dIn, first, dpc, dic)
    cu.mask_bwd(dIn.cuda(), first.cuda(), dpg, dig)
    close(dpg, dpc, what="mask_bwd prev")
    close(dig, dic, what="mask_bwd init")


@pytest.mark.parametrize("M,S,D", [(16, 32, 32), (1024, 32, 32), (9, 6, 5), (33, 1, 2), (12, 1, 18), (5, 4, 40)])
@pytest.mark.parametrize("unimix", [0.01, 0.0])
def test_cat_sample_fwd_bwd(ops, M, S, D, unimix):
    cu, em = ops
    raw = rnd(M, S * D, seed=1, scale=2.0)
    q = torch.empty(M, S * D).exponential_(1.0, generator=torch.Generator().manual_seed(2))
    for noise in (q, None):
        hc, mc = torch.empty(M, S * D), torch.empty(M, S * D)
        hg, mg = torch.empty(M, S * D, device="cuda"), torch.empty(M, S * D, device="cuda")
        em.cat_sample(raw, noise, unimix, S, D, hc, mc)
        cu.cat_sample(raw.cuda(), None if noise is None else noise.cuda(), unimix, S, D, hg, mg)
        close(mg, mc, rtol=2e-6, atol=2e-6, what="unimix logits")
        mism = (hg.cpu() != hc).reshape(M * S, D).any(-1).float().mean()
        assert float(mism) <= 1e-3, float(mism)  # only exact near-ties of p/q may differ
    dz, dmix = rnd(M, S * D, seed=3), rnd(M, S * D, seed=4)
    for a, b in ((dz, dmix), (dz, None), (None, dmix)):
        oc, og = torch.empty(M, S * D), torch.empty(M, S * D, device="cuda")
        em.cat_sample_bwd(raw, a, b, unimix, S, D, oc)
        cu.cat_sample_bwd(raw.cuda(), None if a is None else a.cuda(), None if b is None else b.cuda(), unimix, S, D, og)
        close(og, oc, rtol=1e-5, what="cat_sample_bwd")


@pytest.mark.parametrize("M,S,D,free", [(1024, 32, 32, 1.0), (64, 6, 5, 0.05), (16, 4, 8, 100.0)])
def test_kl_loss_grad(ops, M, S, D, free):
    cu, em = ops
    post = torch.log_softmax(rnd(M, S, D, seed=1), -1).reshape(M, -1) + 0.01
    prior = torch.log_softmax(rnd(M, S, D, seed=2), -1).reshape(M, -1)
    outs_c = [torch.empty(M, S * D), torch.empty(M, S * D), torch.empty(M, 4)]
    outs_g = [t.cuda() for t in outs_c]
    em.kl_loss_grad(post, prior, S, D, 0.5, 0.1, free, 1.0, 1.0 / M, *outs_c)
    cu.kl_loss_grad(post.cuda(), prior.cuda(), S, D, 0.5, 0.1, free, 1.0, 1.0 / M, *outs_g)
    for g, c, n in zip(outs_g, outs_c, ("d_post", "d_prior", "rows")):
        close(g, c, rtol=2e-5, what=n)


def test_losses(ops):
    cu, em = ops
    M, P, nb = 96, 12288, 255
    pred, tgt = rnd(M, P, seed=1), rnd(M, P, seed=2)
    lc, gc = torch.empty(M), torch.empty(M, P)
    lg, pg = torch.empty(M, device="cuda"), pred.cuda()
    em.mse_loss_grad(pred, tgt, 1.0 / M, lc, gc)
    cu.mse_loss_grad(pg, tgt.cuda(), 1.0 / M, lg, pg)  # in place
    close(lg, lc, rtol=1e-5, what="mse loss")
    close(pg, gc, what="mse grad")
    logits = rnd(M, nb, seed=3, scale=2.0)
    x = torch.cat((rnd(M - 6, seed=4, scale=30.0), torch.tensor([0.0, 1e9, -1e9, 20.0, -20.0, 0.157])))
    w = torch.rand(M, generator=torch.Generator().manual_seed(5))
    for weight in (None, w):
        lc, dc = torch.zeros(M), torch.zeros(M, nb)
        lg, dg = torch.zeros(M, device="cuda"), torch.zeros(M, nb, device="cuda")
        for accumulate in (False, True):
            em.twohot_loss_grad(logits, x, weight, 1.0 / M, -20.0, 20.0, lc, dc, accumulate)
            cu.twohot_loss_grad(logits.cuda(), x.cuda(), None if weight is None else weight.cuda(), 1.0 / M, -20.0,
                                20.0, lg, dg, accumulate)
        close(lg, lc, rtol=1e-5, what="twohot loss")
        close(dg, dc, rtol=1e-5, what="twohot grad")
    oc, og = torch.empty(M), torch.empty(M, device="cuda")
    em.twohot_mean(logits, -20.0, 20.0, oc)
    cu.twohot_mean(logits.cuda(), -20.0, 20.0, og)
    close(og, oc, rtol=2e-5, what="twohot mean")
    lo, y = rnd(M, seed=6, scale=3.0), (torch.rand(M, generator=torch.Generator().manual_seed(7)) < 0.9).float()
    lc, dc, lg, dg = torch.empty(M), torch.empty(M), torch.empty(M, device="cuda"), torch.empty(M, device="cuda")
    em.bce_loss_grad(lo, y, 1.0, 1.0 / M, lc, dc)
    cu.bce_loss_grad(lo.cuda(), y.cuda(), 1.0, 1.0 / M, lg, dg)
    close(lg, lc, what="bce loss")
    close(dg, dc, what="bce grad")


def test_lambda_returns_and_moments(ops):
    cu, em = ops
    H, N = 15, 1024
    rew, val, cl = rnd(H + 1, N, seed=1), rnd(H + 1, N, seed=2), rnd(H + 1, N, seed=3, scale=2.0)
    tc = (torch.rand(N, generator=torch.Generator().manual_seed(4)) < 0.95).float()
    lc, dc = torch.empty(H, N), torch.empty(H + 1, N)
    lg, dg = torch.empty(H, N, device="cuda"), torch.empty(H + 1, N, device="cuda")
    em.lambda_returns(rew, val, cl, tc, 0.997, 0.95, lc, dc)
    cu.lambda_returns(rew.cuda(), val.cuda(), cl.cuda(), tc.cuda(), 0.997, 0.95, lg, dg)
    close(lg, lc, rtol=1e-5, what="lambda")
    close(dg, dc, rtol=1e-5, what="discount")
    for n in (15360, 7, 1, 122880):
        x = rnd(n, seed=5)
        sc, oc = torch.tensor([0.1, 0.7]), torch.empty(2)
        sg, og = sc.clone().cuda(), torch.empty(2, device="cuda")
        em.moments_update(x, sc, 0.99, 1.0, 0.05, 0.95, oc)
        cu.moments_update(x.cuda(), sg, 0.99, 1.0, 0.05, 0.95, og)
        close(sg, sc, rtol=1e-6, what="moments state")
        close(og, oc, rtol=1e-6, what="moments out")
    # exact order statistics (quantile with weight 0): compare against sort
    x = rnd(1001, seed=6)
    sg, og = torch.zeros(2, device="cuda"), torch.empty(2, device="cuda")
    cu.moments_update(x.cuda(), sg, 0.0, 1e8, 0.25, 0.75, og)
    srt = x.sort().values
    assert float(sg[0]) == float(srt[250]) and float(sg[1]) == float(srt[750])


@pytest.mark.parametrize("heads", [(2,), (3, 2), (18,), (4, 4, 4)])
def test_actor_loss_grad(ops, heads):
    cu, em = ops
    M, A = 960, sum(heads)
    raw = rnd(M, A, seed=1, scale=1.5)
    g = torch.Generator().manual_seed(2)
    acts = torch.cat([torch.nn.functional.one_hot(torch.randint(0, h, (M,), generator=g), h).float() for h in heads], -1)
    lam, val, disc = rnd(M, seed=3), rnd(M, seed=4), torch.rand(M, generator=g)
    mom = torch.tensor([0.05, 1.3])
    rc, dc = torch.empty(M), torch.empty(M, A)
    rg, dg = torch.empty(M, device="cuda"), torch.empty(M, A, device="cuda")
    em.actor_loss_grad(raw, acts, lam, val, disc, mom, heads, 0.01, 3e-4, 1.0 / M, rc, dc)
    cu.actor_loss_grad(raw.cuda(), acts.cuda(), lam.cuda(), val.cuda(), disc.cuda(), mom.cuda(), heads, 0.01, 3e-4,
                       1.0 / M, rg, dg)
    close(rg, rc, rtol=1e-5, what="actor rows")
    close(dg, dc, rtol=1e-5, what="actor draw")


def test_optimizer_and_utils(ops):
    """the noise fills, the step counter and the small utilities; clip + Adam, the EMA and sumsq are held to a float64
    reference in tests/test_gpu_optim_precision.py"""
    cu, em = ops
    e = torch.empty(1 << 20, device="cuda")
    cu.fill_exponential(e, 1234, 7)
    assert float(e.min()) > 0 and abs(float(e.mean()) - 1.0) < 0.01 and abs(float(e.var()) - 1.0) < 0.03
    e2 = torch.empty(1 << 20, device="cuda")
    cu.fill_exponential(e2, 1234, 8)
    assert not torch.equal(e, e2)
    ctr = torch.ones(1, dtype=torch.int32, device="cuda")
    cu.fill_exponential(e2, 1234, 7, ctr)
    assert not torch.equal(e, e2)
    ctr.zero_()
    cu.fill_exponential(e2, 1234, 7, ctr)
    assert torch.equal(e, e2)
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    cu.increment(st), cu.increment(st)
    assert int(st) == 2
    x = rnd(33, 20, seed=5)
    big = torch.zeros(33, 50, device="cuda")
    cu.copy(x.cuda(), big[:, 7:27])
    assert torch.equal(big[:, 7:27].cpu(), x) and float(big[:, :7].abs().sum()) == 0
    y = rnd(100, seed=6).cuda()
    y0 = y.clone()
    cu.axpy(y0, y, 0.5)
    close(y, y0.cpu() * 1.5, what="axpy")
    cu.affine(y0, y, -1.0, 1.0)
    close(y, 1 - y0.cpu(), what="affine")
    cu.tanh_fwd(y0, y)
    close(y, torch.tanh(y0.cpu()), what="tanh")
    d = torch.zeros(100, device="cuda")
    cu.tanh_bwd(y, y0, d)
    close(d, y0.cpu() * (1 - torch.tanh(y0.cpu()) ** 2), what="tanh bwd")
    o = torch.empty(2, device="cuda")
    X = rnd(500, 4, seed=7)
    cu.sum_rows(X.cuda()[:, 1:3], o, 0.5)
    close(o, 0.5 * X[:, 1:3].sum(0), rtol=1e-5, what="sum_rows")
    cu.weighted_mean(X.cuda()[:, 0].contiguous(), X.cuda()[:, 1].contiguous(), 0.1, o[:1])
    close(o[:1], 0.1 * (X[:, 0] * X[:, 1]).sum().reshape(1), rtol=1e-5, what="weighted_mean")


def test_replay_gather_scatter_and_gae(ops):
    cu, em = ops
    rng = np.random.default_rng(0)
    size, row = 500, (3, 8, 8)
    storage = torch.from_numpy(rng.integers(0, 256, size=(size, *row), dtype=np.uint8)).cuda()
    S, B, T = 2, 4, 16
    idx = torch.from_numpy(rng.integers(0, size, size=(S * B * T,))).cuda()
    out = torch.empty(S, T, B, *row, dtype=torch.uint8, device="cuda")
    cu.replay_gather(storage, idx, out, S, B, T)
    want = storage.cpu()[idx.cpu()].reshape(S, B, T, *row).swapaxes(1, 2)
    assert torch.equal(out.cpu(), want)
    fs = torch.from_numpy(rng.standard_normal((size, 5)).astype(np.float32)).cuda()  # 20-byte rows (unaligned path)
    outf = torch.empty(S, T, B, 5, device="cuda")
    cu.replay_gather(fs, idx, outf, S, B, T)
    assert torch.equal(outf.cpu(), fs.cpu()[idx.cpu()].reshape(S, B, T, 5).swapaxes(1, 2))
    rows = torch.tensor([3, 499, 0], device="cuda")
    src = torch.from_numpy(rng.integers(0, 256, size=(3, *row), dtype=np.uint8)).cuda()
    cu.replay_scatter(src, rows, storage)
    assert torch.equal(storage[rows].cpu(), src.cpu())
    Tn, E = 128, 16
    r, v, nv = rnd(Tn, E, 1, seed=1), rnd(Tn, E, 1, seed=2), rnd(E, 1, seed=3)
    d = (torch.rand(Tn, E, 1, generator=torch.Generator().manual_seed(4)) < 0.05).float()
    ret, adv = torch.empty(Tn, E, 1, device="cuda"), torch.empty(Tn, E, 1, device="cuda")
    cu.gae(r.cuda(), v.cuda(), d.cuda(), nv.cuda(), 0.99, 0.95, ret, adv)
    from oracle.ppo_oracle import gae_oracle

    ret_c, adv_c = gae_oracle(r, v, d, nv, Tn, 0.99, 0.95)
    close(adv, adv_c, rtol=1e-5, what="gae adv")
    close(ret, ret_c, rtol=1e-5, what="gae ret")


@pytest.mark.parametrize("M,S,D,A,N", [(1024, 32, 32, 2, 512), (7, 6, 5, 5, 24), (33, 4, 40, 1, 130)])
def test_onehot_linear_and_transpose2d(ops, M, S, D, A, N):
    cu, em = ops
    g = torch.Generator().manual_seed(3)
    z = torch.nn.functional.one_hot(torch.randint(0, D, (M, S), generator=g), D).float().reshape(M, S * D)
    buf = torch.zeros(M, S * D + 7)                          # z lives inside a wider row, as in traj[:, :Z]
    buf[:, : S * D] = z
    act, W = rnd(M, A, seed=1), rnd(N, S * D + A, seed=2, scale=0.1)
    WTc, WTg = torch.empty(S * D + A, N), torch.empty(S * D + A, N, device="cuda")
    em.transpose2d(W, WTc)
    cu.transpose2d(W.cuda(), WTg)
    assert torch.equal(WTg.cpu(), WTc)
    oc, og = torch.empty(M, N), torch.empty(M, N, device="cuda")
    em.onehot_linear(buf[:, : S * D], act, WTc, oc, S, D)
    cu.onehot_linear(buf.cuda()[:, : S * D], act.cuda(), WTg, og, S, D)
    close(og, oc, rtol=1e-5, what="onehot_linear")


def test_continuous_action_kernels(ops):
    """csrc/dv3_cont.cu against the torch test double: scaled_normal sampling fwd/bwd, lambda-return backward,
    two-hot mean backward."""
    cu, em = ops
    M, A, H, N, nb = 300, 5, 4, 75, 31
    head, eps = rnd(M, 2 * A, seed=1) * 2, rnd(M, A, seed=2) * 1.5           # some |a| > clip
    args = (0.1, 1.0, 2.0, 1.0)
    ac, ec = torch.zeros(M, A + 3)[:, 3:], torch.zeros(M)
    ag, eg = torch.zeros(M, A + 3, device="cuda")[:, 3:], torch.zeros(M, device="cuda")
    em.cont_action_fwd(head, eps, ac, ec, *args)
    cu.cont_action_fwd(head.cuda(), eps.cuda(), ag, eg, *args)
    close(ag, ac, rtol=1e-5, what="cont action"), close(eg, ec, rtol=1e-5, what="cont entropy")
    dact, disc = rnd(M, A, seed=3), torch.rand(M)
    dc, dg = torch.zeros(M, 2 * A), torch.zeros(M, 2 * A, device="cuda")
    em.cont_action_bwd(head, eps, dact, disc, dc, *args, -0.01)
    cu.cont_action_bwd(head.cuda(), eps.cuda(), dact.cuda(), disc.cuda(), dg, *args, -0.01)
    close(dg, dc, rtol=1e-5, atol=1e-6, what="cont dhead")
    cont_logit, D = rnd(H + 1, N, seed=4), torch.rand(H + 1, N)
    mom, lam, val, ent = torch.tensor([0.2, 1.7]), rnd(H, N, seed=5), rnd(H + 1, N, seed=6), rnd((H + 1) * N, seed=7)
    outs_c = [torch.zeros(H + 1, N), torch.zeros(H + 1, N), torch.zeros(H, N)]
    outs_g = [t.cuda() for t in outs_c]
    em.lambda_returns_bwd(cont_logit, D, mom, lam, val, ent, 0.997, 0.95, 3e-4, 1.0 / (H * N), *outs_c)
    cu.lambda_returns_bwd(cont_logit.cuda(), D.cuda(), mom.cuda(), lam.cuda(), val.cuda(), ent.cuda(), 0.997, 0.95, 3e-4,
                          1.0 / (H * N), *outs_g)
    for g_, c_, nme in zip(outs_g, outs_c, ("d_val", "d_rew", "rows")):
        close(g_, c_, rtol=1e-5, atol=1e-7, what=nme)
    logits, dm = rnd(M, nb, seed=8) * 3, rnd(M, seed=9)
    lc, lg = torch.zeros(M, nb), torch.zeros(M, nb, device="cuda")
    em.twohot_mean_bwd(logits, dm, -20.0, 20.0, lc)
    cu.twohot_mean_bwd(logits.cuda(), dm.cuda(), -20.0, 20.0, lg)
    close(lg, lc, rtol=2e-5, atol=1e-6, what="twohot mean bwd")
    # and the emulated backward really is the derivative of the forward (autograd check of the specification)
    lt = logits.clone().requires_grad_(True)
    bins = torch.linspace(-20, 20, nb)
    m = (torch.softmax(lt, -1) * bins).sum(-1)
    (torch.sign(m) * (torch.exp(m.abs()) - 1) * dm).sum().backward()
    close(lc, lt.grad, rtol=1e-4, atol=1e-6, what="twohot mean bwd vs autograd")


def test_twohot_kernel_reproduces_the_reference_known_answers(ops):
    """tests/test_utils/test_two_hot_encoder.py:6-88 (2.3 -> {0.7 @ 7, 0.3 @ 8}, 21 buckets, saturation, integers,
    corners) through b200rl_twohot_loss_grad; see tests/test_twohot_kat_cpu.py"""
    from tests.test_twohot_kat_cpu import check, twohot_targets

    check(twohot_targets(ops[0], device="cuda"))


# ---- fused imagination ops: each must equal the composition of the ops it replaces (oracle/ops_emul.py) ---------------------
@pytest.mark.parametrize("M,N,K,act,keep", [(1024, 512, 512, 1, True), (1024, 512, 1536, 1, False), (1024, 1024, 1024, 1, True),
                                            (64, 512, 512, 0, True), (200, 100, 68, 1, True), (4096, 1536, 512, 0, False)])
def test_gemm_ln_act_equals_gemm_then_layernorm(ops, M, N, K, act, keep):
    cu, em = ops
    X, W = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    gamma, beta = 1 + 0.1 * rnd(N, seed=3), 0.1 * rnd(N, seed=4)
    pre_c, out_c = torch.empty(M, N), torch.empty(M, N)
    em.gemm(X, W, pre_c, False, True)
    em.ln_act_fwd(pre_c, gamma, beta, 1e-3, act, out_c)
    Xg, Wg = X.cuda(), W.cuda()
    assert cu.gemm_ln_supported(Xg, Wg)
    wide = torch.zeros(M, N + 8, device="cuda")                # outputs inside wider rows
    out_g, pre_g = wide[:, :N], (torch.empty(M, N, device="cuda") if keep else None)
    cu.gemm_ln_act(Xg, Wg, gamma.cuda(), beta.cuda(), 1e-3, act, out_g, pre_g)
    close(out_g, out_c, rtol=2e-5, atol=2e-6, what="gemm_ln_act")
    if keep:
        close(pre_g, pre_c, rtol=2e-5, what="gemm_ln_act pre")
    assert float(wide[:, N:].abs().max()) == 0.0
    # bit-reproducible: fixed-order partial sums
    out2 = torch.empty(M, N, device="cuda")
    cu.gemm_ln_act(Xg, Wg, gamma.cuda(), beta.cuda(), 1e-3, act, out2, None)
    assert torch.equal(out2, out_g)


@pytest.mark.parametrize("M,R,Kx", [(1024, 512, 512), (1024, 128, 64), (64, 512, 1024), (4096, 384, 384)])
def test_gemm_ln_gru_equals_unfused_cell(ops, M, R, Kx):
    cu, em = ops
    hx = rnd(M, R + Kx, seed=1)
    W = rnd(3 * R, R + Kx, seed=2, scale=(R + Kx) ** -0.5)
    gamma, beta = 1 + 0.1 * rnd(3 * R, seed=3), 0.1 * rnd(3 * R, seed=4)
    h_prev = hx[:, :R].clone()
    g_pre, g_ln, h_c = torch.empty(M, 3 * R), torch.empty(M, 3 * R), torch.empty(M, R)
    em.gemm(hx, W, g_pre, False, True)
    em.ln_act_fwd(g_pre, gamma, beta, 1e-3, 0, g_ln)
    em.gru_gate_fwd(g_ln, h_prev, h_c)
    hxg, Wg = hx.cuda(), W.cuda()
    assert cu.gemm_ln_supported(hxg, Wg, 1)
    traj = torch.zeros(M, 40 + R, device="cuda")
    nxt = torch.zeros(M, R + Kx, device="cuda")
    pre_g, ln_g = torch.empty(M, 3 * R, device="cuda"), torch.empty(M, 3 * R, device="cuda")
    cu.gemm_ln_gru(hxg, Wg, gamma.cuda(), beta.cuda(), 1e-3, h_prev.cuda(), traj[:, 40:], nxt[:, :R], pre_g, ln_g)
    close(traj[:, 40:], h_c, rtol=2e-5, atol=2e-6, what="fused GRU h")
    assert torch.equal(nxt[:, :R], traj[:, 40:]) and float(nxt[:, R:].abs().max()) == 0.0
    close(pre_g, g_pre, rtol=2e-5, what="fused GRU pre"), close(ln_g, g_ln, rtol=2e-5, atol=2e-5, what="fused GRU ln")
    # in place on the [h | x] buffer it just read (the discrete-action rollout), without the optional saves
    h2 = torch.empty(M, R, device="cuda")
    cu.gemm_ln_gru(hxg, Wg, gamma.cuda(), beta.cuda(), 1e-3, h_prev.cuda(), h2, hxg[:, :R])
    assert torch.equal(h2, traj[:, 40:]) and torch.equal(hxg[:, :R], h2)


@pytest.mark.parametrize("M,S,D,A,N,keep", [(1024, 32, 32, 2, 512, False), (64, 6, 5, 3, 128, True), (256, 32, 32, 18, 1024, True), (33, 64, 3, 1, 384, True)])
def test_onehot_linear_ln_equals_gather_then_layernorm(ops, M, S, D, A, N, keep):
    cu, em = ops
    g = torch.Generator().manual_seed(3)
    z = torch.nn.functional.one_hot(torch.randint(0, D, (M, S), generator=g), D).float().reshape(M, S * D)
    act, W = rnd(M, A, seed=1), rnd(N, S * D + A, seed=2, scale=0.1)
    gamma, beta = 1 + 0.1 * rnd(N, seed=5), 0.1 * rnd(N, seed=6)
    WT = W.t().contiguous()
    pre_c, out_c = torch.empty(M, N), torch.empty(M, N)
    em.onehot_linear(z, act, WT, pre_c, S, D)
    em.ln_act_fwd(pre_c, gamma, beta, 1e-3, 1, out_c)
    hx = torch.zeros(M, 16 + N, device="cuda")
    pre_g = torch.empty(M, N, device="cuda") if keep else None
    cu.onehot_linear_ln(z.cuda(), act.cuda(), WT.cuda(), gamma.cuda(), beta.cuda(), 1e-3, hx[:, 16:], S, D, pre=pre_g)
    close(hx[:, 16:], out_c, rtol=1e-5, atol=2e-6, what="onehot_linear_ln")
    if keep:
        close(pre_g, pre_c, rtol=1e-5, what="onehot_linear_ln pre")
    assert float(hx[:, :16].abs().max()) == 0.0


@pytest.mark.parametrize("M,Kin,A,unimix", [(1024, 512, 2, 0.01), (1024, 1024, 18, 0.01), (100, 64, 6, 0.0), (300, 400, 32, 0.01)])
def test_head_sample_equals_linear_then_cat_sample(ops, M, Kin, A, unimix):
    cu, em = ops
    X, W, b = rnd(M, Kin, seed=1), rnd(A, Kin, seed=2, scale=Kin ** -0.5), 0.1 * rnd(A, seed=3)
    q = torch.empty(M, A + 5).exponential_(1.0, generator=torch.Generator().manual_seed(4))[:, 2:2 + A]
    raw_c, hot_c = torch.empty(M, A), torch.empty(M, A)
    em.gemm(X, W, raw_c, False, True, bias=b)
    em.cat_sample(raw_c, q, unimix, 1, A, hot_c)
    Xg, Wg = X.cuda(), W.cuda()
    assert cu.head_sample_supported(Xg, Wg)
    raw_all, act_all = torch.zeros(M, A + 3, device="cuda"), torch.zeros(M, A + 3, device="cuda")
    qg = torch.zeros(M, A + 5, device="cuda")
    qg[:, 2:2 + A] = q.cuda()
    cu.head_sample(Xg, Wg, b.cuda(), qg[:, 2:2 + A], unimix, raw_all[:, 3:], act_all[:, 3:])
    close(raw_all[:, 3:], raw_c, rtol=1e-5, atol=1e-6, what="head logits")
    assert float((act_all[:, 3:].sum(-1) - 1).abs().max()) == 0.0
    mism = (act_all[:, 3:].cpu() != hot_c).any(-1).float().mean()
    assert float(mism) <= 2e-3, float(mism)                   # only near-ties of p/q may differ
    # identical to the two-launch CUDA path on the logits it wrote
    hot2 = torch.empty(M, A, device="cuda")
    cu.cat_sample(raw_all[:, 3:], qg[:, 2:2 + A], unimix, 1, A, hot2)
    assert torch.equal(hot2, act_all[:, 3:])
    assert float(raw_all[:, :3].abs().max()) == 0.0 and float(act_all[:, :3].abs().max()) == 0.0


def _nan(n, off=0):
    """n NaN floats starting `off` floats into a fresh (16-byte aligned) allocation"""
    return torch.full((n + off,), float("nan"), device="cuda")[off:]


def _runs_iff(ok, launch, *guards):
    """`launch` runs when its query accepted the shape; otherwise it raises before any kernel runs and every guard keeps
    its NaNs"""
    from sheeprl_b200.lib import B200RLError

    if ok:
        launch()
    else:
        with pytest.raises(B200RLError, match="bad argument"):
            launch()
    torch.cuda.synchronize()
    for g in guards:
        assert bool(g.isnan().all()) != ok


@pytest.mark.parametrize("case", list(HEAD_SAMPLE))
def test_head_sample_launch_accepts_what_its_query_accepts(ops, case):
    cu, _ = ops
    Kin, A, xo, wo, ok = HEAD_SAMPLE[case]
    M = 8
    X, W = _nan(M * Kin, xo).view(M, Kin).normal_(), _nan(A * Kin, wo).view(A, Kin).normal_()
    raw, hot = _nan(M * A).view(M, A), _nan(M * A).view(M, A)
    assert cu.head_sample_supported(X, W) == ok
    _runs_iff(ok, lambda: cu.head_sample(X, W, None, None, 0.01, raw, hot), raw, hot)


@pytest.mark.parametrize("case", list(ONEHOT_LINEAR))
def test_onehot_linear_launches_accept_what_their_queries_accept(ops, case):
    """the engine asks onehot_linear_supported, then onehot_linear_ln_supported for the fused form"""
    cu, _ = ops
    S, K, A, N, oo, gather, ln = ONEHOT_LINEAR[case]
    M = 8
    z = torch.nn.functional.one_hot(torch.randint(0, K, (M, S)), K).float().reshape(M, S * K).cuda()
    act, WT = torch.randn(M, A, device="cuda"), 0.1 * torch.randn(S * K + A, N, device="cuda")
    gamma, beta = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    out, out_ln = _nan(M * N, oo).view(M, N), _nan(M * N, oo).view(M, N)
    assert cu.onehot_linear_supported(S, K, A, N) == gather
    assert (gather and cu.onehot_linear_ln_supported(WT, out_ln)) == ln
    _runs_iff(gather, lambda: cu.onehot_linear(z, act, WT, out, S, K), out)
    _runs_iff(ln, lambda: cu.onehot_linear_ln(z, act, WT, gamma, beta, 1e-3, out_ln, S, K), out_ln)


@pytest.mark.parametrize("case", [c for c, (NB, h, w, *_, ok) in WGRAD_TC.items() if not ok or NB * h * w <= 1 << 20])
def test_conv_wgrad_tc_launch_accepts_what_its_query_accepts(ops, case):
    cu, _ = ops
    NB, h, w, Cs, Cb, ok = WGRAD_TC[case]
    assert cu.lib.b200rl_conv_wgrad_tc_supported(NB, h, w, Cs, Cb) == ok
    if NB * h * w <= 1 << 20:
        small, big = torch.randn(NB, h, w, Cs, device="cuda"), torch.randn(NB, 2 * h, 2 * w, Cb, device="cuda")
        ws = torch.empty(cu.lib.b200rl_conv_wgrad_tc_workspace(NB, h, w, Cs, Cb), device="cuda")
    else:                       # a refused pixel count beyond any buffer: the launch reads no operand before refusing
        small = big = ws = _nan(16)
    dW = _nan(Cs * Cb * 16)
    rc = cu.lib.b200rl_conv_wgrad_tc(small.data_ptr(), big.data_ptr(), dW.data_ptr(), ws.data_ptr(), NB, h, w, Cs, Cb,
                                     0, cu._st())
    torch.cuda.synchronize()
    assert (rc == 0) == ok and bool(dW.isnan().all()) != ok
