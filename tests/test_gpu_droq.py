"""DroQ on the GPU through the C-ABI: the dropout keep masks, the fused Dropout-LayerNorm-ReLU forward / backward against
their specification (oracle/ops_emul_droq.py) evaluated in float64, DroQ's policy loss, the whole engine against the
executed reference (tests/golden/droq_*.pt), and one gradient step replayed from a CUDA graph against eager launches."""
import math

import pytest
import torch

from oracle.ops_emul_droq import DroQEmulOps, mask_words, pack_masks, unpack_masks
from tests.test_droq_cpu import check_engine, check_engine_first_minibatch, load, make_engine

pytestmark = pytest.mark.gpu
SPEC = DroQEmulOps()


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


def gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------ masks
@pytest.mark.parametrize("p", [0.01, 0.5])
def test_mask_keep_fraction(cu, p):
    words = torch.zeros(64, 2, 256, 8, dtype=torch.int32, device="cuda")
    cnt = torch.full((1,), 3, dtype=torch.int32, device="cuda")
    cu.dropout_mask(words, p, 11, 3, cnt)
    keep = unpack_masks(words.cpu(), 256)
    n = keep.numel()
    frac = float(keep.float().mean())
    assert abs(frac - (1 - p)) <= 5 * math.sqrt(p * (1 - p) / n), (p, frac)
    # every bit position carries the same rate (no stuck bit of the packing)
    per_bit = keep.reshape(-1, 32).float().mean(0)
    assert float((per_bit - (1 - p)).abs().max()) <= 5 * math.sqrt(p * (1 - p) / (n / 32))


def test_mask_keys(cu):
    def draw(seed, stream, counter):
        w = torch.zeros(4, 100, 3, dtype=torch.int32, device="cuda")
        cu.dropout_mask(w, 0.3, seed, stream, torch.full((1,), counter, dtype=torch.int32, device="cuda"))
        return w.cpu()

    a = draw(5, 3, 7)
    assert torch.equal(a, draw(5, 3, 7))
    for other in (draw(5, 3, 8), draw(5, 4, 7), draw(6, 3, 7)):
        assert float((a != other).float().mean()) > 0.5


# ------------------------------------------------------------------------------------------------ fused miniblock
def make_case(nets, B, H, p, seed, stride_pad=37):
    """inputs on the host (float64 copies are the reference); gamma / beta / dgamma live in flat buffers at a
    constant inter-critic stride H + stride_pad, with the gaps guarded"""
    g = gen(seed)
    sp = H + stride_pad
    z = torch.randn(nets, B, H, generator=g) * 2 + 0.3
    dy = torch.randn(nets, B, H, generator=g)
    flat_g = torch.full((nets * sp,), float("nan"))
    flat_b = torch.full((nets * sp,), float("nan"))
    gamma = torch.as_strided(flat_g, (nets, H), (sp, 1))
    beta = torch.as_strided(flat_b, (nets, H), (sp, 1))
    gamma.copy_(1 + 0.3 * torch.randn(nets, H, generator=g))
    beta.copy_(0.2 * torch.randn(nets, H, generator=g))
    words = None
    if p > 0:
        keep = torch.rand(nets, B, H, generator=g) >= p
        words = pack_masks(keep)
        pad = 32 * mask_words(H) - H
        if pad:                                      # padding bits set at random: they must never be read
            junk = torch.randint(0, 2 ** 31 - 1, words.shape[:-1], generator=g, dtype=torch.int64)
            junk = (junk << (32 - pad)) & 0xFFFFFFFF
            last = (words[..., -1].to(torch.int64) & 0xFFFFFFFF) | junk
            words[..., -1] = torch.where(last >= 2 ** 31, last - 2 ** 32, last).to(torch.int32)
    return dict(z=z, dy=dy, flat_g=flat_g, flat_b=flat_b, gamma=gamma, beta=beta, words=words, sp=sp)


def to_cuda_strided(flat, nets, H, sp):
    f = flat.cuda()
    return f, torch.as_strided(f, (nets, H), (sp, 1))


def guarded(shape, guard=64):
    """a CUDA tensor of `shape` inside a NaN-filled allocation; returns (view, whole)"""
    n = math.prod(shape)
    whole = torch.full((n + 2 * guard,), float("nan"), device="cuda")
    return whole[guard:guard + n].view(shape), whole


def assert_guard(whole, n, guard=64):
    w = whole.cpu()
    assert bool(torch.isnan(w[:guard]).all() and torch.isnan(w[guard + n:]).all()), "write outside the output range"


CASES = [(nets, B, H, p) for nets in (1, 2, 5) for B in (1, 7, 256, 2048) for H in (16, 64, 255, 256, 1024)
         for p in (0.0, 0.01, 0.5)]


@pytest.mark.parametrize("nets,B,H,p", CASES)
def test_dropout_ln_relu_fwd_bwd(cu, nets, B, H, p):
    c = make_case(nets, B, H, p, seed=nets * 1000 + B * 7 + H + int(p * 100))
    sp = c["sp"]
    # ---- device
    z, dy = c["z"].cuda(), c["dy"].cuda()
    _, gam = to_cuda_strided(c["flat_g"], nets, H, sp)
    _, bet = to_cuda_strided(c["flat_b"], nets, H, sp)
    words = None if c["words"] is None else c["words"].cuda()
    y, y_all = guarded((nets, B, H))
    st, st_all = guarded((nets, B, 2))
    cu.dropout_ln_relu_fwd(z, words, p, gam, bet, 1e-5, y, st)
    dz, dz_all = guarded((nets, B, H))
    dg_flat = torch.full((nets * sp,), float("nan"), device="cuda")
    db_flat = torch.full((nets * sp,), float("nan"), device="cuda")
    dg, db = (torch.as_strided(f, (nets, H), (sp, 1)) for f in (dg_flat, db_flat))
    cu.dropout_ln_relu_bwd(dy, y, z, words, p, st, gam, dz, dg, db)
    dz2, _ = guarded((nets, B, H))
    dg2_flat, db2_flat = dg_flat.clone(), db_flat.clone()
    dg2, db2 = (torch.as_strided(f, (nets, H), (sp, 1)) for f in (dg2_flat, db2_flat))
    cu.dropout_ln_relu_bwd(dy, y, z, words, p, st, gam, dz2, dg2, db2)
    dz3, _ = guarded((nets, B, H))
    cu.dropout_ln_relu_bwd(dy, y, z, words, p, st, gam, dz3)               # input-gradient-only mode
    torch.cuda.synchronize()
    for whole, n in ((y_all, y.numel()), (st_all, st.numel()), (dz_all, dz.numel())):
        assert_guard(whole, n)
    gaps = torch.ones(nets * sp, dtype=torch.bool)
    torch.as_strided(gaps, (nets, H), (sp, 1)).fill_(False)
    assert bool(torch.isnan(dg_flat.cpu()[gaps]).all() and torch.isnan(db_flat.cpu()[gaps]).all()), "dgamma stride"
    # ---- float64 reference (the specification on double inputs; the ReLU gate is the kernel's own y)
    D = torch.float64
    y64, st64 = torch.empty(nets, B, H, dtype=D), torch.empty(nets, B, 2, dtype=D)
    w = c["words"]
    SPEC.dropout_ln_relu_fwd(c["z"].to(D), w, p, c["gamma"].to(D), c["beta"].to(D), 1e-5, y64, st64)
    assert float((y.cpu().to(D) - y64).abs().max()) <= 2e-5 * max(1.0, float(y64.abs().max()))
    assert float((st.cpu().to(D) - st64).abs().max() / st64.abs().max()) <= 2e-5
    dz64, dg64, db64 = torch.empty(nets, B, H, dtype=D), torch.empty(nets, H, dtype=D), torch.empty(nets, H, dtype=D)
    SPEC.dropout_ln_relu_bwd(c["dy"].to(D), y.cpu().to(D), c["z"].to(D), w, p, st64, c["gamma"].to(D), dz64, dg64, db64)
    assert float((dz.cpu().to(D) - dz64).abs().max()) <= 1e-4 * max(1e-3, float(dz64.abs().max()))
    # column sums over B rows: bounded by the sums of the magnitudes they add
    x64 = c["z"].to(D) if w is None else c["z"].to(D) * unpack_masks(w, H).to(D) / (1.0 - p)
    xh64 = (x64 - st64[..., :1]) * st64[..., 1:]
    g64 = c["dy"].to(D) * (y.cpu() > 0).to(D)
    assert bool(((dg.cpu().to(D) - dg64).abs() <= 1e-5 * (g64 * xh64).abs().sum(1) + 1e-6).all())
    assert bool(((db.cpu().to(D) - db64).abs() <= 1e-5 * g64.abs().sum(1) + 1e-6).all())
    # bit-identical reductions run to run, and the input-only mode gives the same dz
    assert torch.equal(dg_flat.nan_to_num(), dg2_flat.nan_to_num()) and torch.equal(db_flat.nan_to_num(), db2_flat.nan_to_num())
    assert torch.equal(dz, dz2)
    assert torch.allclose(dz3, dz, rtol=1e-6, atol=1e-7)


def test_dropout_ln_relu_refusals(cu):
    z = torch.zeros(1, 4, 8, device="cuda")
    g = torch.ones(1, 8, device="cuda")
    st = torch.zeros(1, 4, 2, device="cuda")
    assert not cu.dropout_ln_relu_supported(1025) and cu.dropout_ln_relu_supported(1024)
    from sheeprl_b200.lib import B200RLError

    with pytest.raises(B200RLError, match="mask"):
        cu.dropout_ln_relu_fwd(z, None, 0.5, g, g, 1e-5, z.clone(), st)          # p > 0 needs a mask


# ------------------------------------------------------------------------------------------------ policy loss
@pytest.mark.parametrize("nets,B", [(1, 7), (2, 256), (5, 1000)])
def test_droq_actor_loss(cu, nets, B):
    g = gen(nets + B)
    q, logp, la = torch.randn(nets, B, generator=g), torch.randn(B, generator=g), torch.tensor([0.3])
    outs = [torch.zeros(nets, B), torch.zeros(1), torch.zeros(1), torch.zeros(1)]
    SPEC.droq_actor_loss(q, logp, la, -2.0, *outs)
    got = [t.cuda() for t in outs]
    for t in got:
        t.fill_(float("nan"))
    cu.droq_actor_loss(q.cuda(), logp.cuda(), la.cuda(), -2.0, *got)
    for a, b in zip(got, outs):
        assert torch.allclose(a.cpu(), b, rtol=1e-5, atol=1e-6), (a, b)


# ------------------------------------------------------------------------------------------------ engine
@pytest.mark.parametrize("name", ["droq_tiny", "droq_tiny_p0", "droq_exp"])
def test_engine_matches_reference(cu, name):
    fx = load(name)
    check_engine(fx, make_engine(fx, device="cuda", ops=cu), name)


def test_engine_first_minibatch_of_exp_droq(cu):
    fx = load("droq_exp")
    check_engine_first_minibatch(fx, make_engine(fx, device="cuda", ops=cu))


def test_gradient_step_is_graph_capturable(cu):
    """one gradient step and the actor step, with the noise and masks drawn on the device, replayed from a CUDA graph ==
    eager launches (so the call has no host synchronisation)"""
    fx = load("droq_tiny")
    sp = fx["spec"]
    e1, e2 = make_engine(fx, "cuda", cu), make_engine(fx, "cuda", cu)
    call = fx["calls"][0]
    B = sp["B"]
    critic = {k: v[:B].cuda() for k, v in call["critic_data"].items()}
    actor_obs = call["actor_obs"].cuda()
    for _ in range(3):
        e1.train_call(critic, actor_obs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        e2.train_call(critic, actor_obs)                     # warm-up on the side stream (call 1)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        e2.train_call(critic, actor_obs)                     # captured: call 2 happens at the first replay
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    a, b = e1.export_reference_state(), e2.export_reference_state()
    for grp in a:
        for k in a[grp]:
            assert torch.allclose(b[grp][k].cpu(), a[grp][k].cpu(), rtol=1e-5, atol=1e-6), (grp, k)
    assert torch.equal(e1.masks.cpu(), e2.masks.cpu())
