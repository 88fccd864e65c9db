"""The float64 references of the CUDA-core products (oracle/simt_ref.py) against the fp32 op emulators
(oracle/ops_emul.py, oracle/ops_emul_recurrent.py) and float64 autograd, on small shapes, so that a layout or
recurrence mistake in a reference fails without a GPU.  The GPU precision tests (tests/test_gpu_simt_precision.py) hold
the kernels to these references."""
import pytest
import torch

from oracle import simt_ref
from oracle.ops_emul_recurrent import RecurrentEmulOps

em = RecurrentEmulOps()


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel(got, ref, mag):
    return float(((got.double() - ref).abs() / (mag + 1e-30)).max())


@pytest.mark.parametrize("epi", ["none", "relu", "tanh", "drelu", "dtanh"])
@pytest.mark.parametrize("shared_a", [False, True], ids=["per_net", "broadcast_a"])
@pytest.mark.parametrize("acc", [False, True], ids=["store", "accumulate"])
def test_bgemm64(epi, shared_a, acc):
    nets, M, N, K = 3, 11, 7, 19
    A = rnd(1 if shared_a else nets, M, K, seed=1)
    W = rnd(nets, N, K, seed=2)
    bias = rnd(nets, N, seed=3)
    aux = torch.relu(rnd(nets, M, N, seed=4)) if epi == "drelu" else torch.tanh(rnd(nets, M, N, seed=4))
    C0, r0 = rnd(nets, M, N, seed=5), rnd(nets, M, seed=6)
    C, rsum = (C0.clone(), r0.clone()) if acc else (torch.empty(nets, M, N), torch.empty(nets, M))
    em.bgemm(A, W.transpose(1, 2), C, bias=bias, aux=aux, rsum=rsum, epi=epi, accumulate=acc)
    ref, mag, rs = simt_ref.bgemm64(A, W.transpose(1, 2), bias, aux, epi, C0 if acc else None)
    assert ref.dtype == torch.float64 and ref.shape == (nets, M, N) and rs.shape == (nets, M)
    assert bool((mag >= (ref - (C0.double() if acc else 0)).abs() * (1 - 1e-12) - 1e-12).all()) or epi != "none"
    assert rel(C, ref, mag) < 1e-6, epi
    want_rs = rs + (r0.double() if acc else 0)
    assert float((rsum.double() - want_rs).abs().max()) < 1e-5
    # the magnitude is the product of the absolute operands (+ |bias| + |C0|), independent of the epilogue
    a = A.double().abs().expand(nets, -1, -1)
    want = a @ W.double().abs().transpose(1, 2) + bias.double().abs().unsqueeze(1) + (C0.double().abs() if acc else 0)
    assert torch.allclose(mag, want, rtol=1e-12, atol=0)


def test_bgemm64_drelu_masks_exact_zeros():
    A, B = rnd(1, 4, 5, seed=1), rnd(1, 5, 6, seed=2)
    aux = torch.relu(rnd(1, 4, 6, seed=3))
    assert bool((aux == 0).any())
    ref, _, _ = simt_ref.bgemm64(A, B, aux=aux, epi="drelu")
    assert bool((ref[aux == 0] == 0).all()) and bool((ref[aux > 0] != 0).all())


def lstm_case(T, B, H, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T
    return (rnd(T, B, 4 * H, seed=seed + 1), rnd(4 * H, H, seed=seed + 2, scale=H ** -0.5),
            rnd(B, H, seed=seed + 3, scale=0.5), rnd(B, H, seed=seed + 4, scale=0.5), lengths,
            rnd(T, B, H, seed=seed + 5))


def fwd64(xw, W, h0, c0, lengths, requires_grad=False):
    """float64 forward built from lstm_step64, with padded steps as the kernel has them; the pre-activations are leaves
    of the graph when requires_grad, so autograd gives d_gates"""
    T, B, G = xw.shape
    H = G // 4
    xw = xw.double().clone().requires_grad_(requires_grad)
    h, c = h0.double(), c0.double()
    outs, gates, cs = [], [], []
    for t in range(T):
        v = (t < lengths.long()).unsqueeze(-1)
        g, cn, hn, _ = simt_ref.lstm_step64(xw[t], W, h, c)
        outs.append(torch.where(v, hn, torch.zeros_like(hn)))
        gates.append(torch.where(v, g, torch.zeros_like(g)))
        cs.append(torch.where(v, cn, torch.zeros_like(cn)))
        h, c = torch.where(v, hn, h), torch.where(v, cn, c)
    return xw, torch.stack(outs), torch.stack(gates), torch.stack(cs), h, c


@pytest.mark.parametrize("T,B,H", [(1, 3, 4), (5, 6, 8), (9, 4, 12)])
def test_lstm_step64_matches_emulator(T, B, H):
    xw, W, h0, c0, lengths, _ = lstm_case(T, B, H, seed=T + B + H)
    out, gates, cs, hT, cT = (torch.zeros(T, B, H), torch.zeros(T, B, 4 * H), torch.zeros(T, B, H), torch.zeros(B, H),
                              torch.zeros(B, H))
    em.lstm_seq_fwd(xw, W, h0, c0, lengths, out, gates, cs, hT, cT)
    _, o64, g64, c64, h64T, c64T = fwd64(xw, W, h0, c0, lengths)
    for got, want in ((out, o64), (gates, g64), (cs, c64), (hT, h64T), (cT, c64T)):
        assert float((got.double() - want).abs().max()) < 1e-5
    # teacher-forced: one step from the emulator's own state reproduces its next step
    t = T - 1
    hp, cp = (out[t - 1], cs[t - 1]) if t > 0 else (h0, c0)
    g, c, h, mag = simt_ref.lstm_step64(xw[t], W, hp, cp)
    v = (t < lengths.long()).unsqueeze(-1)
    assert float(((h - out[t].double()).abs() * v).max()) < 1e-5
    assert float(((g - gates[t].double()).abs() * v).max()) < 1e-5
    assert bool((mag >= (xw[t].double() + hp.double() @ W.double().t()).abs() * (1 - 1e-12)).all())


def lstm_bwd_checks(T, B, H, seed):
    """(error vs float64 autograd, largest emulator error / propagated bound) of lstm_bwd64.  The saved forward is
    rounded to fp32 first and both backward passes read those same values, as the kernel's backward does."""
    xw, W, h0, c0, lengths, d_out = lstm_case(T, B, H, seed)
    xw64, out, gates, cs, _, _ = fwd64(xw, W, h0, c0, lengths, requires_grad=True)
    (out * d_out.double()).sum().backward()
    gates, cs = gates.detach(), cs.detach()
    dg, bound = simt_ref.lstm_bwd64(d_out, W, gates, cs, c0, lengths)
    auto = float((dg - xw64.grad).abs().max())
    g32, c32 = gates.float(), cs.float()
    dg_r, bound_r = simt_ref.lstm_bwd64(d_out, W, g32, c32, c0, lengths)
    dg32 = torch.zeros(T, B, 4 * H)
    em.lstm_seq_bwd(d_out, W, g32, c32, c0, lengths, dg32)
    d = (dg32.double() - dg_r).abs()
    ratio = float(torch.where(d == 0, torch.zeros_like(d), d / bound_r).max())
    pad = (torch.arange(T).unsqueeze(1) >= lengths.long().unsqueeze(0))
    assert bool((dg[pad] == 0).all()) and bool((bound[pad] == 0).all())
    return auto, ratio


@pytest.mark.parametrize("T,B,H", [(1, 3, 4), (6, 5, 8), (12, 4, 16)])
def test_lstm_bwd64_matches_autograd_and_bounds_the_emulator(T, B, H):
    auto, ratio = lstm_bwd_checks(T, B, H, seed=7 * T + H)
    assert auto < 1e-12, auto
    # the fp32 emulator is one fp32 implementation of the same recurrence: its error is inside the propagated bound
    assert ratio <= 1.0, ratio


def test_lstm_bwd64_checks_catch_a_dropped_forget_gate(monkeypatch):
    """a mutation of the reference (the cell gradient carried without the forget gate) must fail both comparisons"""
    monkeypatch.setattr(simt_ref, "_carry_dc", lambda dc, f: dc)
    auto, ratio = lstm_bwd_checks(6, 5, 8, seed=50)
    assert auto > 1e-3 and ratio > 1.0, (auto, ratio)


def test_tau1():
    u = 2.0 ** -24
    assert simt_ref.tau1(0) == 16 * u
    assert simt_ref.tau1(65536) == (16 + 512) * u
    # one dropped 16-wide k-step of positive U(0.5, 1) products (~16 / K of the sum) is far outside tau1 at K = 65536
    assert 16 / 65536 > 7 * simt_ref.tau1(65536)
