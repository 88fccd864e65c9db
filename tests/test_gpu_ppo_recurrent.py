"""Recurrent PPO on the GPU through the C-ABI: the LSTM sequence kernels and the masked PPO objective against their
torch specifications (oracle/ops_emul_recurrent.py), and the whole train() / player against the executed reference
(tests/golden/ppo_rec_*.pt)."""
import pytest
import torch

from oracle.ops_emul_recurrent import RecurrentEmulOps as EmulOps
from tests.test_ppo_recurrent_cpu import NAMES, check_engine, check_player, load, make_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def close(a, b, rtol=1e-4, atol=1e-5, what=""):
    a, b = a.detach().cpu(), b.detach().cpu()
    err = (a - b).abs()
    assert bool((err <= atol + rtol * b.abs()).all()), (what, float(err.max()))


def _lstm_case(T, B, H, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T
    xw = rnd(T, B, 4 * H, seed=seed + 1)
    W = rnd(4 * H, H, seed=seed + 2, scale=1.0 / H ** 0.5)
    h0, c0 = rnd(B, H, seed=seed + 3, scale=0.5), rnd(B, H, seed=seed + 4, scale=0.5)
    d_out = rnd(T, B, H, seed=seed + 5)
    return xw, W, h0, c0, lengths, d_out


def _run_cuda(cu, xw, W, h0, c0, lengths, d_out):
    T, B, G = xw.shape
    H = G // 4
    z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
    out, gates, cs, hT, cT, dg = z(T, B, H), z(T, B, G), z(T, B, H), z(B, H), z(B, H), z(T, B, G)
    a = [t.cuda() for t in (xw, W, h0, c0, lengths)]
    cu.lstm_seq_fwd(*a, out, gates, cs, hT, cT)
    cu.lstm_seq_bwd(d_out.cuda(), a[1], gates, cs, a[3], a[4], dg)
    torch.cuda.synchronize()
    return out, gates, cs, hT, cT, dg


@pytest.mark.parametrize("T,B,H", [(1, 16, 64), (16, 64, 64), (16, 600, 64), (16, 40, 128), (16, 33, 256),
                                   (7, 300, 96), (1, 5, 256)])
def test_lstm_seq_matches_spec_and_is_bit_reproducible(cu, T, B, H):
    em = EmulOps()
    xw, W, h0, c0, lengths, d_out = _lstm_case(T, B, H, seed=T * 1000 + B + H)
    G = 4 * H
    out_w, gates_w, cs_w, hT_w, cT_w, dg_w = (torch.zeros(T, B, H), torch.zeros(T, B, G), torch.zeros(T, B, H),
                                              torch.zeros(B, H), torch.zeros(B, H), torch.zeros(T, B, G))
    em.lstm_seq_fwd(xw, W, h0, c0, lengths, out_w, gates_w, cs_w, hT_w, cT_w)
    em.lstm_seq_bwd(d_out, W, gates_w, cs_w, c0, lengths, dg_w)
    first = _run_cuda(cu, xw, W, h0, c0, lengths, d_out)
    for got, want, what in zip(first, (out_w, gates_w, cs_w, hT_w, cT_w, dg_w), ("out", "gates", "cs", "hT", "cT", "dgates")):
        close(got, want, rtol=2e-4, atol=2e-5, what=what)
    pad = torch.arange(T).unsqueeze(1) >= lengths.long().unsqueeze(0)
    assert float(first[0].cpu()[pad].abs().sum()) == 0.0 and float(first[5].cpu()[pad].abs().sum()) == 0.0
    second = _run_cuda(cu, xw, W, h0, c0, lengths, d_out)
    for a, b in zip(first, second):
        assert torch.equal(a, b)                                     # no atomics: bit-identical run to run


def test_lstm_seq_fwd_without_saved_state(cu):
    """acting: gates / cs are not kept; out and (hT, cT) are the same as with them"""
    xw, W, h0, c0, lengths, d_out = _lstm_case(1, 9, 64, seed=5)
    full = _run_cuda(cu, xw, W, h0, c0, lengths, d_out)
    out, hT, cT = torch.zeros(1, 9, 64, device="cuda"), torch.zeros(9, 64, device="cuda"), torch.zeros(9, 64, device="cuda")
    cu.lstm_seq_fwd(*(t.cuda() for t in (xw, W, h0, c0, lengths)), out, None, None, hT, cT)
    assert torch.equal(out, full[0]) and torch.equal(hT, full[3]) and torch.equal(cT, full[4])


@pytest.mark.parametrize("n_keep,clipv,norm", [(200, False, False), (200, True, True), (1, True, True),
                                               (0, False, True), (300, True, True)])
def test_ppo_loss_masked_kernel(cu, n_keep, clipv, norm):
    em = EmulOps()
    B, dims = 300, [4, 3]
    g = torch.Generator().manual_seed(7)
    head = rnd(B, sum(dims), seed=1)
    actions = torch.cat([torch.nn.functional.one_hot(torch.randint(0, n, (B,), generator=g), n).float() for n in dims], -1)
    old_lp, adv, val, old_v, ret = (rnd(B, seed=i) * 0.3 for i in range(3, 8))
    mask = torch.zeros(B)
    mask[torch.randperm(B, generator=g)[:n_keep]] = 1
    outs_w = [torch.full((B, sum(dims)), 7.0), torch.full((B,), 7.0), torch.zeros(3)]
    outs_g = [t.cuda() for t in outs_w]
    args = (dims, 0, clipv, norm, 0.2, 0.5, 0.01)
    em.ppo_loss_masked(head, actions, old_lp - 2, adv, val, old_v, ret, mask, *outs_w, *args)
    cu.ppo_loss_masked(head.cuda(), actions.cuda(), (old_lp - 2).cuda(), adv.cuda(), val.cuda(), old_v.cuda(),
                       ret.cuda(), mask.cuda(), *outs_g, *args)
    for gg, w, nme in zip(outs_g, outs_w, ("dhead", "dvalues", "losses")):
        close(gg, w, rtol=2e-4, atol=1e-6, what=nme)


def test_ppo_loss_masked_all_ones_equals_ppo_loss(cu):
    """with every row kept the masked objective is the unmasked one, bit for bit"""
    B, dims = 129, [5]
    g = torch.Generator().manual_seed(3)
    head = rnd(B, 5, seed=1).cuda()
    actions = torch.nn.functional.one_hot(torch.randint(0, 5, (B,), generator=g), 5).float().cuda()
    cols = [(rnd(B, seed=i) * 0.3).cuda() for i in range(3, 8)]
    a = [torch.zeros(B, 5, device="cuda"), torch.zeros(B, device="cuda"), torch.zeros(3, device="cuda")]
    b = [torch.zeros_like(t) for t in a]
    cu.ppo_loss(head, actions, *cols, *a, dims, 0, True, True, 0.2, 0.5, 0.01)
    cu.ppo_loss_masked(head, actions, *cols, torch.ones(B, device="cuda"), *b, dims, 0, True, True, 0.2, 0.5, 0.01)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("name", NAMES)
def test_engine_matches_reference(cu, name):
    fx = load(name)
    check_engine(fx, make_engine(fx, device="cuda", ops=cu), name, uint8_image=True)


@pytest.mark.parametrize("name", NAMES)
def test_public_train_matches_reference(cu, name):
    from oracle.make_golden_ppo import obs_space
    from oracle.make_golden_ppo_recurrent import rec_cfg
    from sheeprl_b200.algos.ppo_recurrent.agent import build_agent
    from sheeprl_b200.algos.ppo_recurrent.ppo_recurrent import make_optimizer, train
    from tests.test_ppo_cpu import assert_params_close

    fx = load(name)

    class Fab:
        device, world_size, global_rank = torch.device("cuda"), 1, 0

    cfg = rec_cfg(fx["spec"], fx["hp"], fx["batches"], fx["epochs"])
    agent, _ = build_agent(Fab, fx["spec"]["actions_dim"], False, cfg, obs_space(fx["spec"]), agent_state=fx["init"],
                           ops=cu)
    opt = make_optimizer(agent, cfg)
    data = {k: v.cuda() for k, v in fx["data"].items()}
    train(Fab, agent, opt, data, None, cfg, index_batches=fx["index_batches"])
    assert_params_close(agent.state_dict(), fx["after"], name, steps=len(fx["losses"]))


@pytest.mark.parametrize("name", NAMES)
def test_player_matches_reference(cu, name):
    check_player(name, device="cuda", ops=cu)
