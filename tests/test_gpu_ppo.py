"""PPO on the GPU through the C-ABI: the new kernels against the torch test double and the whole train() against the
executed reference (tests/golden/ppo_*.pt; 1e-4 relative fp32), plus the full-size pixel minibatch (BASELINE config
2 shape: 64 x 12x84x84, NatureCNN 512 features) against the oracle."""
import pytest
import torch

from oracle.ops_emul import EmulOps
from tests.test_ppo_cpu import NAMES, assert_params_close, check_engine, load, make_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def close(a, b, rtol=1e-4, atol=1e-5, what=""):
    a, b = a.detach().cpu(), b.detach().cpu()
    err = (a - b).abs()
    assert bool((err <= atol + rtol * b.abs()).all()), (what, float(err.max()))


@pytest.mark.parametrize("cont,clipv,norm", [(False, False, False), (False, True, True), (True, False, True), (True, True, False),
                                             (2, True, True), (2, False, False)])
def test_ppo_loss_kernel(cu, cont, clipv, norm):
    """cont: False discrete, True `normal`, 2 `tanh_normal` (stored actions tanh-squashed, some at the clamp)"""
    em = EmulOps()
    B, dims = 300, [4, 3]
    width = 2 * sum(dims) if cont else sum(dims)
    g = torch.Generator().manual_seed(5)
    head = rnd(B, width, seed=1)
    if cont == 2:
        actions = torch.tanh(rnd(B, sum(dims), seed=2) * 1.5)
        actions[:5] = torch.tensor([1.0, -1.0, 0.9999995, 0.0, -0.99999]).unsqueeze(-1)      # clamp region of safeatanh
    elif cont:
        actions = rnd(B, sum(dims), seed=2)
    else:
        actions = torch.cat([torch.nn.functional.one_hot(torch.randint(0, n, (B,), generator=g), n).float() for n in dims], -1)
    old_lp, adv, val, old_v, ret = (rnd(B, seed=i) * 0.3 for i in range(3, 8))
    outs_w = [torch.zeros(B, width), torch.zeros(B), torch.zeros(3)]
    outs_g = [t.cuda() for t in outs_w]
    args = (dims, cont, clipv, norm, 0.2, 0.5, 0.01)
    em.ppo_loss(head, actions, old_lp - 2, adv, val, old_v, ret, *outs_w, *args)
    cu.ppo_loss(head.cuda(), actions.cuda(), (old_lp - 2).cuda(), adv.cuda(), val.cuda(), old_v.cuda(), ret.cuda(), *outs_g, *args)
    for gg, w, nme in zip(outs_g, outs_w, ("dhead", "dvalues", "losses")):
        close(gg, w, rtol=2e-4, atol=1e-6, what=nme)


@pytest.mark.parametrize("name", NAMES)
def test_engine_matches_reference(cu, name):
    fx = load(name)
    check_engine(fx, make_engine(fx, device="cuda", ops=cu), name, uint8_image=True)


def test_full_size_pixel_minibatch_against_oracle(cu):
    """BASELINE config 2 shapes: minibatch 64 of 12x84x84 uint8, NatureCNN -> 512, 2x64 tanh MLPs, 6 actions."""
    from oracle import ppo_oracle as PO
    from oracle.dv3_oracle import AdamState
    from sheeprl_b200.algos.ppo.agent import default_init
    from sheeprl_b200.algos.ppo.engine import PPOEngine

    spec = dict(cnn_channels=12, screen=84, mlp_dim=0, dense=64, layers=2, cnn_features=512, mlp_features=64,
                actions_dim=(6,), is_continuous=False, act="tanh")
    hp = dict(clip_coef=0.2, vf_coef=1.0, ent_coef=0.01, clip_vloss=True, normalize_advantages=True, max_grad_norm=0.5)
    opt = {"lr": 1e-3, "eps": 1e-4, "betas": (0.9, 0.999)}
    eng = PPOEngine(spec, hp, opt, "cuda", cu)
    init = default_init(eng.reference_shapes(), torch.Generator().manual_seed(0))
    eng.load_reference_state(init)
    data = PO.make_rollout(spec, 128, seed=1)
    batches = [list(range(0, 64)), list(range(64, 128))]
    p = {k: v.clone() for k, v in init.items()}
    want = PO.ppo_train(p, AdamState(p, 1e-3, 1e-4), spec, data, batches, hp)
    dev = {k: v.cuda() for k, v in data.items()}
    dev["rgb"] = dev["rgb"].to(torch.uint8)
    logs = []
    eng.train(dev, batches, lambda l: logs.append(l.cpu()))
    for got, w in zip(logs, want):
        for i, k in enumerate(("Loss/policy_loss", "Loss/value_loss", "Loss/entropy_loss")):
            assert abs(float(got[i]) - w[k]) <= 1e-4 * max(1.0, abs(w[k])), (k, float(got[i]), w[k])
    assert_params_close(eng.export_reference_state(), p, "pixel64", steps=2)


@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("greedy", [False, True])
def test_ppo_act_continuous_modes(cu, mode, greedy):
    """b200rl_ppo_act on a Normal head: 1 `normal`, 2 `tanh_normal` as forward() returns it, 3 as get_actions() does"""
    em = EmulOps()
    B, dims = 257, [3, 2]
    A = sum(dims)
    head, noise = rnd(B, 2 * A, seed=1), rnd(B, A, seed=2)
    head[:4, :A] = torch.tensor([9.0, -9.0, 0.0, 20.0]).unsqueeze(-1)                        # saturating tanh / clamp
    aw, lw = torch.zeros(B, A), torch.zeros(B)
    ag, lg = torch.zeros(B, A, device="cuda"), torch.zeros(B, device="cuda")
    em.ppo_act(head, noise, aw, lw, dims, mode, greedy)
    cu.ppo_act(head.cuda(), noise.cuda(), ag, lg, dims, mode, greedy)
    close(ag, aw, rtol=2e-5, atol=2e-6, what="actions")
    close(lg, lw, rtol=1e-4, atol=1e-5, what="logp")


@pytest.mark.parametrize("name", ["ppo_branches", "ppo_continuous", "ppo_pixel", "ppo_tanh_ln", "ppo_multikey"])
@pytest.mark.parametrize("uint8_image", [False, True])
def test_player_matches_reference(cu, name, uint8_image):
    from tests.test_ppo_cpu import check_player

    check_player(name, device="cuda", ops=cu, uint8_image=uint8_image)
