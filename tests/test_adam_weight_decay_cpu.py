"""Adam with L2 weight decay on a GPU-less host: the torch specification of `b200rl_adam_step_wd` against
torch.optim.Adam(weight_decay=...), the `B200Adam` handle's state against torch's, and the engines stepping their
groups with the handle's weight decay (the torch test double in place of the CUDA ops)."""
import copy

import pytest
import torch

from oracle.ops_emul_dv2 import DV2EmulOps
from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import B200Adam, make_optimizers
from sheeprl_b200.engine import DV3Engine
from sheeprl_b200.params import FlatGroup
from tests.helpers import load_fixture

LR, BETAS, EPS = 1e-2, (0.9, 0.999), 1e-6


def torch_adam_run(p0, grads, max_norm, wd):
    """fabric.clip_gradients + torch.optim.Adam(weight_decay=wd) in float64: the reference of the fp32 update"""
    p = torch.nn.Parameter(p0.double().clone())
    opt = torch.optim.Adam([p], lr=LR, betas=BETAS, eps=EPS, weight_decay=wd, foreach=False)
    for g in grads:
        p.grad = g.double().clone()
        if max_norm > 0:
            torch.nn.utils.clip_grad_norm_([p], max_norm)
        opt.step()
    return p.detach(), opt.state[p]


def spec_run(ops, p0, grads, max_norm, wd):
    p, m, v, out = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0), torch.zeros(1)
    step, normsq = torch.zeros(1, dtype=torch.int32), torch.zeros((), dtype=torch.float64)
    for g in grads:
        step += 1
        ops.sumsq(g, normsq)
        ops.adam_step(p, g, m, v, normsq, max_norm, LR, *BETAS, EPS, step, out, weight_decay=wd)
    return p, m, v


def case(n=1003, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(n, generator=gen), [torch.randn(n, generator=gen) * (0.1 * (s + 1)) for s in range(3)]


@pytest.mark.parametrize("wd", [1e-6, 1e-2, 0.5])
@pytest.mark.parametrize("max_norm", [0.0, 0.5])
def test_spec_matches_torch_adam_with_weight_decay(wd, max_norm):
    p0, grads = case(seed=int(wd * 1e6) + int(max_norm * 10))
    want, st = torch_adam_run(p0, grads, max_norm, wd)
    p, m, v = spec_run(DV2EmulOps(), p0, grads, max_norm, wd)
    torch.testing.assert_close(p.double(), want, rtol=0, atol=1e-6)
    torch.testing.assert_close(m.double(), st["exp_avg"], rtol=1e-5, atol=1e-8)
    torch.testing.assert_close(v.double(), st["exp_avg_sq"], rtol=1e-5, atol=1e-10)


def test_spec_weight_decay_enters_the_moments_before_the_update():
    """the decay is torch's coupled L2 term (Adam), not AdamW's decoupled shrink: the results differ"""
    p0, grads = case(seed=3)
    p, _, _ = spec_run(DV2EmulOps(), p0, grads, 0.0, 0.5)
    pw = torch.nn.Parameter(p0.double().clone())
    adamw = torch.optim.AdamW([pw], lr=LR, betas=BETAS, eps=EPS, weight_decay=0.5, foreach=False)
    for g in grads:
        pw.grad = g.double().clone()
        adamw.step()
    assert float((p.double() - pw.detach()).abs().max()) > 1e-4
    torch.testing.assert_close(p.double(), torch_adam_run(p0, grads, 0.0, 0.5)[0], rtol=0, atol=1e-6)


def test_spec_without_weight_decay_is_plain_adam():
    p0, grads = case(seed=4)
    a = spec_run(DV2EmulOps(), p0, grads, 0.5, 0.0)
    b = spec_run(DV2EmulOps(), p0, grads, 0.5, 0.0)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    torch.testing.assert_close(a[0].double(), torch_adam_run(p0, grads, 0.5, 0.0)[0], rtol=0, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------
# the B200Adam handle
# ---------------------------------------------------------------------------------------------------------
SHAPES = {"a.weight": (5, 7), "a.bias": (5,), "b.weight": (3, 5)}


def test_handle_state_round_trips_with_torch_adam():
    gen = torch.Generator().manual_seed(0)
    group = FlatGroup(SHAPES, "cpu")
    for v in group.views.values():
        v.copy_(torch.randn(v.shape, generator=gen))
    opt = B200Adam(group, list(SHAPES), LR, EPS, BETAS, weight_decay=1e-2)
    assert opt.weight_decay == 1e-2 and group.adam_kwargs() == {"weight_decay": 1e-2}
    params = [torch.nn.Parameter(v.clone()) for v in group.views.values()]
    ref = torch.optim.Adam(params, lr=LR, betas=BETAS, eps=EPS, weight_decay=1e-2, foreach=False)
    ops, normsq = DV2EmulOps(), torch.zeros((), dtype=torch.float64)
    for _ in range(3):
        for gv, p in zip(group.gviews.values(), params):
            g = torch.randn(p.shape, generator=gen)
            gv.copy_(g)
            p.grad = g.clone()
        ref.step()
        ops.sumsq(group.grad, normsq)
        group.step += 1
        ops.increment(group.step_t)
        ops.adam_step(group.flat, group.grad, group.exp_avg, group.exp_avg_sq, normsq, 0.0, opt.lr, *BETAS, EPS,
                      group.step_t, torch.zeros(1), **group.adam_kwargs())
    for v, p in zip(group.views.values(), params):
        torch.testing.assert_close(v, p.detach(), rtol=0, atol=1e-6)
    mine, theirs = opt.state_dict(), ref.state_dict()
    for k in ("lr", "betas", "eps", "weight_decay", "amsgrad"):
        assert mine["param_groups"][0][k] == theirs["param_groups"][0][k], k
    for i in theirs["state"]:
        assert float(mine["state"][i]["step"]) == float(theirs["state"][i]["step"]) == 3.0
        for k in ("exp_avg", "exp_avg_sq"):
            torch.testing.assert_close(mine["state"][i][k], theirs["state"][i][k], rtol=1e-5, atol=1e-9)
    # torch's dict loads into a handle built without decay and carries the decay over, as torch's own load does
    group2 = FlatGroup(SHAPES, "cpu")
    opt2 = B200Adam(group2, list(SHAPES), 1e-3, 1e-8)
    opt2.load_state_dict(theirs)
    assert opt2.weight_decay == 1e-2 and group2.adam_kwargs() == {"weight_decay": 1e-2} and group2.step == 3
    ref2 = torch.optim.Adam([torch.nn.Parameter(p.detach().clone()) for p in params], lr=1e-3, eps=1e-8)
    ref2.load_state_dict(mine)
    assert ref2.param_groups[0]["weight_decay"] == 1e-2


@pytest.mark.parametrize("wd", [-1e-6, float("nan")])
def test_handle_refuses_a_negative_weight_decay(wd):
    with pytest.raises(ValueError, match="weight_decay"):
        B200Adam(FlatGroup(SHAPES, "cpu"), list(SHAPES), LR, EPS, BETAS, weight_decay=wd)


def test_group_without_decay_keeps_the_plain_call():
    group = FlatGroup(SHAPES, "cpu")
    assert group.adam_kwargs() == {} and group.adam_kwargs(0.0) == {} and group.adam_kwargs(1e-6) == {"weight_decay": 1e-6}
    B200Adam(group, list(SHAPES), LR, EPS, BETAS)
    assert group.adam_kwargs(1e-6) == {}                  # the handle's value wins over the engine's config


# ---------------------------------------------------------------------------------------------------------
# engines
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("handles", [True, False])
def test_dv3_engine_steps_every_group_with_its_weight_decay(handles):
    """one Dreamer-V3 step with decay on every optimizer: each group's parameters move as torch.optim.Adam with that
    decay moves them from the same clipped gradient.  Without optimizer handles (an engine driven directly) the decay
    comes from the engine's optimizer config, as the reference's `instantiate(cfg.algo.*.optimizer)` applies it"""
    fx, cfg = load_fixture("dv3_tiny_a")
    decays = {"wm": 0.5, "actor": 0.25, "critic": 0.125}
    ocfgs = {"wm": cfg.algo.world_model, "actor": cfg.algo.actor, "critic": cfg.algo.critic}
    for n, wd in decays.items():
        ocfgs[n].optimizer.weight_decay = wd
    eng = DV3Engine(cfg, fx["actions_dim"], in_channels=3, device="cpu", ops=DV2EmulOps())
    if handles:
        make_optimizers(eng, cfg)
    groups = {"wm": eng.wm, "actor": eng.actor, "critic": eng.critic}
    for n in ("wm", "actor", "critic", "target"):
        getattr(eng, n).load(fx["init"][n])
    before = {n: g.flat.clone() for n, g in groups.items()}
    eng.train_step(copy.deepcopy({k: v.clone().float() for k, v in fx["data"][0].items()}), fx["noise"][0])
    for slot, (n, g) in enumerate(groups.items()):
        o, clip = ocfgs[n].optimizer, float(ocfgs[n].clip_gradients or 0.0)
        norm = float(eng.norms[slot])
        coef = min(1.0, clip / (norm + 1e-6)) if clip > 0 else 1.0
        p = torch.nn.Parameter(before[n].double().clone())
        p.grad = g.grad.double() * coef
        ref = torch.optim.Adam([p], lr=float(o.lr), betas=tuple(o.betas), eps=float(o.eps), weight_decay=decays[n])
        ref.step()
        torch.testing.assert_close(g.flat.double(), p.detach(), rtol=0, atol=2e-7, msg=n)
        plain = torch.nn.Parameter(before[n].double().clone())
        plain.grad = p.grad
        torch.optim.Adam([plain], lr=float(o.lr), betas=tuple(o.betas), eps=float(o.eps)).step()
        assert float((g.flat.double() - plain.detach()).abs().max()) > 1e-6, n   # the decay took effect
    if handles:
        assert eng.graph_key()[:3] == tuple((float(ocfgs[n].optimizer.lr), wd) for n, wd in decays.items())


@pytest.mark.parametrize("handle", [True, False])
def test_a2c_engine_steps_with_the_adam_weight_decay(handle):
    """A2C with an Adam config that sets weight_decay: the handle is accepted and the engine's update is
    torch.optim.Adam(weight_decay=...) over the same clipped gradient.  Without the handle the engine takes the decay
    from the optimizer config build_agent read"""
    from oracle.ops_emul_a2c import A2CEmulOps
    from tests.test_a2c_cpu import build, engine_grads, load

    class Ops(DV2EmulOps, A2CEmulOps):
        pass

    r = load("a2c_branches")[0]
    opt_cfg = {"_target_": "torch.optim.Adam", "lr": 1e-3, "eps": 1e-4, "weight_decay": 0.5}
    agent, opt, _ = build(dict(r, opt=opt_cfg), ops=Ops())
    assert isinstance(opt, B200Adam) and opt.weight_decay == 0.5
    eng = agent._b200_engine
    if not handle:
        eng.group.optimizer = None
    c = r["calls"][0]
    eng.train(c["data"], c["index_batches"])
    p = {k: torch.nn.Parameter(v.double().clone()) for k, v in r["init"].items()}
    ref = torch.optim.Adam(list(p.values()), lr=1e-3, eps=1e-4, weight_decay=0.5)
    grads = engine_grads(eng)
    for k, t in p.items():
        t.grad = grads[k].double().clone()
    ref.step()
    got = agent.state_dict()
    for k, t in p.items():
        torch.testing.assert_close(got[k].double(), t.detach(), rtol=0, atol=2e-7, msg=k)
