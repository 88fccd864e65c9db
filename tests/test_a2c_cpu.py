"""A2C on a GPU-less host: the oracle against the executed reference (tests/golden/a2c_*.pt), the engine's one-pass
schedule against the same fixtures with the torch test double in place of the CUDA ops, the RMSprop handle against
torch.optim.RMSprop, the refusals, and a two-rank data-parallel run."""
import math
import os

import pytest
import torch

from oracle import a2c_oracle as AO
from oracle import ppo_oracle as PO
from oracle.make_golden_a2c import a2c_cfg
from oracle.make_golden_ppo import obs_space
from oracle.ops_emul_a2c import A2CEmulOps
from tests.helpers import assert_params_close

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ["a2c_vector", "a2c_branches", "a2c_continuous", "a2c_pixel"]
LOGGED = ("Loss/policy_loss", "Loss/value_loss")
GRAD_RTOL = 1e-4           # per gradient tensor, l2 norms (the rule of tests/test_gpu_engine.py::check_grads)


def load(name):
    """a fixture with what it stores as seeds regenerated: the initial parameters, each call's rollout (rgb raw 0..255
    as float, as the reference received it) and the parameters after the run (torch's optimizer replayed over the
    recorded gradients, bit-identical to the reference's, oracle/make_golden_a2c.py)"""
    runs = torch.load(os.path.join(GOLDEN, f"{name}.pt"), weights_only=False)
    for r in runs:
        r["init"] = AO.init_params(r["spec"], r["init_seed"])
        for c in r["calls"]:
            c["data"] = PO.make_rollout(r["spec"], c["N"], c["data_seed"])
        r["after"] = AO.replay_updates(r["init"], r["opt"], [c["grads"] for c in r["calls"]])
    return runs


def step_size(opt_cfg) -> float:
    """the largest move of one element per optimizer step (the sign-flip bound of assert_params_close): Adam ~lr,
    RMSprop's first steps ~lr / sqrt(1 - alpha), momentum accumulates up to 1 / (1 - momentum) of that"""
    lr = float(opt_cfg["lr"])
    if opt_cfg["_target_"].endswith("Adam"):
        return lr
    return lr / math.sqrt(1 - float(opt_cfg.get("alpha", 0.99))) / (1 - float(opt_cfg.get("momentum", 0)))


def check_grads(got, want, what):
    gnorm = float(torch.sqrt(sum((v.double() ** 2).sum() for v in want.values())))
    gmax = max(float(v.abs().max()) for v in want.values())
    for k, w in want.items():
        diff = got[k].detach().cpu().float() - w
        assert float(diff.abs().max()) <= GRAD_RTOL * gmax + 1e-9, (what, k, float(diff.abs().max()), gmax)
        rel = float(diff.double().norm()) / (float(w.double().norm()) + 1e-6 * gnorm + 1e-30)
        assert rel <= GRAD_RTOL, (what, k, rel)


def check_losses(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for g, w in zip(got, want):
        for k, v in w.items():
            assert abs(g[k] - v) <= 1e-4 * max(1.0, abs(v)), (what, k, g[k], v)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    for j, r in enumerate(load(name)):
        p = {k: v.clone() for k, v in r["init"].items()}
        opt = AO.make_optimizer(p, r["opt"])
        for i, c in enumerate(r["calls"]):
            grads = {}
            logs = AO.a2c_train(p, opt, r["spec"], c["data"], c["index_batches"], r["hp"], grads_out=grads)
            check_losses(logs, c["losses"], (name, j, i))
            check_grads(grads, c["grads"], (name, j, i))
        assert_params_close({k: v.detach() for k, v in p.items()}, r["after"], step_size(r["opt"]), len(r["calls"]),
                            label=f"{name}/{j}")


# ---------------------------------------------------------------------------------------------------------
# engine schedule with the torch test double
# ---------------------------------------------------------------------------------------------------------
class Fab:
    device, world_size, global_rank = torch.device("cpu"), 1, 0


def build(r, device="cpu", ops=None, fab=None):
    """the public build_agent + the optimizer handle the reference's main gets from hydra, on `ops`"""
    from sheeprl_b200.algos.a2c.a2c import _optimizer_factory
    from sheeprl_b200.algos.a2c.agent import build_agent

    class F(Fab):
        pass

    F.device = torch.device(device)
    spec = r["spec"]
    cfg = a2c_cfg(spec, r["hp"], r["calls"][0]["batch"], r["opt"])
    agent, player = build_agent(fab or F, spec["actions_dim"], spec["is_continuous"], cfg, obs_space(spec),
                                agent_state=r["init"], ops=ops or A2CEmulOps())
    opt = _optimizer_factory([agent])(dict(r["opt"]), list(agent.parameters()))
    return agent, opt, cfg


def engine_grads(eng):
    """the accumulated gradient the last update stepped with, clipped as the reference's clip_gradients does, in the
    reference's layout"""
    coef = 1.0
    if eng.hp["max_grad_norm"] > 0:
        coef = min(1.0, eng.hp["max_grad_norm"] / (float(eng.norm_out) + 1e-6))
    return {k: v * coef for k, v in eng.export_reference_state(eng.group.gviews).items()}


def check_engine(name, device="cpu", ops=None, uint8_image=False):
    for j, r in enumerate(load(name)):
        agent, opt, _ = build(r, device, ops)
        eng = agent._b200_engine
        for i, c in enumerate(r["calls"]):
            data = {k: v.to(device) for k, v in c["data"].items()}
            if uint8_image and "rgb" in data:
                data["rgb"] = data["rgb"].to(torch.uint8)
            logs = []
            eng.train(data, c["index_batches"], lambda l: logs.append(dict(zip(LOGGED, l.tolist()))))
            check_losses(logs, c["losses"], (name, j, i))
            check_grads(engine_grads(eng), c["grads"], (name, j, i))
        assert_params_close({k: v.cpu() for k, v in agent.state_dict().items()}, r["after"], step_size(r["opt"]),
                            len(r["calls"]), label=f"{name}/{j}")
        assert opt.state_dict()["state"][0]["step"] == len(r["calls"])


@pytest.mark.parametrize("name", NAMES)
def test_engine_schedule_matches_reference(name):
    check_engine(name)


@pytest.mark.parametrize("name", NAMES)
def test_public_train_draws_the_reference_minibatches(name):
    """train() without explicit indices draws the reference's one-epoch RandomSampler / BatchSampler stream: under
    each call's sampler seed it visits the recorded minibatches and logs two losses per minibatch"""
    from sheeprl_b200.algos.a2c.a2c import train

    for j, r in enumerate(load(name)):
        agent, opt, _ = build(r)
        for i, c in enumerate(r["calls"]):
            cfg = a2c_cfg(r["spec"], r["hp"], c["batch"], r["opt"])

            class Agg:
                disabled, rows = False, []

                def update(self, k, v):
                    self.rows.append((k, float(v)))

            agg = Agg()
            torch.manual_seed(c["sampler_seed"])
            train(Fab, agent, opt, {k: v.clone() for k, v in c["data"].items()}, agg, cfg)
            assert [k for k, _ in agg.rows] == list(LOGGED) * len(c["losses"])
            check_losses([dict(agg.rows[2 * m: 2 * m + 2]) for m in range(len(c["losses"]))], c["losses"], (name, j, i))
        assert_params_close(agent.state_dict(), r["after"], step_size(r["opt"]), len(r["calls"]), label=f"{name}/{j}")


# ---------------------------------------------------------------------------------------------------------
# the RMSprop handle against torch.optim.RMSprop
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, {"momentum": 0.9}, {"centered": True}, {"momentum": 0.5, "centered": True,
                                                                            "weight_decay": 1e-3}])
def test_rmsprop_handle_state_dict_matches_torch(kw):
    r = load("a2c_branches")[0]
    opt_cfg = dict({"_target_": "torch.optim.RMSprop", "lr": 1e-3, "eps": 1e-4}, **kw)
    agent, opt, _ = build(dict(r, opt=opt_cfg))
    eng = agent._b200_engine
    c = r["calls"][0]
    eng.train(c["data"], c["index_batches"])
    # torch's RMSprop over the same parameter list, stepped once with the same gradient
    p = {k: v.clone().requires_grad_(True) for k, v in r["init"].items()}
    ref = torch.optim.RMSprop(list(p.values()), **{k: v for k, v in opt_cfg.items() if k != "_target_"})
    grads = engine_grads(eng)
    for k, t in p.items():
        t.grad = grads[k].clone()
    ref.step()
    mine, theirs = opt.state_dict(), ref.state_dict()
    assert mine["param_groups"][0].keys() == theirs["param_groups"][0].keys()
    assert mine["param_groups"] == theirs["param_groups"]
    assert set(mine["state"]) == set(theirs["state"])
    for i in theirs["state"]:
        assert mine["state"][i].keys() == theirs["state"][i].keys()
        for k, v in theirs["state"][i].items():
            assert mine["state"][i][k].shape == v.shape and mine["state"][i][k].dtype == v.dtype, (i, k)
            assert torch.allclose(mine["state"][i][k], v, rtol=1e-5, atol=1e-7), (i, k)
    # a torch-written state loads into a fresh handle and continues identically
    agent2, opt2, _ = build(dict(r, opt=opt_cfg))
    agent2.load_state_dict({k: v.detach() for k, v in p.items()})
    opt2.load_state_dict(theirs)
    agent.load_state_dict({k: v.detach() for k, v in p.items()})
    opt.load_state_dict(theirs)
    c2 = r["calls"][1]
    for a in (agent, agent2):
        a._b200_engine.train(c2["data"], c2["index_batches"])
    for k, v in agent.state_dict().items():
        assert torch.equal(v, agent2.state_dict()[k]), k
    assert opt2.state_dict()["state"][0]["step"] == 2


def test_rmsprop_handle_refuses_a_foreign_layout_and_unsupported_flags():
    from sheeprl_b200.algos.a2c.a2c import B200RMSprop

    r = load("a2c_vector")[0]
    agent, opt, _ = build(r)
    sd = opt.state_dict()
    sd["param_groups"][0]["params"] = sd["param_groups"][0]["params"][:-1]
    with pytest.raises(ValueError, match="layout"):
        opt.load_state_dict(sd)
    for flag in ("maximize", "differentiable", "capturable"):
        with pytest.raises(NotImplementedError, match=flag):
            B200RMSprop(agent._b200_engine, lr=1e-3, **{flag: True})


# ---------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------
def test_loss_reduction_none_is_refused():
    r = load("a2c_vector")[0]
    with pytest.raises(ValueError, match="loss_reduction"):
        build(dict(r, hp=dict(r["hp"], loss_reduction="none")))


def test_one_row_minibatch_with_normalisation_is_refused():
    r = load("a2c_branches")[0]
    agent, _, _ = build(r)
    c = r["calls"][0]
    plan = [list(range(0, 23)), [23]]
    with pytest.raises(ValueError, match="one-row minibatch"):
        agent._b200_engine.train(c["data"], plan)
    em = A2CEmulOps()                      # the op specification refuses it too
    z = torch.zeros
    with pytest.raises(ValueError):
        em.a2c_loss(z(3, 5), z(3, 5), z(3), z(3), z(3), z(3, 5), z(3), z(2, 3), 2, [3, 2], 0, True, False, 0.5, 0.0)


def test_unequal_minibatches_are_refused():
    r = load("a2c_vector")[0]
    agent, _, _ = build(r)
    c = r["calls"][0]
    with pytest.raises(ValueError, match="share one size"):
        agent._b200_engine.train(c["data"], [list(range(0, 5)), list(range(5, 15)), list(range(15, 20))])


@pytest.mark.parametrize("target", ["torch.optim.SGD", "torch.optim.AdamW", "torch.optim.Adagrad"])
def test_other_optimizers_are_refused(target):
    from sheeprl_b200.algos.a2c.a2c import _optimizer_factory

    r = load("a2c_vector")[0]
    agent, _, _ = build(r)
    with pytest.raises(NotImplementedError, match="RMSprop"):
        _optimizer_factory([agent])({"_target_": target, "lr": 1e-3}, list(agent.parameters()))


def test_rmsprop_maximize_is_refused_through_the_factory():
    from sheeprl_b200.algos.a2c.a2c import _optimizer_factory

    r = load("a2c_vector")[0]
    agent, _, _ = build(r)
    with pytest.raises(NotImplementedError, match="maximize"):
        _optimizer_factory([agent])(dict(r["opt"], maximize=True), list(agent.parameters()))


def test_oversized_pixel_rollout_is_refused():
    """84x84x4 frames: the first conv's patch matrix (20*20 rows x 8*8*4 columns per image) passes 2^31 - 1 elements
    above 20 971 images"""
    from sheeprl_b200.algos.a2c.engine import A2CEngine

    spec = dict(cnn_channels=4, screen=84, mlp_dim=0, dense=64, layers=1, cnn_features=512, mlp_features=0,
                actions_dim=(6,), is_continuous=False, act="relu")
    hp = dict(vf_coef=0.25, ent_coef=0.01, normalize_advantages=True, max_grad_norm=0.5, loss_reduction="mean")
    eng = A2CEngine(spec, hp, {"name": "rmsprop", "lr": 1e-4}, "cpu", A2CEmulOps())
    assert eng._check_rows([40])[1] == 40
    assert eng._check_rows([64] * 327)[1] == 20928
    with pytest.raises(ValueError, match="32-bit"):
        eng._check_rows([64] * 328)


# ---------------------------------------------------------------------------------------------------------
# two ranks (gloo): the gradient is averaged once per train() call
# ---------------------------------------------------------------------------------------------------------
def _rank(rank, world, port, out):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    import torch.distributed as dist

    from sheeprl_b200.parallel import attach_data_parallel, init_process_group_from_env
    from tests.test_a2c_cpu import build, load

    init_process_group_from_env("gloo")
    r = load("a2c_vector")[0]
    agent, _, _ = build(r)
    eng = agent._b200_engine
    attach_data_parallel(eng)
    inner, calls = eng.allreduce, []

    def counting(t, name):
        calls.append(name)
        return inner(t, name)

    eng.allreduce = counting
    c = r["calls"][0]
    eng.train(c["data"], [ib for m, ib in enumerate(c["index_batches"]) if m % world == rank])
    out[rank] = {"calls": len(calls), "flat": eng.group.flat.clone(), "grad": eng.group.grad.clone()}
    dist.destroy_process_group()


def test_two_rank_gloo_averages_the_gradient_once_per_call():
    """each rank trains on half of the minibatches: one all-reduce per train() call (what no_backward_sync gives the
    reference), replicas identical, gradient = mean of the ranks' gradients"""
    import torch.multiprocessing as mp

    mp.set_start_method("spawn", force=True)
    out = mp.Manager().dict()
    mp.spawn(_rank, args=(2, 32300 + (os.getpid() % 500), out), nprocs=2, join=True)
    a, b = out[0], out[1]
    assert a["calls"] == b["calls"] == 1
    assert torch.equal(a["flat"], b["flat"]) and torch.equal(a["grad"], b["grad"])
    r = load("a2c_vector")[0]
    c = r["calls"][0]
    gs = []
    for rank in range(2):
        agent, _, _ = build(r)
        agent._b200_engine.train(c["data"], [ib for m, ib in enumerate(c["index_batches"]) if m % 2 == rank])
        gs.append(agent._b200_engine.group.grad.clone())
    want = 0.5 * (gs[0] + gs[1])
    assert float((a["grad"] - want).abs().max()) <= 1e-6 * float(want.abs().max())
