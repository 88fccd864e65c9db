"""DroQ on a GPU-less host: the oracle against the executed reference (tests/golden/droq_*.pt, and the reference run live
where its checkout is present), the engine's kernel schedule against the same fixtures with the torch test double in
place of the CUDA ops, and the public surface: reference state-dict keys, torch's Adam state layout, the replay rows,
the logged metrics and the refusals."""
import os

import numpy as np
import pytest
import torch

from oracle import droq_oracle as DO
from oracle import ref_harness
from oracle.dv3_oracle import AdamState
from oracle.ops_emul_droq import DroQEmulOps, pack_masks
from tests.test_sac_cpu import assert_group_close

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ["droq_tiny", "droq_tiny_p0", "droq_exp"]
LR = 3e-4


def load(name):
    """a fixture; the large one keeps no initial parameters (they come from a seed, as its generator made them)"""
    fx = torch.load(os.path.join(GOLDEN, f"{name}.pt"), weights_only=False)
    sp = fx["spec"]
    if "init" not in fx:
        fx["init"] = DO.init_params(sp["obs_dim"], sp["act_dim"], sp["hidden"], sp["n_critics"], sp["p"], sp["seed"])
    return fx


def kept(fx, state):
    """`state` as the fixture keeps it: whole tensors, or the large fixture's fixed sampled entries"""
    return DO.sample_state(state) if fx["spec"].get("sampled") else state


def bounds(sp):
    low, high = torch.tensor(sp["low"]), torch.tensor(sp["high"])
    return (high - low) / 2, (high + low) / 2


def call_inputs(fx, c):
    """(critic rows, actor observations, eps_next, eps_cur, bool keep masks) of fixture call c"""
    sp, call = fx["spec"], fx["calls"][c]
    if "critic_data" in call:
        return call["critic_data"], call["actor_obs"], call["eps_next"], call["eps_cur"], call["keep"]
    from oracle.make_golden_droq import exp_data

    critic, actor = exp_data(sp)
    eps_next, eps_cur, keep = DO.draw_noise(sp["G"], sp["B"], sp["act_dim"], sp["n_critics"], sp["hidden"], sp["p"],
                                            call["noise_seed"])
    return critic, actor["observations"], eps_next, eps_cur, keep


def assert_losses(got, want, what, rtol=1e-4):
    gv, wv = [float(v) for v in got["Loss/value_loss"]], want["Loss/value_loss"]
    assert len(gv) == len(wv), what
    for a, b in zip(gv, wv):
        assert abs(a - b) <= rtol * max(1.0, abs(b)), (what, a, b)
    for k in ("Loss/policy_loss", "Loss/alpha_loss"):
        assert abs(float(got[k]) - want[k]) <= rtol * max(1.0, abs(want[k])), (what, k, float(got[k]), want[k])


def assert_params(got, want, what, steps):
    """assert_group_close for one or a few Adam steps.  After many steps (the 80 of `exp=droq`) fp32 summation-order
    differences flip the sign of near-zero gradient entries and Adam moves those by ~lr each time: every entry stays
    within a few lr, and most agree far tighter."""
    for g in ("actor", "qf", "qf_target", "log_alpha"):
        if steps <= 3:
            assert_group_close(got[g], want[g], f"{what}/{g}")
            continue
        for k, w in want[g].items():
            d = (got[g][k].detach().cpu() - w).abs()
            assert float(d.max()) <= 4 * LR and float(d.median()) <= 0.1 * LR, (what, g, k, float(d.max()))


def run_oracle(fx):
    sp = fx["spec"]
    P = {g: {k: v.clone() for k, v in d.items()} for g, d in fx["init"].items()}
    opts = [AdamState(P[g], LR, 1e-4) for g in ("qf", "actor", "log_alpha")]
    scale, bias = bounds(sp)
    for c in range(len(fx["calls"])):
        critic, actor_obs, eps_next, eps_cur, keep = call_inputs(fx, c)
        losses = DO.droq_train(P, *opts, critic, actor_obs, eps_next, eps_cur, keep, 0.99, 0.005, sp["n_critics"],
                               sp["p"], scale, bias, -float(sp["act_dim"]))
        yield fx["calls"][c], P, losses


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    fx = load(name)
    for call, P, losses in run_oracle(fx):
        assert_losses(losses, call["losses"], name)
        got = kept(fx, P)
        for g in ("actor", "qf", "qf_target", "log_alpha"):
            assert_group_close(got[g], call["after"][g], f"{name}/{g}")


@pytest.mark.skipif(not ref_harness.reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("name", ["droq_tiny", "droq_tiny_p0"])
def test_reference_regenerated_live_matches_fixture(name):
    from oracle import make_golden_droq as MG

    ref_harness.install()
    fx, live = load(name), MG.run(MG.FIXTURES[name])
    assert live["state_dict_keys"] == fx["state_dict_keys"]
    for a, b in zip(live["calls"], fx["calls"]):
        assert_losses(a["losses"], b["losses"], name)
        for g in ("actor", "qf", "qf_target"):
            for k, v in b["after"][g].items():
                assert torch.equal(a["after"][g][k], v), (name, g, k)


# ---------------------------------------------------------------------------------------------------------
# engine schedule (hand-derived backward) with the torch test double
# ---------------------------------------------------------------------------------------------------------
def make_engine(fx, device="cpu", ops=None):
    from sheeprl_b200.algos.droq.engine import DroQEngine

    sp = fx["spec"]
    opt = {"lr": LR, "eps": 1e-4, "betas": (0.9, 0.999)}
    eng = DroQEngine(sp["obs_dim"], sp["act_dim"], sp["hidden"], sp["hidden"], sp["n_critics"], sp["B"], 0.99, 0.005,
                     1.0, sp["p"], sp["low"], sp["high"], opt, opt, opt, device, ops or DroQEmulOps())
    init = fx["init"]
    eng.load_reference_state(init["actor"], init["qf"], init["qf_target"], init["log_alpha"]["log_alpha"])
    return eng


def engine_noise(eps_next, eps_cur, keep, dev):
    return {"eps_next": eps_next.to(dev), "eps_cur": eps_cur.to(dev), "masks": pack_masks(keep).to(dev)}


def check_engine(fx, eng, name):
    dev, sp = eng.device, fx["spec"]
    for c, call in enumerate(fx["calls"]):
        critic, actor_obs, eps_next, eps_cur, keep = call_inputs(fx, c)
        eng.train_call({k: v.to(dev) for k, v in critic.items()}, actor_obs.to(dev),
                       engine_noise(eps_next, eps_cur, keep, dev))
        # the late minibatches of an 80-step call see parameters that drifted as assert_params describes
        assert_losses({k: v.cpu() for k, v in eng.metrics_dict().items()}, call["losses"], name,
                      1e-4 if sp["G"] <= 3 else 5e-4)
        assert_params(kept(fx, eng.export_reference_state()), call["after"], name, sp["G"])


def check_engine_first_minibatch(fx, eng):
    """the `exp=droq` fixture's parameters after critic minibatch 1: a one-minibatch call with the same noise"""
    sp, dev = fx["spec"], eng.device
    critic, actor_obs, eps_next, eps_cur, keep = call_inputs(fx, 0)
    G, B = sp["G"], sp["B"]
    one = torch.cat([keep[:4], keep[4 * G:4 * G + 2]])
    eng.train_call({k: v[:B].to(dev) for k, v in critic.items()}, actor_obs.to(dev),
                   engine_noise(eps_next[:1], eps_cur, one, dev))
    got = kept(fx, eng.export_reference_state())
    for g in ("qf", "qf_target"):
        assert_group_close(got[g], fx["calls"][0]["after_minibatch1"][g], f"minibatch1/{g}")
    vl = eng.metrics_dict()["Loss/value_loss"].cpu()
    for a, b in zip(vl.tolist(), fx["calls"][0]["losses"]["Loss/value_loss"][:sp["n_critics"]]):
        assert abs(a - b) <= 1e-4 * max(1.0, abs(b))


@pytest.mark.parametrize("name", NAMES)
def test_engine_schedule_matches_reference(name):
    fx = load(name)
    check_engine(fx, make_engine(fx), name)


def test_engine_first_minibatch_of_exp_droq():
    fx = load("droq_exp")
    check_engine_first_minibatch(fx, make_engine(fx))


# ---------------------------------------------------------------------------------------------------------
# public surface
# ---------------------------------------------------------------------------------------------------------
class Fab:
    device, world_size, global_rank = torch.device("cpu"), 1, 0


class Space:
    def __init__(self, shape):
        self.shape = shape


def make_cfg(spec):
    from oracle.make_golden_droq import droq_cfg

    return droq_cfg(spec)


def box(sp):
    class Box:
        shape = (sp["act_dim"],)
        low = np.asarray(sp["low"], np.float32)
        high = np.asarray(sp["high"], np.float32)

    return Box


def build(sp, fab=Fab, cfg=None):
    from sheeprl_b200.algos.droq.agent import build_agent

    return build_agent(fab, cfg or make_cfg(sp), {"state": Space((sp["obs_dim"],))}, box(sp), ops=DroQEmulOps())


def reference_state_dict(fx):
    sd = {"_log_alpha": fx["init"]["log_alpha"]["log_alpha"]}
    for k, v in fx["init"]["actor"].items():
        sd[f"_actor._forward_module.{k}"] = v
    for k, v in fx["init"]["qf"].items():
        sd[f"_qfs.{k}"] = v
        sd[f"_qfs_unwrapped.{k}"] = v
    for k, v in fx["init"]["qf_target"].items():
        sd[f"_qfs_target.{k}"] = v
    return sd


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_keys_match_reference_and_round_trip(name):
    fx = load(name)
    agent, _ = build(fx["spec"])
    assert list(agent.state_dict()) == fx["state_dict_keys"]
    agent.load_state_dict(reference_state_dict(fx))
    sd = agent.state_dict()
    for k, v in fx["init"]["qf"].items():
        assert torch.equal(sd[f"_qfs.{k}"], v) and torch.equal(sd[f"_qfs_unwrapped.{k}"], v), k
    for k, v in fx["init"]["actor"].items():
        assert torch.equal(sd[f"_actor.{k}"], v), k
    agent2, _ = build(fx["spec"])
    agent2.load_state_dict(sd)
    for k, v in agent2.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_qf_adam_state_has_torch_layout_and_loads_torch_state():
    from sheeprl_b200.algos.droq.droq import make_optimizers

    fx = load("droq_tiny_p0")                       # n = 2: ten tensors per critic
    agent, _ = build(fx["spec"])
    _, qf_opt, _ = make_optimizers(agent, make_cfg(fx["spec"]))
    assert fx["calls"][0]["qf_opt_state_len"] == 20
    assert [p.shape for p in qf_opt.param_groups[0]["params"]] == [v.shape for v in fx["init"]["qf"].values()]
    fx3 = load("droq_tiny")                         # a torch.optim.Adam state written by the reference (n = 3)
    agent3, _ = build(fx3["spec"])
    _, qf3, _ = make_optimizers(agent3, make_cfg(fx3["spec"]))
    torch_sd = fx3["qf_opt_state"]
    qf3.load_state_dict(torch_sd)
    out = qf3.state_dict()
    assert len(out["state"]) == len(torch_sd["state"]) == 30
    for i, st in torch_sd["state"].items():
        assert int(out["state"][i]["step"]) == int(st["step"]) == fx3["spec"]["G"] * fx3["spec"]["calls"]
        assert torch.equal(out["state"][i]["exp_avg"], st["exp_avg"])
        assert torch.equal(out["state"][i]["exp_avg_sq"], st["exp_avg_sq"])


class MeanMetricState:
    """torchmetrics.MeanMetric's state: update(x) adds x.sum() to `sum` and x.numel() to `weight`"""

    disabled = False

    def __init__(self):
        self.sum, self.weight, self.calls = {}, {}, {}

    def update(self, k, v):
        v = torch.as_tensor(v, dtype=torch.float64).detach()
        self.sum[k] = self.sum.get(k, 0.0) + float(v.sum())
        self.weight[k] = self.weight.get(k, 0) + v.numel()
        self.calls[k] = self.calls.get(k, 0) + 1


@pytest.mark.parametrize("name", ["droq_tiny", "droq_tiny_p0"])
def test_public_train_on_our_replay_buffer_uses_reference_rows(name):
    from sheeprl_b200.algos.droq.droq import make_optimizers, train
    from sheeprl_b200.data.buffers import ReplayBuffer

    fx = load(name)
    sp = fx["spec"]
    cfg = make_cfg(sp)
    agent, _ = build(sp)
    agent.load_state_dict(reference_state_dict(fx))
    opts = make_optimizers(agent, cfg)
    r = fx["rb"]
    rb = ReplayBuffer(r["size"], r["n_envs"], device="cpu", ops=DroQEmulOps())
    rb.add({k: v.numpy() for k, v in r["contents"].items()})
    rb._rng = np.random.default_rng(r["rng"])
    sampled = []
    real = rb.sample_tensors

    def recording(*a, **k):
        out = real(*a, **k)
        sampled.append({key: v.flatten(0, 1).clone() for key, v in out.items()})
        return out

    rb.sample_tensors = recording
    for c, call in enumerate(fx["calls"]):
        agg = MeanMetricState()
        _, _, eps_next, eps_cur, keep = call_inputs(fx, c)
        train(Fab, agent, *opts, rb, agg, cfg, sp["G"], noise=engine_noise(eps_next, eps_cur, keep, "cpu"))
        for k, v in call["critic_data"].items():
            assert torch.equal(sampled[2 * c][k], v), k
        assert torch.equal(sampled[2 * c + 1]["observations"], call["actor_obs"])
        # one update with the [G*n] tensor = the reference's G*n scalar updates of the value-loss MeanMetric
        want = call["losses"]["Loss/value_loss"]
        assert agg.calls["Loss/value_loss"] == 1 and agg.weight["Loss/value_loss"] == len(want) == sp["G"] * sp["n_critics"]
        assert abs(agg.sum["Loss/value_loss"] - sum(want)) <= 1e-4 * max(1.0, abs(sum(want)))
        assert agg.weight["Loss/policy_loss"] == agg.weight["Loss/alpha_loss"] == 1
        assert_params(agent._b200_engine.export_reference_state(), call["after"], name, sp["G"])
    assert opts[1].state_dict()["state"][0]["step"] == sp["G"] * len(fx["calls"])


def test_refusals():
    from sheeprl_b200.algos.droq.droq import train

    sp = load("droq_tiny")["spec"]

    class Fab2(Fab):
        world_size = 2

    with pytest.raises(NotImplementedError, match="multi-process DroQ"):
        build(sp, Fab2)
    agent, _ = build(sp)
    with pytest.raises(NotImplementedError, match="multi-process DroQ"):
        train(Fab2, agent, None, None, None, None, None, make_cfg(sp), 1)
    for bad in (1.0, -0.1, 1.5):
        cfg = make_cfg(sp)
        cfg.algo.critic.dropout = bad
        with pytest.raises(ValueError, match="dropout"):
            build(sp, cfg=cfg)
    cfg = make_cfg(sp)
    cfg.algo.critic.optimizer["_target_"] = "torch.optim.SGD"
    with pytest.raises(NotImplementedError, match="Adam"):
        build(sp, cfg=cfg)
    cfg = make_cfg(sp)
    cfg.algo.critic.hidden_size = 1025
    with pytest.raises(ValueError, match="1024"):
        build(sp, cfg=cfg)


def test_optimizer_factory_refuses_other_optimizers():
    from sheeprl_b200.algos.droq.droq import _optimizer_factory

    agent, _ = build(load("droq_tiny")["spec"])
    make = _optimizer_factory([agent])
    with pytest.raises(NotImplementedError, match="Adam"):
        make({"_target_": "torch.optim.SGD", "lr": 1e-3}, list(agent.qfs.parameters()))
