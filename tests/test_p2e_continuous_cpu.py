"""Plan2Explore (Dreamer-V3) with continuous `scaled_normal` actions on a GPU-less host: the oracle against the EXECUTED
reference (tests/golden/p2e_tiny_c.pt, oracle/make_golden_p2e_continuous.py: two
`p2e_dv3_exploration.train(is_continuous=True)` calls on state-vector observations), the engine's kernel schedule and
the public build_agent()/train() surface against the same fixture with the torch test double in place of the CUDA ops,
and the finetuning / acting paths of a continuous P2E agent."""
import copy
import os

import pytest
import torch

from sheeprl_b200.configs import make_p2e_dv3_cfg
from tests.helpers import GOLDEN, assert_params_close
from tests.test_p2e_cpu import LR, check_metrics, check_moments


def load():
    fx = torch.load(os.path.join(GOLDEN, "p2e_tiny_c.pt"), weights_only=False)
    assert fx["is_continuous"]
    return fx, make_p2e_dv3_cfg(**fx["cfg"])


def obs_space(cfg, space):
    """the state-vector observation space of the fixture's config"""
    return {k: space((d,)) for k, d in cfg.env.mlp_dims.items()}


def to(dev, fx, s):
    data = {k: v.clone().float().to(dev) for k, v in fx["data"][s].items()}
    noise = {k: ([x.to(dev) for x in v] if isinstance(v, list) else v.to(dev)) for k, v in fx["noise"][s].items()}
    return data, noise


def test_oracle_matches_reference():
    from oracle.make_golden_p2e_continuous import run_oracle

    fx, cfg = load()
    p, metrics, moments = run_oracle(cfg, copy.deepcopy(fx["init"]), fx["data"], fx["noise"])
    for s, m in enumerate(fx["metrics"]):
        check_metrics(metrics[s], m, f"step{s}")
    for name, want in fx["after"].items():
        assert_params_close(p[name], want, LR.get(name, 8e-5), len(fx["data"]), label=name)
    check_moments(moments, fx["moments"])


def make_engine(fx, cfg, device="cpu", ops=None):
    from oracle.ops_emul import EmulOps
    from sheeprl_b200.algos.p2e_dv3.engine import P2EDV3Engine

    eng = P2EDV3Engine(cfg, fx["actions_dim"], device=device, ops=ops or EmulOps(), is_continuous=True)
    for name, g in eng.groups().items():
        g.load(fx["init"][name])
    eng.load_ensembles(fx["init"]["ens"])
    return eng


def check_engine(fx, eng):
    for s in range(len(fx["data"])):
        eng.train_step(*to(eng.device, fx, s))
        check_metrics({k: v.cpu() for k, v in eng.metrics_dict().items()}, fx["metrics"][s], f"engine step{s}")
    got = {name: {k: v.cpu() for k, v in g.state_dict().items()} for name, g in eng.groups().items()}
    got["ens"] = {k: v.cpu() for k, v in eng.ensembles_state_dict().items()}
    for name, want in fx["after"].items():
        assert_params_close(got[name], want, LR.get(name, 8e-5), len(fx["data"]), label=name)
    moments = {"task": eng.moments_state.cpu(), **{k: c["moments_state"].cpu() for k, c in eng.critics_expl.items()}}
    check_moments(moments, fx["moments"])


def test_engine_schedule_matches_reference():
    fx, cfg = load()
    check_engine(fx, make_engine(fx, cfg))


def check_public_api(device="cpu", ops=None):
    """build_agent(is_continuous=True) from the fixture's state dicts + train() with the reference's positional signature
    land on the reference's metrics, parameters and Moments"""
    from oracle.ops_emul import EmulOps
    from sheeprl_b200.algos.p2e_dv3.agent import build_agent
    from sheeprl_b200.algos.p2e_dv3.p2e_dv3_exploration import make_optimizers, train
    from sheeprl_b200.algos.p2e_dv3.utils import Moments

    fx, cfg = load()
    init = fx["init"]

    class Fab:
        pass

    Fab.device = torch.device(device)

    class Space:
        def __init__(self, shape):
            self.shape = shape

    class Agg:
        disabled = False

        def __init__(self):
            self.values = {}

        def update(self, k, v):
            self.values[k] = float(v)

    crit_state = {k[len("critic_expl_"):]: {"module": init[k], "target_module": init["target_expl_" + k[len("critic_expl_"):]]}
                  for k in init if k.startswith("critic_expl_")}
    wm, ens, actor_t, critic_t, target_t, actor_e, critics_e, player = build_agent(
        Fab, fx["actions_dim"], True, cfg, obs_space(cfg, Space), init["wm"], init["ens"], init["actor_task"],
        init["critic_task"], init["target_task"], init["actor_expl"], crit_state, ops=ops or EmulOps())
    eng = wm._b200_engine
    assert eng.is_continuous and player.actor.is_continuous
    wo, ato, cto, eo, aeo, crit_opts = make_optimizers(eng, cfg)
    for k, c in critics_e.items():
        c["optimizer"] = crit_opts[k]
    mo = cfg.algo.actor.moments
    new_m = lambda: Moments(mo.decay, mo.max, mo.percentile.low, mo.percentile.high)  # noqa: E731
    m_task, m_expl = new_m(), {k: new_m() for k in critics_e}
    for s in range(len(fx["data"])):
        agg = Agg()
        data, noise = to(device, fx, s)
        train(Fab, wm, actor_t, critic_t, target_t, wo, ato, cto, data, agg, cfg, ens, eo, actor_e, critics_e, aeo, m_expl,
              m_task, True, fx["actions_dim"], noise=noise)
        check_metrics(agg.values, fx["metrics"][s], f"public step{s}")
    got = {"wm": wm.state_dict(), "ens": ens.state_dict(), "actor_task": actor_t.state_dict(), "actor_expl": actor_e.state_dict(),
           "critic_task": critic_t.state_dict()}
    for k, c in critics_e.items():
        got[f"critic_expl_{k}"] = c["module"].state_dict()
    for name, sd in got.items():
        assert_params_close({k: v.cpu() for k, v in sd.items()}, fx["after"][name], LR.get(name, 8e-5), len(fx["data"]), label=name)
    check_moments({"task": {"low": m_task.low, "high": m_task.high},
                   **{k: {"low": m.low, "high": m.high} for k, m in m_expl.items()}}, fx["moments"])
    assert aeo.state_dict()["state"][0]["step"] == len(fx["data"])


def test_public_api_matches_reference():
    check_public_api()


def test_public_train_refuses_a_mismatched_action_space():
    from oracle.ops_emul import EmulOps
    from sheeprl_b200.algos.p2e_dv3.agent import build_agent
    from sheeprl_b200.algos.p2e_dv3.p2e_dv3_exploration import train

    fx, cfg = load()

    class Fab:
        device = torch.device("cpu")

    class Space:
        def __init__(self, shape):
            self.shape = shape

    out = build_agent(Fab, fx["actions_dim"], True, cfg, obs_space(cfg, Space), ops=EmulOps())
    data, noise = to("cpu", fx, 0)
    with pytest.raises(ValueError):
        train(Fab, out[0], out[2], out[3], out[4], None, None, None, data, None, cfg, out[1], None, out[5], out[6], None,
              None, None, False, fx["actions_dim"], noise=noise)


def test_continuous_finetuning_update_is_the_task_behaviour_step():
    """p2e_dv3_finetuning.train(is_continuous=True) on a continuous P2E engine runs the continuous Dreamer-V3 step on the
    task actor / critic: bit-equal to a plain continuous Dreamer-V3 engine with the same task weights"""
    from oracle.ops_emul import EmulOps
    from sheeprl_b200.algos.dreamer_v3.agent import ParamTree
    from sheeprl_b200.algos.p2e_dv3.p2e_dv3_finetuning import train
    from sheeprl_b200.engine import DV3Engine

    fx, cfg = load()
    p2e = make_engine(fx, cfg)
    plain = DV3Engine(cfg, fx["actions_dim"], device="cpu", ops=EmulOps(), is_continuous=True)
    for g, n in ((plain.wm, "wm"), (plain.actor, "actor_task"), (plain.critic, "critic_task"), (plain.target, "target_task")):
        g.load(fx["init"][n])
    noise = {"post": fx["noise"][0]["post"], "img_state": fx["noise"][0]["img_state_task"],
             "img_action": fx["noise"][0]["img_action_task"]}
    data = lambda: {k: v.clone().float() for k, v in fx["data"][0].items()}  # noqa: E731
    wm = ParamTree(p2e.wm.views)
    object.__setattr__(wm, "_b200_engine", p2e)
    DV3Engine.train_step(plain, data(), noise)
    train(None, wm, None, None, None, None, None, None, data(), None, cfg, True, fx["actions_dim"], None, noise=noise)
    for a, b in ((plain.wm, p2e.wm), (plain.actor, p2e.actor), (plain.critic, p2e.critic)):
        assert torch.equal(a.flat, b.flat)
    assert torch.equal(plain.metrics, p2e.metrics)
    with pytest.raises(ValueError):
        train(None, wm, None, None, None, None, None, None, data(), None, cfg, False, fx["actions_dim"], None, noise=noise)


def test_player_acts_with_the_continuous_exploration_actor():
    """the player of a continuous P2E agent acts with the exploration actor's `scaled_normal` head: bit-equal to a plain
    continuous player that holds the exploration actor's weights"""
    from oracle.ops_emul import EmulOps
    from sheeprl_b200.algos.dreamer_v3.player import PlayerDV3
    from sheeprl_b200.engine import DV3Engine

    fx, cfg = load()
    eng = make_engine(fx, cfg)
    p2e_player = PlayerDV3(eng, 2, actor_type="exploration", actor_group=eng.actor_expl)
    assert p2e_player.eng.actor is eng.actor_expl and p2e_player.actor.is_continuous
    plain = DV3Engine(cfg, fx["actions_dim"], device="cpu", ops=EmulOps(), is_continuous=True)
    plain.wm.load(fx["init"]["wm"]), plain.actor.load(fx["init"]["actor_expl"])
    ref_player = PlayerDV3(plain, 2)
    g = torch.Generator().manual_seed(0)
    obs = {k: torch.randn(1, 2, d, generator=g) * 3 for k, d in cfg.env.mlp_dims.items()}
    noise = {"z": torch.empty(2, eng.Z).exponential_(1.0, generator=g), "a": torch.randn(2, eng.A, generator=g)}
    for p in (p2e_player, ref_player):
        p.init_states()
    for _ in range(2):
        (a,), (b,) = p2e_player.get_actions(obs, noise=noise), ref_player.get_actions(obs, noise=noise)
        assert a.shape == (1, 2, eng.A) and torch.equal(a, b)
    # the task actor differs from the exploration actor, so acting with it would not match
    assert not torch.equal(eng.actor.flat, eng.actor_expl.flat)
