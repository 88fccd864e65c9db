"""Plan2Explore exploration update on the DIAMBRA shape (`reward` encoded only, the MLP decoder over `[opp, own]`):
the decoder-keys oracle and the engine's kernel schedule on the torch test double against the executed reference
(tests/golden/p2e_dec_diambra.pt, oracle/make_golden_p2e_decoder_keys.py), and the state dicts of the reference's
Plan2Explore `build_agent`."""
import copy
import os

import torch

from sheeprl_b200.configs import make_p2e_dv3_cfg
from tests.helpers import GOLDEN, assert_params_close
from tests.test_p2e_cpu import LR, check_engine, check_metrics, check_moments, make_engine

NAME = "p2e_dec_diambra"


def load():
    fx = torch.load(os.path.join(GOLDEN, NAME + ".pt"), weights_only=False)
    return fx, make_p2e_dv3_cfg(**fx["cfg"])


def test_fixture_is_a_decoder_subset():
    _, cfg = load()
    assert list(cfg.algo.mlp_keys.encoder) == ["own", "opp", "reward"]
    assert list(cfg.algo.mlp_keys.decoder) == ["opp", "own"]


def test_oracle_matches_reference():
    from oracle.make_golden_p2e_decoder_keys import run_oracle

    fx, cfg = load()
    p, metrics, moments = run_oracle(cfg, copy.deepcopy(fx["init"]), [{k: v.float() for k, v in d.items()} for d in fx["data"]],
                                     fx["noise"])
    for s, m in enumerate(fx["metrics"]):
        check_metrics(metrics[s], m, f"step{s}")
    for name, want in fx["after"].items():
        assert_params_close(p[name], want, LR.get(name, 8e-5), len(fx["data"]), label=name)
    check_moments(moments, fx["moments"])


def test_engine_schedule_matches_reference():
    from oracle.ops_emul_decoupled import DecoupledEmulOps

    fx, cfg = load()
    eng = make_engine(fx, cfg, ops=DecoupledEmulOps())
    assert eng.has_vec_dec and not eng.vec_dec_same and eng.dec_vec_keys == ["opp", "own"]
    check_engine(fx, cfg, eng)


def test_state_dicts_are_the_reference_build_agent_ones():
    """fx["init"] holds the reference Plan2Explore build_agent's state dicts: same keys and shapes here, and the
    Hafner scale map covers the two decoder heads (uniform init; a truncated normal would exceed its bound)"""
    from oracle.ops_emul_decoupled import DecoupledEmulOps
    from sheeprl_b200.algos.p2e_dv3.agent import build_agent

    fx, cfg = load()

    class Fab:
        device = torch.device("cpu")

    class Space:
        def __init__(self, *shape):
            self.shape = shape

    space = {"rgb": Space(3, 64, 64), **{k: Space(d) for k, d in cfg.env.mlp_dims.items()}}
    wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl, player = build_agent(
        Fab, fx["actions_dim"], False, cfg, space, ops=DecoupledEmulOps())
    mods = {"wm": wm, "ens": ens, "actor_task": actor_task, "critic_task": critic_task, "target_task": target_task,
            "actor_expl": actor_expl}
    for k, c in critics_expl.items():
        mods[f"critic_expl_{k}"], mods[f"target_expl_{k}"] = c["module"], c["target_module"]
    for n, m in mods.items():
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == \
            {k: tuple(v.shape) for k, v in fx["init"][n].items()}, n
    sd = wm.state_dict()
    for i in range(2):                  # uniform(scale 1) init: |w| <= sqrt(3 / fan_avg)
        w = sd[f"observation_model.mlp_decoder.heads.{i}.weight"]
        assert float(w.abs().max()) <= (3.0 / ((w.shape[0] + w.shape[1]) / 2)) ** 0.5 + 1e-6
    assert "observation_model.mlp_decoder.heads.2.weight" not in sd
    wm.load_state_dict(fx["init"]["wm"])
    assert torch.equal(wm.state_dict()["observation_model.mlp_decoder.heads.1.bias"],
                       fx["init"]["wm"]["observation_model.mlp_decoder.heads.1.bias"])
