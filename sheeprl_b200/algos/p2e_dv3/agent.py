"""`build_agent` for Plan2Explore on the B200 engine — the reference's signature and return tuple
(`sheeprl/algos/p2e_dv3/agent.py:27-220`): world model, ensembles, task actor / critic / target critic, exploration
actor, the `critics_exploration` dict ({name: {"weight", "reward_type", "module", "target_module"}}) and the player.
Every module is a parameter container over the engine's flat HBM groups with the reference's state-dict keys."""
from __future__ import annotations

import math
from typing import Any, Dict, Optional, Sequence

import torch

from sheeprl_b200.algos.dreamer_v3.agent import ParamTree, WorldModel, initial_state
from sheeprl_b200.algos.dreamer_v3.player import PlayerDV3
from sheeprl_b200.algos.p2e_dv3.engine import P2EDV3Engine


class _Views:
    """adapter: several FlatGroups seen as one name -> tensor mapping (the ensembles' ModuleList)"""

    def __init__(self, *groups):
        self.views = {}
        for g in groups:
            if g is not None:
                self.views.update(g.views)


def build_agent(
    fabric,
    actions_dim: Sequence[int],
    is_continuous: bool,
    cfg: Dict[str, Any],
    obs_space,
    world_model_state: Optional[Dict[str, torch.Tensor]] = None,
    ensembles_state: Optional[Dict[str, torch.Tensor]] = None,
    actor_task_state: Optional[Dict[str, torch.Tensor]] = None,
    critic_task_state: Optional[Dict[str, torch.Tensor]] = None,
    target_critic_task_state: Optional[Dict[str, torch.Tensor]] = None,
    actor_exploration_state: Optional[Dict[str, torch.Tensor]] = None,
    critics_exploration_state: Optional[Dict[str, Dict[str, Any]]] = None,
    ops=None,
):
    cnn_keys, mlp_keys = list(cfg.algo.cnn_keys.encoder or []), list(cfg.algo.mlp_keys.encoder or [])
    cnn_dims = {k: int(math.prod(obs_space[k].shape[:-2])) for k in cnn_keys}
    in_channels = sum(cnn_dims.values()) if cnn_keys else 3    # agent.py:984
    eng = P2EDV3Engine(cfg, actions_dim, in_channels=in_channels, device=fabric.device, ops=ops, is_continuous=is_continuous,
                       mlp_dims={k: int(obs_space[k].shape[0]) for k in mlp_keys}, cnn_dims=cnn_dims)
    seed = int(cfg.get("seed", 0) or 0)
    g = torch.Generator().manual_seed(seed)
    nh, haf = cfg.algo.mlp_layers, bool(cfg.algo.hafner_initialization)
    wm_scale = {"rssm.transition_model._model.3.weight": 1.0, "rssm.representation_model._model.3.weight": 1.0,
                f"reward_model._model.{3 * nh}.weight": 0.0, f"continue_model._model.{3 * nh}.weight": 1.0,
                **{f"observation_model.mlp_decoder.heads.{i}.weight": 1.0
                   for i in range(len(cfg.algo.mlp_keys.decoder or []))}} if haf else {}
    n_heads = 1 if is_continuous else len(actions_dim)
    ac_scale = {f"mlp_heads.{i}.weight": 1.0 for i in range(n_heads)} if haf else {}
    cr_scale = {f"_model.{3 * nh}.weight": 0.0} if haf else {}
    eng.wm.load(initial_state(eng.wm, wm_scale, g) if world_model_state is None else world_model_state)
    eng.actor.load(initial_state(eng.actor, ac_scale, g) if actor_task_state is None else actor_task_state)
    eng.critic.load(initial_state(eng.critic, cr_scale, g) if critic_task_state is None else critic_task_state)
    eng.target.load(eng.critic.state_dict() if target_critic_task_state is None else target_critic_task_state)
    eng.actor_expl.load(initial_state(eng.actor_expl, ac_scale, g) if actor_exploration_state is None else actor_exploration_state)
    critics_exploration = {}
    for k, c in eng.critics_expl.items():
        st = (critics_exploration_state or {}).get(k)
        c["group"].load(initial_state(c["group"], cr_scale, g) if st is None else st["module"])
        c["target"].load(c["group"].state_dict() if st is None else st["target_module"])
        critics_exploration[k] = {"weight": c["weight"], "reward_type": c["reward_type"], "module": ParamTree(c["group"].views),
                                  "target_module": ParamTree(c["target"].views)}
    if ensembles_state is None:
        # each member from its own seed (the reference seeds `cfg.seed + i` per member, agent.py:177-199)
        state = {}
        for i in range(eng.n_ens):
            grp = eng.ens_last if i == eng.n_ens - 1 else eng.ens_rest
            gi = torch.Generator().manual_seed(seed + i)
            member = initial_state(grp, {}, gi)
            state.update({n: v for n, v in member.items() if n.startswith(f"{i}.")})
        ensembles_state = state
    eng.load_ensembles(ensembles_state)

    world_model = WorldModel(eng.wm.views)
    ensembles = ParamTree(_Views(eng.ens_rest, eng.ens_last).views)
    actor_task, critic_task, target_task = ParamTree(eng.actor.views), ParamTree(eng.critic.views), ParamTree(eng.target.views)
    actor_exploration = ParamTree(eng.actor_expl.views)
    modules = [world_model, ensembles, actor_task, critic_task, target_task, actor_exploration]
    modules += [m for c in critics_exploration.values() for m in (c["module"], c["target_module"])]
    for m in modules:
        object.__setattr__(m, "_b200_engine", eng)
    exploring = str(cfg.algo.player.get("actor_type", "exploration")) == "exploration"
    player = PlayerDV3(eng, cfg.env.num_envs, actor_type="exploration" if exploring else "task",
                       actor_group=eng.actor_expl if exploring else eng.actor)
    return world_model, ensembles, actor_task, critic_task, target_task, actor_exploration, critics_exploration, player
