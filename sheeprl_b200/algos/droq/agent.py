"""`build_agent` for the DroQ engine — same signature / return tuple as the reference
(`sheeprl/algos/droq/agent.py:270-336`).

`DroQAgent` is a parameter container: its tensors are views into the engine's flat groups and its `state_dict()` keys
follow the reference module tree (`_log_alpha`, `_actor.*`, `_qfs.{i}.*`, `_qfs_unwrapped.{i}.*` — a second
registration of the same critics that reference checkpoints carry — and `_qfs_target.{i}.*`).  The arithmetic of
`train()` runs in `DroQEngine` kernels; acting is `SACPlayer` on the shared actor group.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Any, Dict, Optional, Tuple

import torch

from sheeprl_b200.algos.droq.engine import DroQEngine
from sheeprl_b200.algos.sac.agent import SACAgent, SACPlayer, _default_linear_init


class _Parameters:
    """`.parameters()` of a flat group, in the reference module's order (what `hydra.utils.instantiate(<optimizer>,
    params=agent.qfs.parameters())` receives in the reference's `main`)"""

    def __init__(self, group):
        self._group = group

    def parameters(self):
        return iter(self._group.views.values())


class DroQAgent(SACAgent):
    """Reference surface used by `droq.main` / checkpoints (droq/agent.py:50-267)."""

    @property
    def qfs(self) -> _Parameters:
        return _Parameters(self._b200_engine.qf)

    @property
    def actor(self) -> _Parameters:
        return _Parameters(self._b200_engine.actor)

    def qfs_target_ema(self, critic_idx: int) -> None:
        e = self._b200_engine
        s = e.critic_slice(critic_idx)
        e.ops.ema(e.qf_target.flat[s], e.qf.flat[s], e.tau)

    def state_dict(self) -> "OrderedDict[str, torch.Tensor]":
        """the reference's key order: the agent's own parameter, then its modules as registered (SACActor's buffers
        before its submodules)"""
        e = self._b200_engine
        s = e.export_reference_state()
        out = OrderedDict([("_log_alpha", s["log_alpha"]["log_alpha"]), ("_actor.action_scale", e.scale.clone()),
                           ("_actor.action_bias", e.abias.clone())])
        for k in ("model._model.0.weight", "model._model.0.bias", "model._model.2.weight", "model._model.2.bias",
                  "fc_mean.weight", "fc_mean.bias", "fc_logstd.weight", "fc_logstd.bias"):
            out[f"_actor.{k}"] = s["actor"][k]
        for prefix, group in (("_qfs.", "qf"), ("_qfs_unwrapped.", "qf"), ("_qfs_target.", "qf_target")):
            for k, v in s[group].items():
                out[prefix + k] = v.clone()
        return out


def _init_critics(shapes, generator: torch.Generator) -> Dict[str, torch.Tensor]:
    """Linear: torch's default init; LayerNorm: weight 1, bias 0"""
    linear = OrderedDict((k, s) for k, s in shapes.items() if len(shapes[k.rsplit(".", 1)[0] + ".weight"]) == 2)
    out = _default_linear_init(linear, generator)
    for k, s in shapes.items():
        if k not in out:
            out[k] = torch.ones(s) if k.endswith(".weight") else torch.zeros(s)
    return out


def build_agent(fabric, cfg: Dict[str, Any], obs_space, action_space, agent_state: Optional[Dict[str, torch.Tensor]] = None,
                ops=None) -> Tuple[DroQAgent, SACPlayer]:
    if int(getattr(fabric, "world_size", 1) or 1) > 1:
        raise NotImplementedError(
            "multi-process DroQ is not supported: the reference's actor step indexes its gathered minibatch with a "
            "single DistributedSampler index (sheeprl/algos/droq/droq.py:108-117) and so trains the actor on one row")
    dropout = float(cfg.algo.critic.get("dropout", 0.0) or 0.0)
    if not 0.0 <= dropout < 1.0:
        raise ValueError(f"algo.critic.dropout must be in [0, 1), got {dropout}")
    act_dim = int(math.prod(action_space.shape))
    obs_dim = int(sum(math.prod(obs_space[k].shape) for k in cfg.algo.mlp_keys.encoder))
    if ops is None:
        from sheeprl_b200.lib import CudaOps

        ops = CudaOps()

    def opt(o):
        target = str(o.get("_target_", "torch.optim.Adam"))
        if not target.endswith("Adam"):
            raise NotImplementedError(f"optimizer {target}: the fused update kernel implements torch.optim.Adam")
        return {"lr": float(o.lr), "eps": float(o.eps), "betas": tuple(o.get("betas", (0.9, 0.999))),
                "weight_decay": float(o.get("weight_decay", 0) or 0)}

    eng = DroQEngine(obs_dim, act_dim, int(cfg.algo.actor.hidden_size), int(cfg.algo.critic.hidden_size),
                     int(cfg.algo.critic.n), int(cfg.algo.get("per_rank_batch_size", 256)), float(cfg.algo.gamma),
                     float(cfg.algo.tau), float(cfg.algo.alpha.alpha), dropout, action_space.low, action_space.high,
                     opt(cfg.algo.actor.optimizer), opt(cfg.algo.critic.optimizer), opt(cfg.algo.alpha.optimizer),
                     fabric.device, ops, seed=int(cfg.get("seed", 0) or 0))
    g = torch.Generator().manual_seed(int(cfg.get("seed", 0) or 0))
    eng.actor.load(_default_linear_init(eng.actor.shapes, g))
    eng.qf.load(_init_critics(eng.qf.shapes, g))
    eng.qf_target.load(eng.qf.state_dict())
    agent = DroQAgent(eng)
    if agent_state:
        agent.load_state_dict(agent_state)
    return agent, SACPlayer(eng)
