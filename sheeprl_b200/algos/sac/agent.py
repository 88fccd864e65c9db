"""`build_agent` for the B200 SAC engine — same signature / return tuple as the reference
(`sheeprl/algos/sac/agent.py:317-371`).

`SACAgent` is a parameter container: its tensors are views into the engine's flat HBM groups and its
`state_dict()` keys follow the reference module tree (`_actor.*`, `_qfs.{i}.*`, `_qfs_target.{i}.*`, `_log_alpha`).
The arithmetic of `train()` runs in `SACEngine` kernels; acting (`SACPlayer.forward`) is SURVEY §8f.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Any, Dict, Optional, Tuple

import torch

from sheeprl_b200.algos.sac.engine import SACEngine


def _default_linear_init(shapes, generator: torch.Generator) -> Dict[str, torch.Tensor]:
    """torch.nn.Linear.reset_parameters (kaiming-uniform(a=sqrt 5) == U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight
    and bias): what the reference's un-initialised MLPs start from (sac/agent.py:32-38,77-79)."""
    out, bound = {}, None
    for name, shp in shapes.items():
        if name.endswith(".weight"):
            bound = 1.0 / math.sqrt(shp[1])
        out[name] = (torch.rand(*shp, generator=generator) * 2 - 1) * bound
    return out


class SACAgent:
    """Reference surface used by `sac.main` / checkpoints (sac/agent.py:145-267)."""

    def __init__(self, engine: SACEngine):
        self._b200_engine = engine

    # -- properties the reference exposes
    @property
    def num_critics(self) -> int:
        return self._b200_engine.n

    @property
    def log_alpha(self) -> torch.Tensor:
        return self._b200_engine.alpha.views["log_alpha"]

    @property
    def alpha(self) -> float:
        return float(self.log_alpha.exp().item())

    @property
    def target_entropy(self) -> torch.Tensor:
        return torch.tensor(self._b200_engine.target_entropy, device=self._b200_engine.device)

    def qfs_target_ema(self) -> None:
        e = self._b200_engine
        e.ops.ema(e.qf_target.flat, e.qf.flat, e.tau)

    # -- checkpoints: the reference's key layout
    def state_dict(self) -> "OrderedDict[str, torch.Tensor]":
        s = self._b200_engine.export_reference_state()
        out = OrderedDict()
        for k, v in s["actor"].items():
            out[f"_actor.{k}"] = v
        out["_actor.action_scale"] = self._b200_engine.scale.clone()
        out["_actor.action_bias"] = self._b200_engine.abias.clone()
        for k, v in s["qf"].items():
            out[f"_qfs.{k}"] = v
        for k, v in s["qf_target"].items():
            out[f"_qfs_target.{k}"] = v
        out["_log_alpha"] = s["log_alpha"]["log_alpha"]
        return out

    def load_state_dict(self, state: Dict[str, torch.Tensor]) -> None:
        strip = lambda k: k.replace("_forward_module.", "").replace("module.", "", 1) if k.startswith("module.") else k.replace("_forward_module.", "")  # noqa: E731,E501
        grp = {"_actor.": {}, "_qfs.": {}, "_qfs_target.": {}}
        for k, v in state.items():
            k = strip(k)
            for p, d in grp.items():
                if k.startswith(p):
                    d[k[len(p):]] = v
        self._b200_engine.load_reference_state(grp["_actor."], grp["_qfs."], grp["_qfs_target."], state["_log_alpha"])

    def forward(self, *a, **k):
        raise RuntimeError("the B200 SACAgent has no forward(): the update runs in SACEngine kernels")


class SACPlayer:
    """Acting path (reference: sac/agent.py:270-314): tanh-Normal sample (or tanh(mean) when greedy) from the trainer's
    actor parameters — the engine's flat group is shared, so there is nothing to tie or copy."""

    def __init__(self, engine: SACEngine):
        self.engine = engine
        self._bufs = {}

    @torch.no_grad()
    def get_actions(self, obs: torch.Tensor, greedy: bool = False) -> torch.Tensor:
        e, o = self.engine, self.engine.ops
        x = obs.reshape(-1, e.O).float().contiguous()
        E = x.shape[0]
        if E not in self._bufs:
            f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=e.device)  # noqa: E731
            self._bufs[E] = (e.pi.acts(E, grads=False), f(1, E, 2 * e.A), f(E, e.A), f(E), f(E, e.A),
                             torch.zeros(1, dtype=torch.int32, device=e.device))
        acts, head, eps, logp, act, ctr = self._bufs[E]
        e.pi.forward(x.unsqueeze(0), acts, head)
        if greedy:
            eps.zero_()                                       # x_t = mean  ->  tanh(mean) * scale + bias
        else:
            o.increment(ctr)
            o.fill_normal(eps.view(-1), e.rng_seed + 1, 7, ctr)
        o.sac_sample_fwd(head[0], eps, e.scale, e.abias, act, logp)
        return act.clone().reshape(*obs.shape[:-1], e.A)

    __call__ = forward = get_actions

    def eval(self):  # the reference's test loop (sac/utils.py:test) switches the player to inference mode
        return self


def build_agent(fabric, cfg: Dict[str, Any], obs_space, action_space, agent_state: Optional[Dict[str, torch.Tensor]] = None,
                ops=None) -> Tuple[SACAgent, SACPlayer]:
    act_dim = int(math.prod(action_space.shape))
    obs_dim = int(sum(math.prod(obs_space[k].shape) for k in cfg.algo.mlp_keys.encoder))
    if ops is None:
        from sheeprl_b200.lib import CudaOps

        ops = CudaOps()

    def opt(o):
        return {"lr": float(o.lr), "eps": float(o.eps), "betas": tuple(o.get("betas", (0.9, 0.999))),
                "weight_decay": float(o.get("weight_decay", 0) or 0)}

    eng = SACEngine(obs_dim, act_dim, int(cfg.algo.actor.hidden_size), int(cfg.algo.critic.hidden_size),
                    int(cfg.algo.critic.n), int(cfg.algo.get("per_rank_batch_size", 256)), float(cfg.algo.gamma),
                    float(cfg.algo.tau), float(cfg.algo.alpha.alpha), action_space.low, action_space.high,
                    opt(cfg.algo.actor.optimizer), opt(cfg.algo.critic.optimizer), opt(cfg.algo.alpha.optimizer),
                    fabric.device, ops, seed=int(cfg.get("seed", 0) or 0))
    g = torch.Generator().manual_seed(int(cfg.get("seed", 0) or 0))
    eng.actor.load(_default_linear_init(eng.actor.shapes, g))
    eng.qf.load(_default_linear_init(eng.qf.shapes, g))
    eng.qf_target.load(eng.qf.state_dict())
    if int(getattr(fabric, "world_size", 1) or 1) > 1:
        # the reference wraps actor / critics in DDP here (sac/agent.py:351-360, fabric.setup_module)
        import torch.distributed as dist

        from sheeprl_b200.parallel import attach_data_parallel

        if not dist.is_initialized():
            raise RuntimeError("fabric.world_size > 1 but torch.distributed is not initialised (launch through Fabric / torchrun)")
        attach_data_parallel(eng)
    agent = SACAgent(eng)
    if agent_state:
        agent.load_state_dict(agent_state)
    return agent, SACPlayer(eng)
