"""`build_agent` for A2C on the CUDA engine — the signature and `(agent, player)` tuple of the reference's
`sheeprl.algos.ppo.agent.build_agent`, which A2C uses as is (a2c/a2c.py:14).  The agent and player are PPO's
(`PPOAgent` / `PPOPlayer`, reference state-dict keys and shapes); the engine is `A2CEngine`, whose update is A2C's."""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence, Tuple

import torch

from sheeprl_b200.algos.a2c.engine import A2CEngine
from sheeprl_b200.algos.ppo.agent import PPOAgent, PPOPlayer, _attach_if_distributed, default_init, spec_from_cfg

REDUCTIONS = ("mean", "sum")


def hp_from_cfg(cfg) -> dict:
    """A2C's hyper-parameters (configs/algo/a2c.yaml); it has no clip_coef / clip_vloss"""
    a = cfg.algo
    red = str(a.loss_reduction).lower()
    if red not in REDUCTIONS:
        # the reference's train() cannot run with it either: "none" leaves an unreduced loss that fabric.backward
        # refuses, anything else raises in policy_loss (a2c/loss.py:24-32)
        raise ValueError(f"loss_reduction must be one of {REDUCTIONS} for A2C, got {a.loss_reduction!r}")
    return dict(vf_coef=float(a.vf_coef), ent_coef=float(a.ent_coef),
                normalize_advantages=bool(a.get("normalize_advantages", False)),
                max_grad_norm=float(a.max_grad_norm), loss_reduction=red)


def opt_from_cfg(cfg) -> dict:
    """the update `A2CEngine` takes before an optimizer handle is attached: torch's defaults for what the config
    leaves unset (configs/optim/rmsprop.yaml, adam.yaml)"""
    o = cfg.algo.optimizer
    name = str(o.get("_target_", "torch.optim.RMSprop")).rsplit(".", 1)[-1]
    if name not in ("RMSprop", "Adam"):
        raise NotImplementedError(f"optimizer {o.get('_target_')}: A2C's fused update kernels implement "
                                  "torch.optim.RMSprop and torch.optim.Adam")
    if name == "Adam":
        return {"name": "adam", "lr": float(o.lr), "eps": float(o.get("eps", 1e-8)),
                "betas": tuple(o.get("betas", (0.9, 0.999))), "weight_decay": float(o.get("weight_decay", 0) or 0)}
    return {"name": "rmsprop", "lr": float(o.lr), "alpha": float(o.get("alpha", 0.99)), "eps": float(o.get("eps", 1e-8)),
            "weight_decay": float(o.get("weight_decay", 0) or 0), "momentum": float(o.get("momentum", 0) or 0),
            "centered": bool(o.get("centered", False))}


def build_agent(fabric, actions_dim: Sequence[int], is_continuous: bool, cfg: Dict[str, Any], obs_space,
                agent_state: Optional[Dict[str, torch.Tensor]] = None, ops=None) -> Tuple[PPOAgent, PPOPlayer]:
    if ops is None:
        from sheeprl_b200.lib import CudaOps

        ops = CudaOps()
    spec = spec_from_cfg(cfg, actions_dim, is_continuous, obs_space)
    eng = A2CEngine(spec, hp_from_cfg(cfg), opt_from_cfg(cfg), fabric.device, ops, seed=int(cfg.get("seed", 0) or 0))
    g = torch.Generator().manual_seed(int(cfg.get("seed", 0) or 0))
    ortho = "feature_extractor." if cfg.algo.encoder.get("ortho_init", False) else None
    eng.load_reference_state(default_init(eng.reference_shapes(), g, ortho))
    _attach_if_distributed(fabric, eng)
    agent = PPOAgent(eng)
    if agent_state:
        agent.load_state_dict(agent_state)
    return agent, PPOPlayer(eng)
