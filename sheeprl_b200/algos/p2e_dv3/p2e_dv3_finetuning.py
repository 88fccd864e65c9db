"""Plan2Explore (Dreamer-V3) finetuning phase — reference `sheeprl/algos/p2e_dv3/p2e_dv3_finetuning.py`: its update is
the plain Dreamer-V3 `train()` (imported at :14 there) on the TASK actor / critic of the agent built by
`sheeprl_b200.algos.p2e_dv3.agent.build_agent`; the engine of that agent IS a Dreamer-V3 engine, so the same function
drives it."""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence

import torch

from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import METRIC_ORDER, make_optimizers  # noqa: F401
from sheeprl_b200.engine import DV3Engine
from sheeprl_b200.utils.registry import register_algorithm


def train(fabric, world_model, actor, critic, target_critic, world_optimizer, actor_optimizer, critic_optimizer,
          data: Dict[str, torch.Tensor], aggregator, cfg: Dict[str, Any], is_continuous: bool, actions_dim: Sequence[int],
          moments, noise: Optional[Dict[str, torch.Tensor]] = None) -> None:
    """`dreamer_v3.train` (same signature) on the engine of a Plan2Explore agent: the PLAIN Dreamer-V3 step — world
    model with attached reward / continue heads, task actor and critic — not the exploration step the engine's own
    `train_step` runs."""
    eng = getattr(world_model, "_b200_engine", None)
    if not isinstance(eng, DV3Engine):
        raise TypeError("train() needs the modules returned by sheeprl_b200.algos.p2e_dv3.agent.build_agent")
    if bool(is_continuous) != eng.is_continuous:
        raise ValueError("is_continuous differs from the value build_agent() was called with")
    if moments is not None and getattr(moments, "low", None) is not None and moments.low.data_ptr() != eng.moments_state.data_ptr():
        moments.bind(eng.moments_state)
    DV3Engine.train_step(eng, data, noise)
    if aggregator and not aggregator.disabled:
        md = DV3Engine.metrics_dict(eng)
        for k in METRIC_ORDER:
            aggregator.update(k, md[k])


@register_algorithm()
def main(fabric, cfg: Dict[str, Any], exploration_cfg: Dict[str, Any] | None = None):
    """Entry point for `algo.name=p2e_dv3_finetuning`: the reference's own loop (p2e_dv3_finetuning.py:28-470) with this
    package's `build_agent` / `train` / Adam handles / Moments / replay rings substituted (see dreamer_v3.main)."""
    from sheeprl_b200.algos.dreamer_v3 import utils as U
    from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import _optimizer_factory
    from sheeprl_b200.algos.p2e_dv3 import agent as A
    from sheeprl_b200.utils.delegate import run_reference_main

    engines = []

    def build_agent(*a, **k):
        out = A.build_agent(*a, **k)
        engines.append(out[0]._b200_engine)
        return out

    names = {"build_agent": build_agent, "train": train, "Moments": U.Moments, "prepare_obs": U.prepare_obs}
    if bool(cfg.buffer.get("device_rings", True)):
        from sheeprl_b200.data import buffers as Bf

        Bf.DEFAULTS["device"] = fabric.device
        names.update(EnvIndependentReplayBuffer=Bf.EnvIndependentReplayBuffer, SequentialReplayBuffer=Bf.SequentialReplayBuffer)
    ref = "sheeprl.algos.p2e_dv3.p2e_dv3_finetuning"
    from sheeprl_b200.utils.delegate import _InstantiateProxy, import_reference, substituted

    mod = import_reference(ref)
    subs = dict(names, hydra=_InstantiateProxy(mod.hydra, _optimizer_factory(engines)))
    with substituted(mod, subs):
        return mod.main(fabric, cfg, exploration_cfg) if exploration_cfg is not None else mod.main(fabric, cfg)
