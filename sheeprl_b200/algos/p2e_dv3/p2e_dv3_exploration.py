"""Plan2Explore (Dreamer-V3) exploration `train()` on the B200 engine — the reference's positional signature and side
effects (`sheeprl/algos/p2e_dv3/p2e_dv3_exploration.py:41-520`): every module / optimiser state / Moments buffer updated
in place, the same `aggregator.update` keys.  The body is one `P2EDV3Engine.train_step`."""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence

import torch

from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import B200Adam
from sheeprl_b200.utils.registry import register_algorithm


def make_optimizers(engine, cfg):
    """(world, actor_task, critic_task, ensembles, actor_exploration) handles + one per exploration critic, in torch's
    `Optimizer.state_dict()` layout.  The ensembles' handle covers the last member (the only clipped one) — the other
    members' Adam state lives in `engine.ens_rest`."""
    a = cfg.algo
    mk = lambda g, o: B200Adam(g, list(g.shapes), float(o.lr), float(o.eps), tuple(o.betas), float(o.weight_decay))  # noqa
    critics = {k: mk(c["group"], a.critic.optimizer) for k, c in engine.critics_expl.items()}
    return (mk(engine.wm, a.world_model.optimizer), mk(engine.actor, a.actor.optimizer), mk(engine.critic, a.critic.optimizer),
            mk(engine.ens_last, a.ensembles.optimizer), mk(engine.actor_expl, a.actor.optimizer), critics)


def train(
    fabric,
    world_model,
    actor_task,
    critic_task,
    target_critic_task,
    world_optimizer,
    actor_task_optimizer,
    critic_task_optimizer,
    data: Dict[str, torch.Tensor],
    aggregator,
    cfg: Dict[str, Any],
    ensembles,
    ensemble_optimizer,
    actor_exploration,
    critics_exploration: Dict[str, Dict[str, Any]],
    actor_exploration_optimizer,
    moments_exploration,
    moments_task,
    is_continuous: bool,
    actions_dim: Sequence[int],
    noise: Optional[Dict[str, torch.Tensor]] = None,
) -> None:
    eng = getattr(world_model, "_b200_engine", None)
    if eng is None or not hasattr(eng, "critics_expl"):
        raise TypeError("train() needs the modules returned by sheeprl_b200.algos.p2e_dv3.agent.build_agent")
    if bool(is_continuous) != eng.is_continuous:
        raise ValueError("is_continuous differs from the value build_agent() was called with")
    bind = lambda m, st: m is not None and m.low.data_ptr() != st.data_ptr() and m.bind(st)  # noqa: E731
    bind(moments_task, eng.moments_state)
    for k, c in eng.critics_expl.items():
        if moments_exploration and k in moments_exploration:
            bind(moments_exploration[k], c["moments_state"])
    eng.train_step(data, noise)
    if aggregator and not aggregator.disabled:
        for k, v in eng.metrics_dict().items():
            aggregator.update(k, v)


@register_algorithm()
def main(fabric, cfg: Dict[str, Any]):
    """Entry point for `algo.name=p2e_dv3_exploration`: the reference's own loop (p2e_dv3_exploration.py:523-1060) with this
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
    return run_reference_main("sheeprl.algos.p2e_dv3.p2e_dv3_exploration", fabric, cfg, names, _optimizer_factory(engines))
