"""`train()` of DroQ on the CUDA engine — the reference's signature and side effects
(sheeprl/algos/droq/droq.py:32-164): two replay samples in the reference's order and arguments (so the buffer's host RNG
stream is the reference's), then one `DroQEngine.train_call` for the G critic steps and the actor / temperature step,
parameters, optimizer states and target critics updated in place, and the three losses logged."""
from __future__ import annotations

from typing import Any, Dict, Optional

import torch

from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import B200Adam
from sheeprl_b200.algos.sac.sac import _optimizer_factory
from sheeprl_b200.utils.registry import register_algorithm

METRIC_ORDER = ("Loss/value_loss", "Loss/policy_loss", "Loss/alpha_loss")


def make_optimizers(agent, cfg):
    """(actor_optimizer, qf_optimizer, alpha_optimizer) handles over the engine's flat groups"""
    e = agent._b200_engine
    mk = lambda g, o: B200Adam(g, list(g.shapes), o["lr"], o["eps"], o["betas"], o["weight_decay"])  # noqa: E731
    return mk(e.actor, e.opt["actor"]), mk(e.qf, e.opt["qf"]), mk(e.alpha, e.opt["alpha"])


def _rows(sample: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """[1, rows, ...] buffer samples as float32 [rows, ...] (droq.py:76-82)"""
    return {k: (v if v.dtype == torch.float32 else v.float()).flatten(0, 1) for k, v in sample.items()}


def train(fabric, agent, actor_optimizer, qf_optimizer, alpha_optimizer, rb, aggregator, cfg: Dict[str, Any],
          per_rank_gradient_steps: int, noise: Optional[Dict[str, torch.Tensor]] = None) -> None:
    """G = per_rank_gradient_steps critic steps on one G*B-row sample, then one actor / temperature step on a second
    B-row sample.  `noise` (extra, optional): injected eps_next / eps_cur / masks for parity tests
    (`DroQEngine.train_call`)."""
    eng = getattr(agent, "_b200_engine", None)
    if eng is None:
        raise TypeError("train() needs the agent returned by sheeprl_b200.algos.droq.agent.build_agent")
    if int(getattr(fabric, "world_size", 1) or 1) > 1:
        raise NotImplementedError("multi-process DroQ is not supported (see sheeprl_b200.algos.droq.agent.build_agent)")
    B = int(cfg.algo.per_rank_batch_size)
    if B != eng.B:
        eng.B = B
        eng._alloc()
    dev = eng.device
    critic = _rows(rb.sample_tensors(per_rank_gradient_steps * B, sample_next_obs=cfg.buffer.sample_next_obs,
                                     from_numpy=cfg.buffer.from_numpy))
    actor = _rows(rb.sample_tensors(B, from_numpy=cfg.buffer.from_numpy))
    critic = {k: v.to(dev) for k, v in critic.items()}
    eng.train_call(critic, actor["observations"].to(dev), noise)
    if aggregator and not aggregator.disabled:
        md = eng.metrics_dict()
        for k in METRIC_ORDER:
            aggregator.update(k, md[k])


def reference_substitutions(cfg, agents):
    """names of `sheeprl/algos/droq/droq.py` replaced while the reference's `main` runs: build_agent (:231-233), train
    (:380-390), ReplayBuffer (:259-265)"""
    from sheeprl_b200.algos.droq import agent as A
    from sheeprl_b200.data.buffers import ReplayBuffer

    def build_agent(*a, **k):
        out = A.build_agent(*a, **k)
        agents.append(out[0])
        return out

    return {"build_agent": build_agent, "train": train, "ReplayBuffer": ReplayBuffer}


@register_algorithm()
def main(fabric, cfg: Dict[str, Any]):
    """Entry point registered for `algo.name=droq` (sheeprl/cli.py:82-98, 199): the reference's own interaction loop
    (droq.py:167-463) with this package's `build_agent` / `train` / Adam handles / device replay buffer."""
    from sheeprl_b200.utils.delegate import run_reference_main

    if int(getattr(fabric, "world_size", 1) or 1) > 1:
        raise NotImplementedError("multi-process DroQ is not supported (see sheeprl_b200.algos.droq.agent.build_agent)")
    agents = []
    return run_reference_main("sheeprl.algos.droq.droq", fabric, cfg, reference_substitutions(cfg, agents),
                              _optimizer_factory(agents))
