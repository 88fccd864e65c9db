"""`train()` of PPO on the B200 engine — the reference's signature and side effects
(sheeprl/algos/ppo/ppo.py:30-102): `update_epochs` passes over the rollout in minibatches drawn by the same
torch samplers (RandomSampler / DistributedSampler + BatchSampler — host-side index plumbing, identical streams
under the same seed), parameters and Adam state updated in place, three `aggregator.update` calls per minibatch.
Each minibatch is one `PPOEngine.minibatch_step` (csrc/ppo.cu + csrc/mlp.cu + replay gather)."""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence

import torch
from torch.utils.data import BatchSampler, DistributedSampler, RandomSampler

from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import B200Adam
from sheeprl_b200.algos.ppo.agent import gather_obs
from sheeprl_b200.utils.registry import register_algorithm

METRIC_ORDER = ("Loss/policy_loss", "Loss/value_loss", "Loss/entropy_loss")


def make_optimizer(agent, cfg=None) -> B200Adam:
    e = agent._b200_engine
    return B200Adam(e.group, list(e.group.shapes), e.opt["lr"], e.opt["eps"], e.opt["betas"])


def minibatch_indices(n_rows: int, fabric, cfg, epochs: Optional[int] = None):
    """The reference's sampler stack (ppo.py:39-56), yielding one list of row indices per minibatch over `epochs`
    passes (default cfg.algo.update_epochs; A2C makes one, a2c.py:40-55)."""
    indexes = list(range(n_rows))
    if cfg.buffer.share_data:
        sampler = DistributedSampler(indexes, num_replicas=fabric.world_size, rank=fabric.global_rank, shuffle=True,
                                     seed=cfg.seed)
    else:
        sampler = RandomSampler(indexes)
    batches = BatchSampler(sampler, batch_size=cfg.algo.per_rank_batch_size, drop_last=False)
    for epoch in range(cfg.algo.update_epochs if epochs is None else epochs):
        if cfg.buffer.share_data:
            batches.sampler.set_epoch(epoch)
        yield from batches


def train(fabric, agent, optimizer, data: Dict[str, torch.Tensor], aggregator, cfg: Dict[str, Any],
          index_batches: Optional[Sequence[Sequence[int]]] = None) -> None:
    """data: flat `[N, ...]` tensors on `fabric.device` with the keys the reference passes (ppo.py:399-407): the
    observation keys (image raw 0..255, float32 or uint8), actions, logprobs, values, returns, advantages.
    `index_batches` (extra, optional): explicit minibatch index lists for parity tests."""
    eng = getattr(agent, "_b200_engine", None)
    if eng is None:
        raise TypeError("train() needs the agent returned by sheeprl_b200.algos.ppo.agent.build_agent")
    s = eng.spec
    # the reference's main anneals cfg.algo.clip_coef / ent_coef between iterations (ppo.py:418-425) and reads them inside
    # train(): take the current values on every call
    for k in ("clip_coef", "ent_coef", "vf_coef"):
        eng.hp[k] = float(cfg.algo[k])
    d = {k: data[k] for k in ("actions", "logprobs", "values", "returns", "advantages")}
    d = {k: (v if v.dtype == torch.float32 else v.float()).contiguous() for k, v in d.items()}
    rgb, state = gather_obs(s, data)                      # per-key tensors -> the encoders' concatenated inputs
    if rgb is not None:
        d["rgb"] = rgb
    if state is not None:
        d["state"] = state
    n_rows = d["actions"].shape[0]
    it = index_batches if index_batches is not None else minibatch_indices(n_rows, fabric, cfg)
    log = aggregator is not None and not aggregator.disabled

    def on_minibatch(losses):
        if log:
            for i, k in enumerate(METRIC_ORDER):
                aggregator.update(k, losses[i])

    eng.train(d, it, on_minibatch)


def _optimizer_factory(agents):
    from sheeprl_b200.utils.delegate import group_of

    def make(config, params):
        if not agents:
            return None
        e = agents[-1]._b200_engine
        if group_of(params, {"agent": e.group}) is None:
            return None
        target = str(config.get("_target_", "torch.optim.Adam"))
        if not target.endswith("Adam"):
            raise NotImplementedError(f"optimizer {target}: the fused update kernel implements torch.optim.Adam")
        return B200Adam(e.group, list(e.group.shapes), float(config["lr"]), float(config.get("eps", 1e-8)),
                        tuple(config.get("betas", (0.9, 0.999))), float(config.get("weight_decay", 0.0) or 0.0))

    return make


def reference_substitutions(cfg, agents):
    """names of `sheeprl/algos/ppo/ppo.py` replaced while the reference's `main` runs: build_agent (:174-181), train
    (:373); `ReplayBuffer` stays the reference's host buffer (the rollout is gathered through `fabric.all_gather`)."""
    from sheeprl_b200.algos.ppo import agent as A

    def build_agent(*a, **k):
        out = A.build_agent(*a, **k)
        agents.append(out[0])
        return out

    return {"build_agent": build_agent, "train": train}


@register_algorithm()
def main(fabric, cfg: Dict[str, Any]):
    """Entry point registered for `algo.name=ppo` (sheeprl/cli.py:82-98, 199): the reference's own interaction loop
    (ppo.py:105-430: rollout, GAE, annealing, checkpoints) with this package's `build_agent` / `train` / Adam handle."""
    from sheeprl_b200.utils.delegate import run_reference_main

    agents = []
    return run_reference_main("sheeprl.algos.ppo.ppo", fabric, cfg, reference_substitutions(cfg, agents),
                              _optimizer_factory(agents))
