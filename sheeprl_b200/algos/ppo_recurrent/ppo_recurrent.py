"""`train()` of recurrent PPO on the CUDA engine — the reference's signature and side effects
(sheeprl/algos/ppo_recurrent/ppo_recurrent.py:31-116): `update_epochs` passes over the padded `[T, S, ...]` sequences in
minibatches of sequences drawn by the same torch samplers (RandomSampler + BatchSampler, host-side index plumbing,
identical streams under the same seed), parameters and Adam state updated in place, three `aggregator.update` calls
per minibatch.  Each minibatch is one `RecurrentPPOEngine.minibatch_step`.

Padded steps drop out through the mask, as in the reference run with torch's distribution argument validation off:
with validation on, the reference itself raises on the all-zero action rows that padding leaves (DESIGN.md)."""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence

import torch
from torch.utils.data import BatchSampler, RandomSampler

from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import B200Adam
from sheeprl_b200.algos.ppo.agent import gather_obs
from sheeprl_b200.utils.registry import register_algorithm

METRIC_ORDER = ("Loss/policy_loss", "Loss/value_loss", "Loss/entropy_loss")
ROLLOUT_KEYS = ("actions", "logprobs", "values", "returns", "advantages", "prev_actions", "prev_hx", "prev_cx", "mask")


def make_optimizer(agent, cfg=None) -> B200Adam:
    e = agent._b200_engine
    return B200Adam(e.group, list(e.group.shapes), e.opt["lr"], e.opt["eps"], e.opt["betas"])


def minibatch_indices(num_sequences: int, cfg):
    """The reference's sampler (ppo_recurrent.py:39-62): one list of sequence indices per minibatch."""
    n = int(cfg.algo.per_rank_num_batches)
    if n > 0:
        batch_size = num_sequences // n
        batch_size = batch_size if batch_size > 0 else num_sequences
    else:
        batch_size = 1
    for _ in range(cfg.algo.update_epochs):
        yield from BatchSampler(RandomSampler(range(num_sequences)), batch_size=batch_size, drop_last=False)


def train(fabric, agent, optimizer, data: Dict[str, torch.Tensor], aggregator, cfg: Dict[str, Any],
          index_batches: Optional[Sequence[Sequence[int]]] = None) -> None:
    """data: `[T, S, ...]` tensors on `fabric.device` with the keys the reference passes (ppo_recurrent.py:438-447):
    the observation keys (images raw 0..255), actions, logprobs, values, returns, advantages, prev_actions, prev_hx,
    prev_cx and the bool `mask` of valid steps.  `index_batches` (extra, optional): explicit lists of sequence
    indices for parity tests."""
    eng = getattr(agent, "_b200_engine", None)
    if eng is None:
        raise TypeError("train() needs the agent returned by sheeprl_b200.algos.ppo_recurrent.agent.build_agent")
    # the reference's main anneals cfg.algo.clip_coef / ent_coef between iterations and reads them inside train()
    for k in ("clip_coef", "ent_coef", "vf_coef"):
        eng.hp[k] = float(cfg.algo[k])
    T, S = data["mask"].shape[:2]
    d = {k: data[k] for k in ROLLOUT_KEYS}
    rgb, state = gather_obs(eng.spec, data)               # per-key tensors -> the encoders' concatenated inputs
    if rgb is not None:
        d["rgb"] = rgb.view(T, S, *rgb.shape[1:])
    if state is not None:
        d["state"] = state.view(T, S, -1)
    it = index_batches if index_batches is not None else minibatch_indices(S, cfg)
    log = aggregator is not None and not aggregator.disabled

    def on_minibatch(losses):
        if log:
            for i, k in enumerate(METRIC_ORDER):
                aggregator.update(k, losses[i])

    eng.train(d, it, on_minibatch)


def _optimizer_factory(agents):
    """`hydra.utils.instantiate(cfg.algo.optimizer, params=agent.parameters())` -> the fused clip+Adam handle.
    configs/algo/ppo_recurrent.yaml selects torch.optim.AdamW with weight_decay 0 (from optim/adam.yaml), which is
    exactly Adam; a nonzero decay is refused."""
    from sheeprl_b200.utils.delegate import group_of

    def make(config, params):
        if not agents:
            return None
        e = agents[-1]._b200_engine
        if group_of(params, {"agent": e.group}) is None:
            return None
        target = str(config.get("_target_", "torch.optim.Adam"))
        name = target.rsplit(".", 1)[-1]
        if name not in ("Adam", "AdamW"):
            raise NotImplementedError(f"optimizer {target}: the fused update kernel implements torch.optim.Adam")
        wd = config.get("weight_decay", None)
        wd = (0.01 if name == "AdamW" else 0.0) if wd is None else float(wd)   # torch's defaults when unset
        if wd != 0.0:
            raise NotImplementedError(f"optimizer {target} with weight_decay={wd}: the fused update kernel implements "
                                      "Adam without weight decay (AdamW with weight_decay 0 is the same update)")
        return B200Adam(e.group, list(e.group.shapes), float(config["lr"]), float(config.get("eps", 1e-8)),
                        tuple(config.get("betas", (0.9, 0.999))))

    return make


def reference_substitutions(cfg, agents):
    """names of `sheeprl/algos/ppo_recurrent/ppo_recurrent.py` replaced while the reference's `main` runs: build_agent
    (:192-199) and train (:447); the rollout buffer and the sequence splitting stay the reference's host code."""
    from sheeprl_b200.algos.ppo_recurrent import agent as A

    def build_agent(*a, **k):
        out = A.build_agent(*a, **k)
        agents.append(out[0])
        return out

    return {"build_agent": build_agent, "train": train}


@register_algorithm()
def main(fabric, cfg: Dict[str, Any]):
    """Entry point registered for `algo.name=ppo_recurrent`: the reference's own interaction loop (rollout with the
    recurrent player, GAE, sequence splitting and padding, annealing, checkpoints) with this package's `build_agent` /
    `train` / Adam handle."""
    from sheeprl_b200.utils.delegate import run_reference_main

    agents = []
    return run_reference_main("sheeprl.algos.ppo_recurrent.ppo_recurrent", fabric, cfg,
                              reference_substitutions(cfg, agents), _optimizer_factory(agents))
