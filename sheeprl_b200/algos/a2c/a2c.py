"""`train()` of A2C on the CUDA engine — the reference's signature and side effects (sheeprl/algos/a2c/a2c.py:26-114):
one epoch of minibatches drawn by the same torch samplers (RandomSampler / DistributedSampler + BatchSampler, identical
index streams under the same seed), their gradients summed, one clip + optimizer step, parameters and optimizer state
updated in place, two `aggregator.update` calls per minibatch.  The whole call is one `A2CEngine.train` pass
(engine.py); the optimizer is `B200RMSprop` (torch.optim.RMSprop, configs/optim/rmsprop.yaml) or `B200Adam`."""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence

import torch

from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import B200Adam
from sheeprl_b200.algos.ppo.agent import gather_obs
from sheeprl_b200.algos.ppo.ppo import minibatch_indices
from sheeprl_b200.utils.registry import register_algorithm

METRIC_ORDER = ("Loss/policy_loss", "Loss/value_loss")       # a2c.py:112-114: no entropy metric


class B200RMSprop(torch.optim.Optimizer):
    """Handle standing where the reference passes a `torch.optim.RMSprop`.  The update itself is the fused
    clip+RMSprop kernel inside the engine; this object is a real `torch.optim.Optimizer` (schedulers such as the
    reference's `PolynomialLR`, a2c.py:258-264, attach to it, and the engine reads `param_groups[0]` before every fused
    step) whose `state_dict()` has torch's RMSprop layout for the reference agent's parameter list (one entry per
    reference parameter, in `agent.parameters()` order and shape), so checkpoints round-trip with torch's optimizer.
    Its `params` are stand-ins of those shapes; the live parameters are the engine's flat group.

    State in the flat group: square_avg -> exp_avg_sq, momentum_buffer -> exp_avg (momentum > 0), grad_avg -> the
    group's grad_avg buffer (centered)."""

    def __init__(self, engine, lr: float = 1e-2, alpha: float = 0.99, eps: float = 1e-8, weight_decay: float = 0,
                 momentum: float = 0, centered: bool = False, capturable: bool = False, foreach=None,
                 maximize: bool = False, differentiable: bool = False):
        for k, v in (("maximize", maximize), ("differentiable", differentiable), ("capturable", capturable)):
            if v:
                raise NotImplementedError(f"RMSprop({k}=True) is not supported by the fused RMSprop kernel")
        if min(float(alpha), float(eps), float(momentum), float(weight_decay)) < 0:
            raise ValueError(f"invalid RMSprop hyper-parameters: alpha={alpha} eps={eps} momentum={momentum} "
                             f"weight_decay={weight_decay}")
        self.engine, self.group = engine, engine.group
        shapes = engine.reference_shapes()
        # the reference registers each action head's weight and bias together, after everything else (ppo/agent.py)
        heads = sorted((k for k in shapes if k.startswith("actor.actor_heads.")),
                       key=lambda k: (int(k.split(".")[2]), k.endswith(".bias")))
        self.names = [k for k in shapes if not k.startswith("actor.actor_heads.")] + heads
        super().__init__([torch.zeros(shapes[n]) for n in self.names],
                         dict(lr=lr, momentum=momentum, alpha=alpha, eps=eps, centered=centered,
                              weight_decay=weight_decay, capturable=False, foreach=foreach, maximize=False,
                              differentiable=False))
        self.group.optimizer = self

    @property
    def lr(self) -> float:
        return float(self.param_groups[0]["lr"])

    def zero_grad(self, set_to_none: bool = True):  # gradients live in the engine's flat buffer
        return None

    def step(self, closure=None):
        raise RuntimeError("B200RMSprop.step() is fused into the engine's train step")

    def _buffers(self):
        """torch's state names -> the flat buffers that hold them"""
        pg, g = self.param_groups[0], self.group
        out = {"square_avg": g.exp_avg_sq}
        if pg["momentum"] > 0:
            out["momentum_buffer"] = g.exp_avg
        if pg["centered"]:
            out["grad_avg"] = g.alloc_grad_avg()
        return out

    def state_dict(self) -> Dict[str, Any]:
        state = {}
        if self.group.step > 0:
            ref = {k: self.engine.export_reference_state(self.group._views(buf)) for k, buf in self._buffers().items()}
            for i, n in enumerate(self.names):
                state[i] = {"step": torch.tensor(float(self.group.step))}
                state[i].update({k: v[n] for k, v in ref.items()})
        pg = {k: val for k, val in self.param_groups[0].items() if k != "params"}
        return {"state": state, "param_groups": [dict(pg, params=list(range(len(self.names))))]}

    def load_state_dict(self, sd: Dict[str, Any]):
        n_saved = len(sd["param_groups"][0]["params"]) if sd.get("param_groups") else len(self.names)
        if n_saved != len(self.names):
            raise ValueError(f"optimizer state holds {n_saved} parameters, this agent has {len(self.names)}: states of "
                             "a different parameter layout are not interchangeable")
        if sd.get("param_groups"):
            for k in ("lr", "momentum", "alpha", "eps", "centered", "weight_decay"):
                if k in sd["param_groups"][0]:
                    self.param_groups[0][k] = sd["param_groups"][0][k]
        states = sd["state"]
        if not states:
            self.group.step = 0
            self.group.step_t.fill_(0)
            return
        if set(states) != set(range(len(self.names))):
            raise ValueError("optimizer state covers only some parameters; the fused kernel keeps one state per group")
        steps = {int(st["step"]) for st in states.values()}
        if len(steps) > 1:
            raise ValueError("per-parameter RMSprop steps differ; the fused kernel keeps one step per group")
        with torch.no_grad():
            for k, buf in self._buffers().items():
                if any(k not in st for st in states.values()):
                    raise ValueError(f"optimizer state has no {k!r} for the configured RMSprop")
                internal = self.engine.internal_state({n: states[i][k] for i, n in enumerate(self.names)})
                views = self.group._views(buf)
                for n, v in internal.items():
                    if tuple(v.shape) != tuple(views[n].shape):
                        raise ValueError(f"optimizer state of {n} has shape {tuple(v.shape)}, expected {tuple(views[n].shape)}")
                    views[n].copy_(v)
        self.group.step = steps.pop()
        self.group.step_t.fill_(self.group.step)


def make_optimizer(agent, cfg=None):
    """the handle `hydra.utils.instantiate(cfg.algo.optimizer, params=agent.parameters())` gives the reference's main"""
    e = agent._b200_engine
    o = dict(e.opt)
    if o.pop("name") == "adam":
        return B200Adam(e.group, list(e.group.shapes), o["lr"], o["eps"], o["betas"])
    return B200RMSprop(e, **o)


def train(fabric, agent, optimizer, data: Dict[str, torch.Tensor], aggregator, cfg: Dict[str, Any],
          index_batches: Optional[Sequence[Sequence[int]]] = None) -> None:
    """data: flat `[N, ...]` tensors on `fabric.device` with the keys the reference passes (a2c.py:366-381): the
    observation keys (image raw 0..255, float32 or uint8), actions, values, returns, advantages (logprobs and the
    other rollout keys are accepted and not read).  `index_batches` (extra, optional): explicit minibatch index lists
    for parity tests."""
    eng = getattr(agent, "_b200_engine", None)
    if eng is None:
        raise TypeError("train() needs the agent returned by sheeprl_b200.algos.a2c.agent.build_agent")
    for k in ("ent_coef", "vf_coef"):                    # read inside the reference's train() on every call
        eng.hp[k] = float(cfg.algo[k])
    d = {k: data[k] for k in ("actions", "values", "returns", "advantages")}
    d = {k: (v if v.dtype == torch.float32 else v.float()).contiguous() for k, v in d.items()}
    rgb, state = gather_obs(eng.spec, data)
    if rgb is not None:
        d["rgb"] = rgb
    if state is not None:
        d["state"] = state
    n_rows = d["actions"].shape[0]
    it = index_batches if index_batches is not None else minibatch_indices(n_rows, fabric, cfg, epochs=1)
    log = aggregator is not None and not aggregator.disabled

    def on_minibatch(losses):
        if log:
            for i, k in enumerate(METRIC_ORDER):
                aggregator.update(k, losses[i])

    eng.train(d, it, on_minibatch)


def _optimizer_factory(agents):
    """`hydra.utils.instantiate(cfg.algo.optimizer, params=agent.parameters())` -> the fused handle of the agent's
    flat group: torch.optim.RMSprop (A2C's default) or torch.optim.Adam"""
    from sheeprl_b200.utils.delegate import group_of

    def make(config, params):
        if not agents:
            return None
        e = agents[-1]._b200_engine
        if group_of(params, {"agent": e.group}) is None:
            return None
        target = str(config.get("_target_", "torch.optim.RMSprop"))
        name = target.rsplit(".", 1)[-1]
        kw = {k: v for k, v in dict(config).items() if not k.startswith("_")}
        if name == "RMSprop":
            return B200RMSprop(e, **kw)
        if name == "Adam":
            return B200Adam(e.group, list(e.group.shapes), float(kw["lr"]), float(kw.get("eps", 1e-8)),
                            tuple(kw.get("betas", (0.9, 0.999))), float(kw.get("weight_decay", 0.0) or 0.0))
        raise NotImplementedError(f"optimizer {target}: A2C's fused update kernels implement torch.optim.RMSprop and "
                                  "torch.optim.Adam")

    return make


def reference_substitutions(cfg, agents):
    """names of `sheeprl/algos/a2c/a2c.py` replaced while the reference's `main` runs: build_agent (:182-189) and
    train (:381); the rollout buffer, GAE and the checkpoints stay the reference's code"""
    from sheeprl_b200.algos.a2c import agent as A

    def build_agent(*a, **k):
        out = A.build_agent(*a, **k)
        agents.append(out[0])
        return out

    return {"build_agent": build_agent, "train": train}


@register_algorithm()
def main(fabric, cfg: Dict[str, Any]):
    """Entry point registered for `algo.name=a2c` (sheeprl/cli.py:82-98): the reference's own interaction loop
    (a2c.py:118-440: rollout, GAE, lr annealing, checkpoints) with this package's `build_agent` / `train` / optimizer
    handle."""
    from sheeprl_b200.utils.delegate import run_reference_main

    agents = []
    return run_reference_main("sheeprl.algos.a2c.a2c", fabric, cfg, reference_substitutions(cfg, agents),
                              _optimizer_factory(agents))
