"""Dreamer-V3 `train()` on the B200 engine — drop-in for `sheeprl/algos/dreamer_v3/dreamer_v3.py:48-357`.

Same positional signature, same side effects (parameters / optimiser state / Moments buffers updated in
place, 13 `aggregator.update` calls, `data["is_first"][0]` forced to 1), but the body is one call into
`DV3Engine.train_step`: ~2.5k hand-written CUDA kernel launches (optionally one CUDA-graph replay), no
autograd, no torch arithmetic.
"""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence

import torch

from sheeprl_b200.engine import DV3Engine
from sheeprl_b200.lib import sync_deterministic
from sheeprl_b200.utils.registry import register_algorithm

METRIC_ORDER = (
    "Loss/world_model_loss", "Loss/observation_loss", "Loss/reward_loss", "Loss/state_loss", "Loss/continue_loss",
    "State/kl", "State/post_entropy", "State/prior_entropy", "Loss/policy_loss", "Loss/value_loss",
    "Grads/world_model", "Grads/actor", "Grads/critic",
)


class B200Adam(torch.optim.Optimizer):
    """Handle standing where the reference passes a `torch.optim.Adam` (dreamer_v3.py:448-457).  The update
    itself is the fused clip+Adam kernel inside the engine; this object is a real `torch.optim.Optimizer` (schedulers
    such as the reference's `PolynomialLR`, ppo.py:236-238, attach to it and the engine reads `param_groups[0]["lr"]`
    before every fused step) whose `state_dict()` has torch's layout, so reference checkpoints round-trip.
    `weight_decay` is torch's L2 term (Dreamer-V2's optimizers default to 1e-6), added to the clipped gradient."""

    def __init__(self, group, names: Sequence[str], lr: float, eps: float, betas=(0.9, 0.999), weight_decay=0.0):
        if not float(weight_decay) >= 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        self.group, self.names = group, list(names)
        super().__init__([group.views[n] for n in self.names],
                         dict(lr=float(lr), betas=tuple(betas), eps=float(eps), weight_decay=float(weight_decay),
                              amsgrad=False))
        group.optimizer = self

    @property
    def lr(self) -> float:
        return float(self.param_groups[0]["lr"])

    @property
    def weight_decay(self) -> float:
        return float(self.param_groups[0]["weight_decay"])

    def zero_grad(self, set_to_none: bool = True):  # gradients live in the engine's flat buffer
        return None

    def step(self, closure=None):
        raise RuntimeError("B200Adam.step() is fused into the engine's train step")

    def state_dict(self) -> Dict[str, Any]:
        m, v = self.group.optimizer_views()
        state = {}
        if self.group.step > 0:
            for i, n in enumerate(self.names):
                state[i] = {"step": torch.tensor(float(self.group.step)), "exp_avg": m[n].detach().clone(),
                            "exp_avg_sq": v[n].detach().clone()}
        pg = {k: val for k, val in self.param_groups[0].items() if k != "params"}
        out = {"state": state, "param_groups": [dict(pg, params=list(range(len(self.names))))]}
        eng = getattr(self, "rng_engine", None)
        if eng is not None:          # Philox position of the sampling noise travels with the world-model optimizer state, so
            out["b200_rng"] = eng.rng_state()      # a resumed run continues the stream (torch's Adam ignores the extra key)
        return out

    def load_state_dict(self, sd: Dict[str, Any]):
        m, v = self.group.optimizer_views()
        n_saved = len(sd["param_groups"][0]["params"]) if sd.get("param_groups") else len(self.names)
        if n_saved != len(self.names):
            raise ValueError(f"optimizer state holds {n_saved} parameters, this group has {len(self.names)}: states of "
                             "a different parameter layout are not interchangeable")
        steps = set()
        with torch.no_grad():
            for i, n in enumerate(self.names):
                st = sd["state"].get(i)
                if st is None:
                    continue
                if tuple(st["exp_avg"].shape) != tuple(m[n].shape):
                    raise ValueError(f"optimizer state of parameter {i} ({n}) has shape {tuple(st['exp_avg'].shape)}, "
                                     f"expected {tuple(m[n].shape)}")
                m[n].copy_(st["exp_avg"])
                v[n].copy_(st["exp_avg_sq"])
                steps.add(int(st["step"]))
        if len(steps) > 1:
            raise ValueError("per-parameter Adam steps differ; the fused kernel keeps one step per group")
        self.group.step = steps.pop() if steps else 0
        self.group.step_t.fill_(self.group.step)
        if sd.get("param_groups"):
            for k in ("lr", "eps", "betas", "weight_decay"):
                if k in sd["param_groups"][0]:
                    self.param_groups[0][k] = sd["param_groups"][0][k]
        eng = getattr(self, "rng_engine", None)
        if eng is not None and "b200_rng" in sd:
            eng.load_rng_state(sd["b200_rng"])


def make_optimizers(engine: DV3Engine, cfg):
    a = cfg.algo
    mk = lambda g, o: B200Adam(g, list(g.shapes), float(o.lr), float(o.eps), tuple(o.betas), float(o.weight_decay))  # noqa
    opts = (mk(engine.wm, a.world_model.optimizer), mk(engine.actor, a.actor.optimizer), mk(engine.critic, a.critic.optimizer))
    opts[0].rng_engine = engine
    return opts


def _engine_of(module) -> DV3Engine:
    eng = getattr(module, "_b200_engine", None)
    if eng is None:
        raise TypeError("train() needs the modules returned by sheeprl_b200.algos.dreamer_v3.agent.build_agent")
    return eng


def train(
    fabric,
    world_model,
    actor,
    critic,
    target_critic,
    world_optimizer,
    actor_optimizer,
    critic_optimizer,
    data: Dict[str, torch.Tensor],
    aggregator,
    cfg: Dict[str, Any],
    is_continuous: bool,
    actions_dim: Sequence[int],
    moments,
    noise: Optional[Dict[str, torch.Tensor]] = None,
) -> None:
    """One Dreamer-V3 update.  `data`: dict of `[T, B, ...]` tensors on `fabric.device` (float32 as the
    reference passes them; the image key may also be uint8).  `noise` (extra, optional): injected Exp(1)
    sampling noise for parity tests; None -> on-device Philox."""
    eng = _engine_of(world_model)
    if bool(is_continuous) != eng.is_continuous:
        raise ValueError("is_continuous differs from the value build_agent() was called with")
    if moments is not None and getattr(moments, "low", None) is not None and moments.low.data_ptr() != eng.moments_state.data_ptr():
        moments.bind(eng.moments_state)
    sync_deterministic(eng.ops)        # before the graph key, which holds the mode
    if noise is None and eng.use_cuda_graph():
        # the whole update as one CUDA-graph replay (sheeprl_b200/graph.py): the batch is copied into the graph's static
        # inputs; the reference's in-place `data["is_first"][0] = 1` (dreamer_v3.py:100) still reaches the caller's tensor
        data["is_first"][0].fill_(1.0)
        eng.step_graph().run(lambda d: eng.train_step(d, None), data, key=eng.graph_key())
    else:
        eng.train_step(data, noise)
    if aggregator and not aggregator.disabled:
        md = eng.metrics_dict()
        for k in METRIC_ORDER:
            aggregator.update(k, md[k])


def _optimizer_factory(engines):
    """`hydra.utils.instantiate(cfg.algo.<model>.optimizer, params=<model>.parameters())` (dreamer_v3.py:448-452) ->
    the fused-Adam handle of the flat group those parameters are views of"""
    from sheeprl_b200.utils.delegate import group_of

    def make(config, params):
        if not engines:
            return None
        eng = engines[-1]
        groups = {"wm": eng.wm, "actor": eng.actor, "critic": eng.critic}
        groups.update(getattr(eng, "extra_groups", lambda: {})())
        name = group_of(params, groups)
        if name is None:
            return None
        target = str(config.get("_target_", "torch.optim.Adam"))
        if not target.endswith("Adam"):
            raise NotImplementedError(f"optimizer {target}: the fused update kernel implements torch.optim.Adam")
        g = groups[name]
        opt = B200Adam(g, list(g.shapes), float(config["lr"]), float(config.get("eps", 1e-8)),
                       tuple(config.get("betas", (0.9, 0.999))), float(config.get("weight_decay", 0.0) or 0.0))
        if name == "wm":
            opt.rng_engine = eng
        return opt

    return make


def reference_substitutions(cfg, engines):
    """Module-level names of `sheeprl/algos/dreamer_v3/dreamer_v3.py` that the B200 package replaces while the
    reference's own `main` runs (dreamer_v3.py:437-447 build_agent, :679-694 train, :459 Moments, :573 prepare_obs,
    :474-480 the replay buffer classes)."""
    from sheeprl_b200.algos.dreamer_v3 import agent as A
    from sheeprl_b200.algos.dreamer_v3 import utils as U

    def build_agent(*a, **k):
        out = A.build_agent(*a, **k)
        engines.append(out[0]._b200_engine)
        return out

    names = {"build_agent": build_agent, "train": train, "Moments": U.Moments, "prepare_obs": U.prepare_obs}
    if bool(cfg.buffer.get("device_rings", True)):
        from sheeprl_b200.data import buffers as Bf

        names.update(EnvIndependentReplayBuffer=Bf.EnvIndependentReplayBuffer,
                     SequentialReplayBuffer=Bf.SequentialReplayBuffer)
    return names


def _bind_buffer_device(fabric):
    """the reference's main builds its buffers without a device argument: the rings default to this rank's GPU"""
    from sheeprl_b200.data import buffers as Bf

    Bf.DEFAULTS["device"] = fabric.device


@register_algorithm()
def main(fabric, cfg: Dict[str, Any]):
    """Entry point registered for `algo.name=dreamer_v3` (looked up and launched by sheeprl/cli.py:82-98, 199).  The
    environment-interaction loop is the reference's own `main` (dreamer_v3.py:361-780), run with this package's
    `build_agent` / `train` / optimizer handles / Moments / device-resident replay rings substituted."""
    from sheeprl_b200.utils.delegate import run_reference_main

    engines = []
    _bind_buffer_device(fabric)
    return run_reference_main("sheeprl.algos.dreamer_v3.dreamer_v3", fabric, cfg, reference_substitutions(cfg, engines),
                              _optimizer_factory(engines))
