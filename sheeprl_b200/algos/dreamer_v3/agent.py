"""`build_agent` for the B200 Dreamer-V3 engine — same signature / return tuple as the reference
(`sheeprl/algos/dreamer_v3/agent.py:935-1236`).

The returned `world_model`, `actor`, `critic`, `target_critic` are `nn.Module` trees whose parameters
are *views into the engine's flat HBM buffers* and whose `state_dict()` keys/shapes are exactly the
reference's (SURVEY.md §8b), so checkpoints interchange.  The arithmetic lives in
`sheeprl_b200.engine.DV3Engine` (CUDA kernels through the C-ABI); these modules have no `forward`.
"""
from __future__ import annotations

import math
from typing import Any, Dict, Mapping, Optional, Sequence, Tuple

import torch
from torch import nn

from sheeprl_b200.algos.dreamer_v3.player import PlayerDV3
from sheeprl_b200.engine import DV3Engine
from sheeprl_b200.params import FlatGroup

# kernel binding used when build_agent() is called without `ops` (the reference's main never passes one): None -> the CUDA
# library.  Tests on a GPU-less host point this at the torch test double.
DEFAULT_OPS = None


class ParamTree(nn.Module):
    """Nested modules mirroring dotted state-dict names; leaves are nn.Parameters aliasing `views`."""

    def __init__(self, views: Mapping[str, torch.Tensor], requires_grad: bool = False):
        super().__init__()
        for name, t in views.items():
            node = self
            parts = name.split(".")
            for p in parts[:-1]:
                if p not in node._modules:
                    node.add_module(p, _Node())
                node = node._modules[p]
            node.register_parameter(parts[-1], nn.Parameter(t, requires_grad=requires_grad))

    @property
    def module(self):  # the reference reaches through fabric wrappers with `.module`
        return self

    def forward(self, *a, **k):
        raise RuntimeError("B200 parameter trees have no forward(): the arithmetic runs in DV3Engine kernels")


class _Node(nn.Module):
    pass


class WorldModel(ParamTree):
    """Parameter container for the world model (reference: dreamer_v2/agent.py:707-732)."""


def _trunc_normal(shape, fan_in, fan_out, g, limit_in_std):
    std = math.sqrt(1.0 / ((fan_in + fan_out) / 2.0)) / 0.87962566103423978
    t = torch.empty(*shape)
    lim = 2.0 * std if limit_in_std else 2.0
    nn.init.trunc_normal_(t, 0.0, std, -lim, lim, generator=g)
    return t


def _uniform(shape, fan_in, fan_out, scale, g):
    if scale == 0.0:
        return torch.zeros(*shape)
    lim = math.sqrt(3 * scale / ((fan_in + fan_out) / 2.0))
    return (torch.rand(*shape, generator=g) * 2 - 1) * lim


def initial_state(group: FlatGroup, outscale: Dict[str, float], generator: torch.Generator) -> Dict[str, torch.Tensor]:
    """Reference initialisation (dreamer_v3/utils.py:143-186 `init_weights` / `uniform_init_weights`,
    hafner_initialization agent.py:1170-1180): truncated-normal fan-avg for Linear / conv weights, ones/zeros
    for LayerNorm, zero biases; `outscale[name]` switches a weight to the uniform(out-scale) init."""
    out = {}
    for name, shp in group.shapes.items():
        if name.endswith(".bias") or name == "rssm.initial_recurrent_state":
            out[name] = torch.zeros(*shp)
        elif len(shp) == 1:
            out[name] = torch.ones(*shp)                      # LayerNorm weight
        elif len(shp) == 4:
            # Conv2d [Cout,Cin,4,4] / ConvTranspose2d [Cin,Cout,4,4]: fan = 16 * channels either way
            if name in outscale:                              # never the case for convs in the reference except
                out[name] = _uniform(shp, 16 * shp[0], 16 * shp[1], outscale[name], generator)
            else:
                out[name] = _trunc_normal(shp, 16 * shp[0], 16 * shp[1], generator, False)
        else:
            o, i = shp
            out[name] = (_uniform(shp, i, o, outscale[name], generator) if name in outscale
                         else _trunc_normal(shp, i, o, generator, True))
    return out


def build_agent(
    fabric,
    actions_dim: Sequence[int],
    is_continuous: bool,
    cfg: Dict[str, Any],
    obs_space,
    world_model_state: Optional[Dict[str, torch.Tensor]] = None,
    actor_state: Optional[Dict[str, torch.Tensor]] = None,
    critic_state: Optional[Dict[str, torch.Tensor]] = None,
    target_critic_state: Optional[Dict[str, torch.Tensor]] = None,
    ops=None,
) -> Tuple[WorldModel, ParamTree, ParamTree, ParamTree, PlayerDV3]:
    """ops (extra, optional): the kernel binding; default `sheeprl_b200.lib.CudaOps` (tests on a GPU-less host pass the
    torch test double)."""
    cnn_keys, mlp_keys = list(cfg.algo.cnn_keys.encoder or []), list(cfg.algo.mlp_keys.encoder or [])
    cnn_dims = {k: int(math.prod(obs_space[k].shape[:-2])) for k in cnn_keys}       # agent.py:984, 1070
    in_channels = sum(cnn_dims.values()) if cnn_keys else 3
    mlp_dims = {k: int(obs_space[k].shape[0]) for k in mlp_keys}          # agent.py:1002
    eng = DV3Engine(cfg, actions_dim, in_channels=in_channels, device=fabric.device, ops=ops if ops is not None else DEFAULT_OPS,
                    is_continuous=is_continuous, mlp_dims=mlp_dims, cnn_dims=cnn_dims)
    seed, rank = int(cfg.get("seed", 0) or 0), int(getattr(fabric, "global_rank", 0) or 0)
    eng.rng_seed = (seed * 1000003 + rank) & 0x7FFFFFFF        # sampling noise follows cfg.seed; ranks draw different streams
    if int(getattr(fabric, "world_size", 1) or 1) > 1:
        # the reference wraps every model in DDP here (agent.py:1205-1214, fabric.setup_module) and reduces inside
        # fabric.backward; the engine's equivalent is one all-reduce per flat gradient + the Moments all-gather
        import torch.distributed as dist

        from sheeprl_b200.parallel import attach_data_parallel

        if not dist.is_initialized():
            raise RuntimeError("fabric.world_size > 1 but torch.distributed is not initialised (launch through Fabric / torchrun)")
        attach_data_parallel(eng)
    g = torch.Generator().manual_seed(int(cfg.get("seed", 0) or 0))
    nh = cfg.algo.mlp_layers
    haf = bool(cfg.algo.hafner_initialization)
    last_dec = f"observation_model.cnn_decoder.model.2._model.{3 * (eng.stages - 1)}.weight"
    wm_scale = {"rssm.transition_model._model.3.weight": 1.0, "rssm.representation_model._model.3.weight": 1.0,
                f"reward_model._model.{3 * nh}.weight": 0.0, f"continue_model._model.{3 * nh}.weight": 1.0} if haf else {}
    if haf:
        # one head per decoded vector key (agent.py:1177-1178)
        wm_scale.update({f"observation_model.mlp_decoder.heads.{i}.weight": 1.0 for i in range(len(eng.dec_vec_keys))})
    wm_init = initial_state(eng.wm, wm_scale, g)
    if haf and eng.has_cnn_dec:
        # `uniform_init_weights` only touches nn.Linear / nn.LayerNorm (dreamer_v3/utils.py:170-186): applied to the
        # last ConvTranspose2d (agent.py:1180) it is a no-op, so that layer keeps its truncated-normal init.
        assert last_dec in wm_init
    eng.wm.load(wm_init if world_model_state is None else world_model_state)
    n_heads = 1 if is_continuous else len(actions_dim)
    ac_scale = {f"mlp_heads.{i}.weight": 1.0 for i in range(n_heads)} if haf else {}
    eng.actor.load(initial_state(eng.actor, ac_scale, g) if actor_state is None else actor_state)
    cr_scale = {f"_model.{3 * nh}.weight": 0.0} if haf else {}
    eng.critic.load(initial_state(eng.critic, cr_scale, g) if critic_state is None else critic_state)
    eng.target.load(eng.critic.state_dict() if target_critic_state is None else target_critic_state)

    world_model = WorldModel(eng.wm.views)
    actor, critic, target_critic = ParamTree(eng.actor.views), ParamTree(eng.critic.views), ParamTree(eng.target.views)
    for m in (world_model, actor, critic, target_critic):
        object.__setattr__(m, "_b200_engine", eng)
    player = PlayerDV3(eng, cfg.env.num_envs)
    player.rng_seed = (eng.rng_seed ^ 0x5EED) & 0x7FFFFFFF
    return world_model, actor, critic, target_critic, player
