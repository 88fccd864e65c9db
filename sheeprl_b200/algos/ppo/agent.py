"""`build_agent` for the B200 PPO engine — same signature / return tuple as the reference
(`sheeprl/algos/ppo/agent.py:325-369`).  `PPOAgent` is a parameter container whose `state_dict()` has the
reference's keys and shapes (conv weights [Cout,Cin,k,k], one Linear per action head); the arithmetic of `train()`
runs in `PPOEngine` kernels.  Acting (`PPOPlayer`) is SURVEY §8f."""
from __future__ import annotations

import math
from typing import Any, Dict, Optional, Sequence, Tuple

import torch

from sheeprl_b200.algos.ppo.engine import PPOEngine


def spec_from_cfg(cfg, actions_dim: Sequence[int], is_continuous: bool, obs_space) -> dict:
    """engine spec from the reference's config tree (ppo/agent.py:99-184, configs/algo/ppo.yaml)"""
    a = cfg.algo
    cnn_keys, mlp_keys = list(a.cnn_keys.encoder or []), list(a.mlp_keys.encoder or [])
    dist = str(cfg.distribution.get("type", "auto")).lower()
    if dist not in ("auto", "normal", "tanh_normal", "discrete"):
        raise ValueError("The distribution must be on of: `auto`, `discrete`, `normal` and `tanh_normal`. "
                         f"Found: {dist}")                                            # ppo/agent.py:109-113
    if dist == "discrete" and is_continuous:
        raise ValueError("You have choose a discrete distribution but `is_continuous` is true")
    if dist not in ("discrete", "auto") and not is_continuous:
        raise ValueError("You have choose a continuous distribution but `is_continuous` is false")
    if dist == "auto":
        dist = "normal" if is_continuous else "discrete"
    acts = {str(a.encoder.dense_act), str(a.actor.dense_act), str(a.critic.dense_act)}
    if len(acts) != 1 or acts.pop().rsplit(".", 1)[-1] not in ("Tanh", "ReLU"):
        raise NotImplementedError("dense_act must be torch.nn.Tanh or torch.nn.ReLU, the same for encoder/actor/critic")
    if mlp_keys and int(a.encoder.mlp_layers) == 0:
        raise NotImplementedError("encoder.mlp_layers == 0 (identity vector encoder) is not built")
    if mlp_keys and not a.encoder.mlp_features_dim:
        raise NotImplementedError("encoder.mlp_features_dim must be set")
    cnn = [(k, int(math.prod(obs_space[k].shape[:-2]))) for k in cnn_keys]
    mlp = [(k, int(obs_space[k].shape[0])) for k in mlp_keys]
    return dict(
        cnn_channels=sum(c for _, c in cnn), screen=int(cfg.env.screen_size) if cnn_keys else 0, cnn_keys=cnn,
        mlp_dim=sum(d for _, d in mlp), mlp_keys=mlp,
        dense=int(a.actor.dense_units), layers=int(a.actor.mlp_layers),
        nets={w: (int(a[w].dense_units), int(a[w].mlp_layers)) for w in ("encoder", "actor", "critic")},
        layer_norm={w: bool(a[w].layer_norm) for w in ("encoder", "actor", "critic")},
        cnn_features=int(a.encoder.cnn_features_dim), mlp_features=int(a.encoder.mlp_features_dim or 0),
        actions_dim=tuple(int(x) for x in actions_dim), is_continuous=bool(is_continuous), dist=dist,
        act="tanh" if str(a.actor.dense_act).endswith("Tanh") else "relu")


def obs_key_names(spec: dict):
    """([image keys], [vector keys]) in the order the encoders concatenate them (ppo/agent.py:34-36, 67-69)"""
    cnn = [k for k, _ in spec.get("cnn_keys") or []] or ([spec.get("cnn_key") or "rgb"] if spec["cnn_channels"] else [])
    mlp = [k for k, _ in spec.get("mlp_keys") or []] or ([spec.get("mlp_key") or "state"] if spec["mlp_dim"] else [])
    return cnn, mlp


def gather_obs(spec: dict, data, lead_dims: int = 1):
    """(image tensor [N, C_total, H, W] or None, vector tensor [N, D_total] or None) from a dict of per-key tensors:
    the concatenation the reference's encoders do on every forward, done once here.  A dict that already holds the
    concatenated "rgb" / "state" tensors is accepted as is."""
    cnn, mlp = obs_key_names(spec)
    rgb = state = None
    if cnn:
        if all(k in data for k in cnn):
            parts = [data[k].reshape(-1, *data[k].shape[-3:]) for k in cnn]
        else:
            parts = [data["rgb"].reshape(-1, *data["rgb"].shape[-3:])]
        if any(p.dtype != parts[0].dtype for p in parts) or parts[0].dtype not in (torch.uint8, torch.float32):
            parts = [p.float() for p in parts]
        rgb = (parts[0] if len(parts) == 1 else torch.cat(parts, 1)).contiguous()
    if mlp:
        if all(k in data for k in mlp):
            parts = [data[k].reshape(-1, data[k].shape[-1]).float() for k in mlp]
        else:
            parts = [data["state"].reshape(-1, data["state"].shape[-1]).float()]
        state = (parts[0] if len(parts) == 1 else torch.cat(parts, 1)).contiguous()
    return rgb, state


def hp_from_cfg(cfg) -> dict:
    a = cfg.algo
    if str(a.loss_reduction).lower() != "mean":
        raise NotImplementedError("loss_reduction must be 'mean'")
    return dict(clip_coef=float(a.clip_coef), vf_coef=float(a.vf_coef), ent_coef=float(a.ent_coef),
                clip_vloss=bool(a.clip_vloss), normalize_advantages=bool(a.normalize_advantages),
                max_grad_norm=float(a.max_grad_norm))


def default_init(shapes, generator: torch.Generator, ortho_linear_prefix: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """torch's default reset_parameters for Conv2d / Linear: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias
    (the reference builds its PPO modules without a custom init unless encoder.ortho_init, ppo/agent.py:140-144)."""
    out, bound = {}, None
    for name, shp in shapes.items():
        if name.endswith(".weight"):
            bound = 1.0 / math.sqrt(math.prod(shp[1:]))
            if ortho_linear_prefix and name.startswith(ortho_linear_prefix) and len(shp) == 2:
                w = torch.empty(*shp)
                torch.nn.init.orthogonal_(w, 1.0, generator=generator)
                out[name], bound = w, 0.0
                continue
        out[name] = (torch.rand(*shp, generator=generator) * 2 - 1) * bound
    return out


class PPOAgent:
    """Reference surface used by `ppo.main` / checkpoints (ppo/agent.py:84-239)."""

    def __init__(self, engine: PPOEngine):
        self._b200_engine = engine
        self.actions_dim = list(engine.spec["actions_dim"])
        self.is_continuous = engine.spec["is_continuous"]

    def state_dict(self):
        return self._b200_engine.export_reference_state()

    def load_state_dict(self, state: Dict[str, torch.Tensor]) -> None:
        self._b200_engine.load_reference_state(state)

    def parameters(self):
        return iter(self._b200_engine.group.views.values())

    def forward(self, *a, **k):
        raise RuntimeError("the B200 PPOAgent has no forward(): the update runs in PPOEngine kernels")

    __call__ = forward


class PPOPlayer:
    """Acting path (reference: ppo/agent.py:242-322): `forward(obs) -> (actions, logprobs, values)`, `get_values`,
    `get_actions(obs, greedy)` on the trainer's flat parameter group (nothing to tie or copy).  obs: the dict the
    rollout loop passes — image key `[E, C, H, W]` float already normalised (ppo.py:283-285) or raw uint8, vector key
    `[E, D]`.  `noise` (extra, optional): injected Exp(1) / N(0,1) draws for parity tests."""

    def __init__(self, engine: PPOEngine):
        self.engine = engine
        self._ctr = torch.zeros(1, dtype=torch.int32, device=engine.device)
        self.rng_seed = 0x9E37
        self._acts: Dict[int, tuple] = {}

    class _ActorInfo:
        def __init__(self, engine):
            self.is_continuous, self.distribution = engine.spec["is_continuous"], engine.dist

    @property
    def actor(self):
        return PPOPlayer._ActorInfo(self.engine)

    def eval(self):
        """the reference's test() puts the player in eval mode first (ppo/utils.py:41); there is nothing to switch"""
        return self

    def _run(self, obs, actor: bool, critic: bool):
        e, s = self.engine, self.engine.spec
        rgb, x_state = gather_obs(s, obs)
        normalized = False
        if rgb is not None:
            E, normalized = rgb.shape[0], rgb.dtype != torch.uint8
        if x_state is not None:
            x_state = x_state.unsqueeze(0)
            E = x_state.shape[1]
        b = e._buffers(E)
        e.forward(b, rgb, x_state, rgb_normalized=normalized, actor=actor, critic=critic)
        return b, E

    def _sample(self, b, E, greedy: bool, noise, get_actions: bool = False):
        e = self.engine
        mode = e.dist_mode + (1 if (get_actions and e.dist == "tanh_normal") else 0)   # csrc/ppo.cu ppo_act modes
        A = sum(e.head_dims)
        if E not in self._acts:
            f = lambda *sh: torch.zeros(*sh, dtype=torch.float32, device=e.device)  # noqa: E731
            self._acts[E] = (f(E, A), f(E), f(E, A))
        acts, logp, nz = self._acts[E]
        if noise is None and not greedy:
            e.ops.increment(self._ctr)
            (e.ops.fill_normal if e.spec["is_continuous"] else e.ops.fill_exponential)(nz.view(-1), self.rng_seed, 21, self._ctr)
            noise = nz
        e.ops.ppo_act(b["head"][0], None if greedy else noise.reshape(E, A).contiguous(), acts, logp, e.head_dims,
                      mode, greedy)
        if e.spec["is_continuous"]:
            return (acts.clone(),), logp.clone().unsqueeze(-1)
        out, off = [], 0
        for ad in e.head_dims:
            out.append(acts[:, off:off + ad].clone())
            off += ad
        return tuple(out), logp.clone().unsqueeze(-1)

    @torch.no_grad()
    def forward(self, obs, noise=None):
        b, E = self._run(obs, True, True)
        actions, logp = self._sample(b, E, False, noise)
        return actions, logp, b["values"][0].clone()

    __call__ = forward

    @torch.no_grad()
    def get_values(self, obs):
        b, _ = self._run(obs, False, True)
        return b["values"][0].clone()

    @torch.no_grad()
    def get_actions(self, obs, greedy: bool = False, noise=None):
        b, E = self._run(obs, True, False)
        return self._sample(b, E, greedy, noise, get_actions=True)[0]


def build_agent(fabric, actions_dim: Sequence[int], is_continuous: bool, cfg: Dict[str, Any], obs_space,
                agent_state: Optional[Dict[str, torch.Tensor]] = None, ops=None) -> Tuple[PPOAgent, PPOPlayer]:
    if ops is None:
        from sheeprl_b200.lib import CudaOps

        ops = CudaOps()
    spec = spec_from_cfg(cfg, actions_dim, is_continuous, obs_space)
    o = cfg.algo.optimizer
    opt = {"lr": float(o.lr), "eps": float(o.eps), "betas": tuple(o.get("betas", (0.9, 0.999))),
           "weight_decay": float(o.get("weight_decay", 0) or 0)}
    eng = PPOEngine(spec, hp_from_cfg(cfg), opt, fabric.device, ops, seed=int(cfg.get("seed", 0) or 0))
    g = torch.Generator().manual_seed(int(cfg.get("seed", 0) or 0))
    ortho = "feature_extractor." if cfg.algo.encoder.ortho_init else None
    eng.load_reference_state(default_init(eng.reference_shapes(), g, ortho))
    _attach_if_distributed(fabric, eng)
    agent = PPOAgent(eng)
    if agent_state:
        agent.load_state_dict(agent_state)
    return agent, PPOPlayer(eng)


def _attach_if_distributed(fabric, eng) -> None:
    """the reference gets DDP from `fabric.setup_module(agent)` (ppo/agent.py:352-356); the engine's equivalent is the
    all-reduce hook on its flat gradient"""
    if int(getattr(fabric, "world_size", 1) or 1) > 1:
        import torch.distributed as dist

        from sheeprl_b200.parallel import attach_data_parallel

        if not dist.is_initialized():
            raise RuntimeError("fabric.world_size > 1 but torch.distributed is not initialised (launch through Fabric / torchrun)")
        attach_data_parallel(eng)
