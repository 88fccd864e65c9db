"""`build_agent` for recurrent PPO on the CUDA engine — same signature / return tuple as the reference
(`sheeprl/algos/ppo_recurrent/agent.py:412-470`).  `RecurrentPPOAgent` is a parameter container whose `state_dict()`
has the reference's keys and shapes; the arithmetic of `train()` runs in `RecurrentPPOEngine` kernels.
`RecurrentPPOPlayer` acts on the trainer's flat parameter group (nothing to tie or copy)."""
from __future__ import annotations

import math
from typing import Any, Dict, Optional, Sequence, Tuple

import torch

from sheeprl_b200.algos.ppo.agent import PPOPlayer, default_init, gather_obs, hp_from_cfg, spec_from_cfg
from sheeprl_b200.algos.ppo_recurrent.engine import RecurrentPPOEngine
from sheeprl_b200.lib import sync_deterministic


def rnn_spec_from_cfg(cfg) -> dict:
    """rnn part of the engine spec from `cfg.algo.rnn` (configs/algo/ppo_recurrent.yaml), with the reference's limits:
    the post-RNN MLP works only at the LSTM width (RecurrentModel.forward reshapes its output to the LSTM output)."""
    r, a = cfg.algo.rnn, cfg.algo
    H = int(r.lstm.hidden_size)
    out = {"hidden": H, "pre": None, "post": None}
    for name, key in (("pre", "pre_rnn_mlp"), ("post", "post_rnn_mlp")):
        m = r[key]
        if not m.apply:
            continue
        if not bool(m.get("bias", True)):
            raise NotImplementedError(f"rnn.{key}.bias=False is not built")
        if str(m.activation).rsplit(".", 1)[-1] != str(a.actor.dense_act).rsplit(".", 1)[-1]:
            raise NotImplementedError(f"rnn.{key}.activation must be the actor / critic / encoder dense_act")
        out[name] = (int(m.dense_units), bool(m.layer_norm))
    if out["post"] and out["post"][0] != H:
        raise ValueError(f"rnn.post_rnn_mlp.dense_units ({out['post'][0]}) must equal rnn.lstm.hidden_size ({H}): the "
                         "reference's RecurrentModel.forward fails at any other width")
    return out


class RecurrentPPOAgent:
    """Reference surface used by `ppo_recurrent.main` / checkpoints (ppo_recurrent/agent.py:83-262)."""

    def __init__(self, engine: RecurrentPPOEngine, num_envs: int):
        self._b200_engine = engine
        self.actions_dim = list(engine.spec["actions_dim"])
        self.is_continuous = False
        self.num_envs = int(num_envs)
        self.rnn_hidden_size = engine.H
        self.device = engine.device
        self._initial_states = self.reset_hidden_states()

    @property
    def initial_states(self) -> Tuple[torch.Tensor, torch.Tensor]:
        return self._initial_states

    @initial_states.setter
    def initial_states(self, value) -> None:
        self._initial_states = value

    def reset_hidden_states(self) -> Tuple[torch.Tensor, torch.Tensor]:
        z = lambda: torch.zeros(1, self.num_envs, self.rnn_hidden_size, device=self.device)  # noqa: E731
        return z(), z()

    def state_dict(self):
        return self._b200_engine.export_reference_state()

    def load_state_dict(self, state: Dict[str, torch.Tensor]) -> None:
        self._b200_engine.load_reference_state(state)

    def parameters(self):
        return iter(self._b200_engine.group.views.values())

    def forward(self, *a, **k):
        raise RuntimeError("the CUDA RecurrentPPOAgent has no forward(): the update runs in RecurrentPPOEngine kernels")

    __call__ = forward


class RecurrentPPOPlayer(PPOPlayer):
    """Acting path (reference: ppo_recurrent/agent.py:265-409).  One env step is the training schedule at T = 1:
    encoders, input projection, `lstm_seq_fwd`, heads and `ppo_act` on the trainer's flat group, with no host
    synchronisation.  obs: the dict the rollout loop passes, `[1, E, ...]` per key (images already normalised, or raw
    uint8); prev_actions `[1, E, sum(actions_dim)]`; prev_states `(hx, cx)`, each `[1, E, H]`.  The returned states are
    fresh tensors.  `noise` (extra, optional): injected Exp(1) draws `[E, sum(actions_dim)]` for parity tests."""

    def __init__(self, engine: RecurrentPPOEngine, num_envs: int = 1):
        super().__init__(engine)
        self.rng_seed = 0x9E38
        self.num_envs = int(num_envs)
        self.rnn_hidden_size = engine.H
        self.actions_dim = list(engine.spec["actions_dim"])
        self.device = engine.device

    def eval(self):
        return self

    def reset_hidden_states(self):
        z = lambda: torch.zeros(1, self.num_envs, self.rnn_hidden_size, device=self.device)  # noqa: E731
        return z(), z()

    def _step(self, obs, prev_actions, prev_states, mask, actor: bool, critic: bool):
        if mask is not None:
            raise NotImplementedError("the player steps one time step per call; mask is not supported")
        e = self.engine
        sync_deterministic(e.ops)
        rgb, x_state = gather_obs(e.spec, obs)
        E = prev_actions.shape[-2]
        H = e.H
        b = e.seq_buffers(1, E)
        e.ops.copy(prev_states[0].reshape(E, H).float().contiguous(), b["hbuf"][0])
        e.ops.copy(prev_states[1].reshape(E, H).float().contiguous(), b["c0"])
        hT = torch.empty(1, E, H, dtype=torch.float32, device=e.device)
        cT = torch.empty(1, E, H, dtype=torch.float32, device=e.device)
        e.seq_forward(b, rgb, None if x_state is None else x_state.unsqueeze(0),
                      prev_actions.reshape(E, -1).float().contiguous(),
                      rgb_normalized=rgb is not None and rgb.dtype != torch.uint8, keep=False, hT=hT, cT=cT,
                      actor=actor, critic=critic)
        return b, E, (hT, cT)

    @torch.no_grad()
    def forward(self, obs, prev_actions, prev_states, actions=None, mask=None, greedy: bool = False, noise=None):
        if actions is not None:
            raise NotImplementedError("the player samples its actions; passing `actions` is not supported")
        b, E, states = self._step(obs, prev_actions, prev_states, mask, True, True)
        acts, logp = self._sample(b, E, greedy, noise)
        return (tuple(a.unsqueeze(0) for a in acts), logp.view(1, E, 1), b["values"][0].clone().view(1, E, 1), states)

    __call__ = forward

    @torch.no_grad()
    def get_values(self, obs, prev_actions, prev_states, mask=None):
        b, E, states = self._step(obs, prev_actions, prev_states, mask, False, True)
        return b["values"][0].clone().view(1, E, 1), states

    @torch.no_grad()
    def get_actions(self, obs, prev_actions, prev_states, mask=None, greedy: bool = False, noise=None):
        b, E, states = self._step(obs, prev_actions, prev_states, mask, True, False)
        acts, _ = self._sample(b, E, greedy, noise, get_actions=True)
        return tuple(a.unsqueeze(0) for a in acts), states


def build_agent(fabric, actions_dim: Sequence[int], is_continuous: bool, cfg: Dict[str, Any], obs_space,
                agent_state: Optional[Dict[str, torch.Tensor]] = None,
                ops=None) -> Tuple[RecurrentPPOAgent, RecurrentPPOPlayer]:
    if is_continuous:
        raise NotImplementedError("recurrent PPO supports discrete actions only: the reference's continuous path fails "
                                  "(RecurrentPPOAgent._get_actions passes a tuple to Normal.log_prob)")
    if int(getattr(fabric, "world_size", 1) or 1) > 1:
        raise NotImplementedError("recurrent PPO runs on one device: the reference relies on DDP Join for uneven "
                                  "minibatch counts across ranks")
    spec = spec_from_cfg(cfg, actions_dim, is_continuous, obs_space)
    spec["rnn"] = rnn_spec_from_cfg(cfg)
    if ops is None:
        from sheeprl_b200.lib import CudaOps

        ops = CudaOps()
    o = cfg.algo.optimizer
    opt = {"lr": float(o.lr), "eps": float(o.eps), "betas": tuple(o.get("betas", (0.9, 0.999)))}
    eng = RecurrentPPOEngine(spec, hp_from_cfg(cfg), opt, fabric.device, ops, seed=int(cfg.get("seed", 0) or 0))
    shapes = eng.reference_shapes()
    init = default_init(shapes, torch.Generator().manual_seed(int(cfg.get("seed", 0) or 0)))
    bound = 1.0 / math.sqrt(eng.H)                   # nn.LSTM.reset_parameters: U(-1/sqrt(H), 1/sqrt(H)) everywhere
    g = torch.Generator().manual_seed(int(cfg.get("seed", 0) or 0) + 1)
    for k, shp in shapes.items():
        if k.startswith("rnn._lstm."):
            init[k] = (torch.rand(*shp, generator=g) * 2 - 1) * bound
        elif len(shp) == 1 and k.endswith(".weight"):  # LayerNorm: weight 1, bias 0
            init[k], init[k[:-6] + "bias"] = torch.ones(shp), torch.zeros(shp)
    eng.load_reference_state(init)
    agent = RecurrentPPOAgent(eng, int(cfg.env.num_envs))
    if agent_state:
        agent.load_state_dict(agent_state)
    return agent, RecurrentPPOPlayer(eng, int(cfg.env.num_envs))
