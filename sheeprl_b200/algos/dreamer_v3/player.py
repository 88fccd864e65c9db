"""PlayerDV3 — the acting path of Dreamer-V3 (SURVEY §8f rank 1) on the B200 kernels.

Mirrors the reference's `PlayerDV3` (sheeprl/algos/dreamer_v3/agent.py:596-691): `init_states(reset_envs)`,
`get_actions(obs, greedy, mask)`, attributes `num_envs`, `actions`, `recurrent_state`, `stochastic_state`.  One env step is
encoder -> GRU step -> posterior sample -> actor -> action sample at M = num_envs rows; the schedule below is ~25
launches on the current stream with no host synchronisation (outputs stay on the device), so `main()`'s loop only pays
the one device->host copy of the actions it needs for `envs.step`.

The player owns a small *acting engine* (`DV3Engine` with T=1, B=num_envs) that ADOPTS the trainer's flat parameter
groups, the counterpart of the reference tying `player_p.data = agent_p.data` (agent.py:1229-1235): a train step is
visible to the next `get_actions` without any copy.
"""
from __future__ import annotations

import copy
from typing import Dict, Optional, Sequence

import torch

from sheeprl_b200.engine import ACT_SILU, DV3Engine
from sheeprl_b200.lib import sync_deterministic


class PlayerDV3:
    def __init__(self, engine: DV3Engine, num_envs: int, actor_type: Optional[str] = None, actor_group=None):
        """actor_group: the flat group of the policy that acts (default the trainer's task actor; Plan2Explore passes
        its exploration actor when `algo.player.actor_type == "exploration"`, p2e_dv3/agent.py:206-212)"""
        self.trainer = engine
        self.actor_type = actor_type
        self.actions_dim = engine.actions_dim
        self.device = engine.device
        self.stochastic_size, self.discrete_size = engine.S, engine.D
        self.recurrent_state_size = engine.R
        self._actor_group = actor_group or engine.actor
        self._num_envs = None
        self.num_envs = num_envs
        self._counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.rng_seed = 0x5EED

    @property
    def num_envs(self) -> int:
        return self._num_envs

    @num_envs.setter
    def num_envs(self, n) -> None:
        """The acting engine and the state tensors are sized for `n` rows; a new `n` re-creates them over the same
        parameter groups (the reference's `test()` sets `player.num_envs = 1`, then calls `init_states()`)."""
        n = int(n)
        if n == self._num_envs:
            return
        self._num_envs = n
        engine = self.trainer
        cfg = copy.deepcopy(engine.cfg)
        cfg.algo.per_rank_sequence_length = 1
        cfg.algo.per_rank_batch_size = n
        cfg.algo.horizon = 1
        self.eng = DV3Engine(cfg, engine.actions_dim, in_channels=engine.Cin, device=engine.device, ops=engine.ops,
                             is_continuous=engine.is_continuous,
                             groups=(engine.wm, self._actor_group, engine.critic, engine.target),
                             mlp_dims=dict(zip(engine.vec_keys, engine.vec_dims)), cnn_dims=engine.cnn_dims)
        e, E = self.eng, n
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        # persistent acting state (reference attribute names; leading dim 1 as in the reference)
        self.actions = f(1, E, e.A)
        self.recurrent_state = f(1, E, e.R)
        self.stochastic_state = f(1, E, e.Z)
        self._h_next = f(E, e.R)
        self._noise_z, self._noise_a = f(E, e.Z), f(E, e.A)

    # ------------------------------------------------------------------ reference surface
    class _ActorInfo:
        def __init__(self, is_continuous):
            self.is_continuous = is_continuous

    @property
    def actor(self):                                     # `player.actor.is_continuous` is read by the reference main
        return PlayerDV3._ActorInfo(self.eng.is_continuous)

    @torch.no_grad()
    def init_states(self, reset_envs: Optional[Sequence[int]] = None) -> None:
        """agent.py:640-659: zero actions, h = tanh(initial_recurrent_state), z = mode of the prior(h)."""
        e, ops = self.eng, self.eng.ops
        ops.tanh_fwd(e._w("rssm.initial_recurrent_state").view(1, e.R), e.h0)
        e._transition_forward(e.h0, e.init_tr_pre, e.init_tr_act, e.init_raw)
        ops.cat_sample(e.init_raw, None, e.unimix, e.S, e.D, e.z0)           # noise=None -> mode
        if reset_envs is None or len(reset_envs) == 0:
            self.actions.zero_()
            self.recurrent_state[0].copy_(e.h0.expand(self.num_envs, -1))
            self.stochastic_state[0].copy_(e.z0.expand(self.num_envs, -1))
        else:
            idx = torch.as_tensor(list(reset_envs), dtype=torch.int64, device=self.device)
            self.actions[0].index_fill_(0, idx, 0.0)
            self.recurrent_state[0].index_copy_(0, idx, e.h0.expand(len(idx), -1))
            self.stochastic_state[0].index_copy_(0, idx, e.z0.expand(len(idx), -1))

    @torch.no_grad()
    def get_actions(self, obs: Dict[str, torch.Tensor], greedy: bool = False, mask=None,
                    noise: Optional[Dict[str, torch.Tensor]] = None) -> Sequence[torch.Tensor]:
        """obs[key]: `[1, num_envs, C, H, W]` — float32 already normalised as the reference's `prepare_obs` passes it
        (dreamer_v3/utils.py:80-91), or raw uint8 (normalised by the kernel: 4x less host->device traffic).
        `noise` (extra, optional): {"z": Exp(1) [E, S*D], "a": Exp(1) / N(0,1) [E, A]} for parity tests.
        `mask` is ignored, as the reference's `Actor.forward` ignores it (the reference's `test()` passes the observation's
        `mask*` keys, an empty dict for environments without them)."""
        e, ops, E = self.eng, self.eng.ops, self.num_envs
        sync_deterministic(ops)
        Z = e.Z
        if e.has_cnn:
            x = e.image_batch(obs, E)
            if x.dtype == torch.uint8:
                ops.obs_prep(x.contiguous(), e.x0)
            else:                                                            # already /255 - 0.5: layout change only
                ops.transpose_batched(x.float().contiguous().view(E, e.Cin, e.img * e.img), e.x0.view(E, e.img * e.img, e.Cin))
        off = 0
        for k, d in zip(e.vec_keys, e.vec_dims):                             # vector keys: symlog into the encoder input
            ops.symlog(obs[k].reshape(E, d).float().contiguous(), e.vx[:, off:off + d])
            off += d
        if noise is None:
            ops.increment(self._counter)
            ops.fill_exponential(self._noise_z.view(-1), self.rng_seed, 11, self._counter)
            if e.is_continuous:
                ops.fill_normal(self._noise_a.view(-1), self.rng_seed, 12, self._counter)
            else:
                ops.fill_exponential(self._noise_a.view(-1), self.rng_seed, 12, self._counter)
            nz, na = self._noise_z, self._noise_a
        else:
            nz, na = noise["z"].reshape(E, Z), noise["a"].reshape(E, e.A)
        e._encoder_forward()                                                 # -> e.emb [E, 4096] / e.venc features
        # recurrent model on (z, a, h) of the previous step (agent.py:676-678)
        e._recurrent_forward(self.stochastic_state[0], self.actions[0], self.recurrent_state[0], e.x_pre, e.x_act,
                             e.g_pre, e.g_ln, self._h_next)
        self.recurrent_state[0].copy_(self._h_next)
        # posterior from [h, embed] (agent.py:451-465; decoupled RSSM: from the embedding alone, :682-683) and its sample
        e._project_embedding(e.rp_pre)
        e._posterior_forward(None if e.decoupled else self._h_next, e.rp_pre, e.rp_act, e.post_raw, nz,
                             self.stochastic_state[0])
        # actor on [z, h] (agent.py:783-837)
        lat = e.latent                                                       # [E, Z+R] scratch row block
        ops.copy(self.stochastic_state[0], lat[:, :Z])
        ops.copy(self._h_next, lat[:, Z:])
        am, cur = e.actor_mlp, lat
        for l in range(am.n_hidden):
            ops.gemm(cur, am.W(l), am.pre[l][:E], False, True)
            ops.ln_act_fwd(am.pre[l][:E], e.actor.views[f"model._model.{3 * l + 1}.weight"],
                           e.actor.views[f"model._model.{3 * l + 1}.bias"], e.eps, ACT_SILU, am.act[l][:E])
            cur = am.act[l][:E]
        raw = e.actor_raw[:E]
        e._actor_heads(cur, raw)
        if e.is_continuous:
            if greedy:
                raise NotImplementedError("greedy continuous actions (100-sample arg-max, agent.py:818-821) are not built")
            ac = e.cfg.algo.actor
            ops.cont_action_fwd(raw, na, self.actions[0], None, float(ac.min_std), float(ac.max_std), float(ac.init_std),
                                float(ac.action_clip))
            return (self.actions.clone(),)
        out, off = [], 0
        for ad in e.actions_dim:
            ops.cat_sample(raw[:, off:off + ad], None if greedy else na[:, off:off + ad], e.unimix, 1, ad,
                           self.actions[0][:, off:off + ad])
            out.append(self.actions[:, :, off:off + ad].clone())
            off += ad
        return tuple(out)

    __call__ = get_actions
