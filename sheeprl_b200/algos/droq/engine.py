"""Kernel schedule of one DroQ `train()` call: G critic gradient steps, then one actor and one temperature step, on one
stream with no autograd, no host synchronisation and no allocation inside the loop.

Reference being replaced: `train` sheeprl/algos/droq/droq.py:32-164, `DROQAgent` / `DROQCritic`
sheeprl/algos/droq/agent.py:19-267.  Built on `SACEngine` (same flat groups, actor, tanh-Normal sampling, target, Adam,
EMA and persistent `[obs | action]` critic inputs); what differs is the critic, `Linear -> Dropout -> LayerNorm -> ReLU`
twice then `Linear`, whose miniblock runs as one fused launch per layer for all n critics (csrc/droq.cu).

Per critic minibatch the reference computes the target once, then for each critic i in turn takes an MSE step with the
qf optimizer and an EMA of critic i's target.  The critics are independent and their Adam step counts stay equal, so one
batched backward, one Adam step over the whole qf group and one EMA per minibatch is the same update.  Dropout is active
in every critic forward (target, online, policy loss); the keep masks of a whole call are drawn by one launch.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional

import torch

from sheeprl_b200.algos.sac.engine import SACEngine
from sheeprl_b200.dense import DropoutLayerNormReLU

LN_EPS = 1e-5                  # nn.LayerNorm(H) (droq/agent.py:40-42)
MASKS_PER_STEP = 4             # target layer 0, 1; online layer 0, 1 (each [n, B, ceil(H/32)] words)


def critic_layout(dropout: float):
    """indices of the critic MLP's Linears and LayerNorms in `model._model` (utils/model.py:34-88: a Dropout module
    sits between Linear and LayerNorm only when dropout > 0)"""
    return ((0, 4, 8), (2, 6)) if dropout > 0 else ((0, 3, 6), (1, 4))


def droq_critic_shapes(obs_dim: int, act_dim: int, hidden: int, n_critics: int, dropout: float):
    lin, ln = critic_layout(dropout)
    qf, dims = OrderedDict(), ((hidden, obs_dim + act_dim), (hidden, hidden), (1, hidden))
    for i in range(n_critics):
        m = f"{i}.model._model"
        for j, (out, inp) in enumerate(dims):          # reference parameter order: Linear, LayerNorm, Linear, ...
            qf[f"{m}.{lin[j]}.weight"], qf[f"{m}.{lin[j]}.bias"] = (out, inp), (out,)
            if j < 2:
                qf[f"{m}.{ln[j]}.weight"], qf[f"{m}.{ln[j]}.bias"] = (hidden,), (hidden,)
    return qf


class DroQEngine(SACEngine):
    ACTOR_LOSS = "droq_actor_loss"                    # the policy loss on the MEAN of the critics (droq.py:147-150)

    def __init__(self, obs_dim: int, act_dim: int, hidden_actor: int, hidden_critic: int, n_critics: int, batch: int,
                 gamma: float, tau: float, alpha: float, dropout: float, action_low, action_high, opt_actor: dict,
                 opt_qf: dict, opt_alpha: dict, device, ops, seed: int = 0):
        if not 0.0 <= float(dropout) < 1.0:
            raise ValueError(f"critic dropout must be in [0, 1), got {dropout}")
        if not ops.dropout_ln_relu_supported(int(hidden_critic)):
            raise ValueError(f"critic hidden_size {hidden_critic}: the fused Dropout-LayerNorm-ReLU kernel takes "
                             "1 to 1024 columns")
        self.p = float(dropout)
        super().__init__(obs_dim, act_dim, hidden_actor, hidden_critic, n_critics, batch, gamma, tau, alpha, action_low,
                         action_high, opt_actor, opt_qf, opt_alpha, device, ops, seed)

    def _param_shapes(self):
        sa, _ = super()._param_shapes()
        return sa, droq_critic_shapes(self.O, self.A, self.Hc, self.n, self.p)

    def _critic_linears(self):
        return critic_layout(self.p)[0]

    def _critic_block(self, j: int, views):
        k = critic_layout(self.p)[1][j]
        (gamma, dgamma), (beta, dbeta) = views(f"{k}.weight"), views(f"{k}.bias")
        return DropoutLayerNormReLU(self.p, LN_EPS, gamma, beta, dgamma, dbeta)

    # ------------------------------------------------------------------ buffers
    def _alloc(self):
        super()._alloc()
        self.G = 0                    # the per-call buffers follow the batch size too

    def _alloc_call(self, G: int):
        """buffers whose size follows the number of critic steps per call"""
        n, B, A = self.n, self.B, self.A
        self.eps_next_all = torch.zeros(G, B, A, dtype=torch.float32, device=self.device)
        words = (self.Hc + 31) // 32
        self.masks = torch.zeros(MASKS_PER_STEP * G + 2, n, B, words, dtype=torch.int32, device=self.device)
        self.value_losses = torch.zeros(G, n, dtype=torch.float32, device=self.device)
        self.G = G

    def critic_slice(self, i: int) -> slice:
        """flat-group range of critic i (its parameters are contiguous in the group)"""
        off, lin = self.qf.offsets, critic_layout(self.p)[0]
        lo = off[f"{i}.model._model.{lin[0]}.weight"]
        hi = off[f"{i + 1}.model._model.{lin[0]}.weight"] if i + 1 < self.n else self.qf.numel
        return slice(lo, hi)

    # ------------------------------------------------------------------ the update
    def train_call(self, critic_data: Dict[str, torch.Tensor], actor_obs: torch.Tensor,
                   noise: Optional[Dict[str, torch.Tensor]] = None):
        """critic_data: observations / next_observations [G*B, O], actions [G*B, A], rewards / terminated [G*B, 1]
        (critic minibatch g is rows [g*B, (g+1)*B)); actor_obs [B, O]; float32 on the device.  noise (parity tests):
        eps_next [G, B, A], eps_cur [B, A] and, when p > 0, masks [4G+2, n, B, ceil(H/32)] int32 in the reference's
        dropout call order: per minibatch the target critics' two layers, then the online critics', then the policy
        loss's."""
        o, O, B = self.ops, self.O, self.B
        rows = critic_data["observations"].shape[0]
        if rows % B or actor_obs.shape != (B, O):
            raise ValueError(f"critic rows {rows} must be a multiple of the batch size {B}; actor rows {tuple(actor_obs.shape)}")
        G = rows // B
        if G != self.G:
            self._alloc_call(G)
        if noise is None:
            o.increment(self.noise_counter)
            o.fill_normal(self.eps_next_all, self.rng_seed, 1, self.noise_counter)
            o.fill_normal(self.eps_cur, self.rng_seed, 2, self.noise_counter)
            if self.p > 0:
                o.dropout_mask(self.masks, self.p, self.rng_seed, 3, self.noise_counter)
            eps_next, eps_cur, masks = self.eps_next_all, self.eps_cur, self.masks
        else:
            eps_next, eps_cur, masks = noise["eps_next"], noise["eps_cur"], noise.get("masks")
        if self.p == 0:
            masks = None
        la = self.alpha.views["log_alpha"]
        obs_all, nobs_all, act_all = critic_data["observations"], critic_data["next_observations"], critic_data["actions"]
        rew_all, term_all = critic_data["rewards"].reshape(-1), critic_data["terminated"].reshape(-1)
        for g in range(G):
            r = slice(g * B, (g + 1) * B)
            mk = (lambda s: None) if masks is None else (lambda s: masks[MASKS_PER_STEP * g + s: MASKS_PER_STEP * g + s + 2])
            o.copy(nobs_all[r], self.x_next[:, :O])
            o.copy(obs_all[r], self.x_cur[:, :O])
            o.copy(act_all[r], self.x_cur[:, O:])
            # target, once for all critics (droq.py:123-128)
            self._actor_fwd(nobs_all[r], eps_next[g], self.x_next[:, O:], save_tanh=False)
            self.q_target.forward(self.x_next.unsqueeze(0), self.q_acts, self.q, mk(0))
            o.sac_target(self.q[:, :, 0], self.logp, rew_all[r], term_all[r], la, self.gamma, self.y)
            # every critic's MSE step, then every critic's EMA (droq.py:129-144)
            self.q_online.forward(self.x_cur.unsqueeze(0), self.q_acts, self.q, mk(2))
            for i in range(self.n):
                o.sac_critic_loss(self.q[i:i + 1, :, 0], self.y, self.dq[i:i + 1, :, 0], self.value_losses[g, i:i + 1])
            self.q_online.backward(self.dq, self.x_cur.unsqueeze(0), self.q_acts, masks=mk(2))
            self._adam(self.qf, self.opt["qf"], "qf")
            o.ema(self.qf_target.flat, self.qf.flat, self.tau)
        # actor and temperature (droq.py:146-160)
        o.copy(actor_obs, self.x_pi[:, :O])
        self._actor_update(actor_obs, eps_cur, None if masks is None else masks[MASKS_PER_STEP * G: MASKS_PER_STEP * G + 2])

    # ------------------------------------------------------------------ state
    def metrics_dict(self) -> Dict[str, torch.Tensor]:
        """Loss/value_loss: the [G*n] critic losses in the reference's update order (minibatch-major)"""
        return {"Loss/value_loss": self.value_losses.reshape(-1), "Loss/policy_loss": self.metrics[1],
                "Loss/alpha_loss": self.metrics[2]}
