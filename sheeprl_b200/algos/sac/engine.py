"""Kernel schedule of one SAC update (SURVEY §8 a20): forward, hand-derived backward and the three fused Adam steps
as ~45 launches on one stream, no autograd, no host synchronisation (the temperature is read on the device), hence
capturable in a CUDA graph.

Reference being replaced: `train` sheeprl/algos/sac/sac.py:32-78, `SACAgent` sheeprl/algos/sac/agent.py:145-267,
losses sheeprl/algos/sac/loss.py.  The `ops` object is `sheeprl_b200.lib.CudaOps` in production (tests on a
GPU-less host pass the torch test double `oracle/ops_emul.py::EmulOps`).

Layout: three flat parameter groups (actor / twin critics / log_alpha) + a target copy of the critics with the same
layout, so that (a) both critics — and both targets — run in one batched launch per layer with a constant
parameter stride, (b) EMA, Adam and the data-parallel all-reduce are single passes over one buffer.  The critics'
input `[obs | action]` is a persistent buffer whose action columns are written directly by the sampling kernel (the
reference's torch.cat, sac/agent.py:50).
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional

import torch

from sheeprl_b200.dense import Act, Linear, Stack, stacked
from sheeprl_b200.params import FlatGroup


def sac_param_shapes(obs_dim: int, act_dim: int, hidden_actor: int, hidden_critic: int, n_critics: int):
    actor = OrderedDict([
        ("model._model.0.weight", (hidden_actor, obs_dim)), ("model._model.0.bias", (hidden_actor,)),
        ("model._model.2.weight", (hidden_actor, hidden_actor)), ("model._model.2.bias", (hidden_actor,)),
        # fc_mean and fc_logstd stacked: one product gives [mean | log_std]
        ("head.weight", (2 * act_dim, hidden_actor)), ("head.bias", (2 * act_dim,)),
    ])
    qf = OrderedDict()
    for i in range(n_critics):
        qf[f"{i}.model._model.0.weight"] = (hidden_critic, obs_dim + act_dim)
        qf[f"{i}.model._model.0.bias"] = (hidden_critic,)
        qf[f"{i}.model._model.2.weight"] = (hidden_critic, hidden_critic)
        qf[f"{i}.model._model.2.bias"] = (hidden_critic,)
        qf[f"{i}.model._model.4.weight"] = (1, hidden_critic)
        qf[f"{i}.model._model.4.bias"] = (1,)
    return actor, qf


class SACEngine:
    ACTOR_LOSS = "sac_actor_loss"                     # the policy loss on the min over the critics

    def __init__(self, obs_dim: int, act_dim: int, hidden_actor: int, hidden_critic: int, n_critics: int, batch: int,
                 gamma: float, tau: float, alpha: float, action_low, action_high, opt_actor: dict, opt_qf: dict,
                 opt_alpha: dict, device, ops, seed: int = 0):
        self.O, self.A, self.Ha, self.Hc, self.n, self.B = obs_dim, act_dim, hidden_actor, hidden_critic, n_critics, batch
        self.gamma, self.tau = float(gamma), float(tau)
        self.target_entropy = -float(act_dim)                               # sac/agent.py:341
        self.device, self.ops = torch.device(device), ops
        self.opt = {"actor": opt_actor, "qf": opt_qf, "alpha": opt_alpha}
        sa, sq = self._param_shapes()
        self.actor = FlatGroup(sa, device)
        self.qf = FlatGroup(sq, device)
        self.qf_target = FlatGroup(sq, device, with_optimizer=False)
        self.alpha = FlatGroup({"log_alpha": (1,)}, device)
        with torch.no_grad():
            self.alpha.views["log_alpha"].fill_(float(torch.log(torch.tensor(float(alpha)))))
        low = torch.as_tensor(action_low, dtype=torch.float32).reshape(-1).expand(act_dim)
        high = torch.as_tensor(action_high, dtype=torch.float32).reshape(-1).expand(act_dim)
        self.scale = ((high - low) / 2.0).to(device).contiguous()           # sac/agent.py:91-92
        self.abias = ((high + low) / 2.0).to(device).contiguous()
        self.rng_seed = seed
        self.allreduce = None      # data-parallel hook: f(flat_grad, name) -> averaged in place (parallel.py)
        # Philox position of the rsample noise: created ONCE — `_alloc()` runs again whenever the minibatch size changes
        # (tail minibatch of a chunk) and must not rewind the stream
        self.noise_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.metrics = torch.zeros(3, dtype=torch.float32, device=self.device)      # value, policy, alpha loss
        lin = lambda k: Linear.of(self.actor, k)  # noqa: E731
        self.pi = Stack(ops, [(lin("model._model.0.weight"), Act("relu")), (lin("model._model.2.weight"), Act("relu")),
                              (lin("head.weight"), Act("none"))])
        self.q_online = self._critic_stack(self.qf.flat, self.qf.grad)
        self.q_target = self._critic_stack(self.qf_target.flat)
        self._alloc()

    def _param_shapes(self):
        return sac_param_shapes(self.O, self.A, self.Ha, self.Hc, self.n)

    def _critic_stack(self, flat: torch.Tensor, grad: Optional[torch.Tensor] = None) -> Stack:
        """the n critics bound to `flat` (and `grad`) as one stack: [n, ...] views with the constant inter-critic stride"""
        n, off, shapes = self.n, self.qf.offsets, self.qf.shapes
        lin = self._critic_linears()
        stride = off[f"1.model._model.{lin[0]}.weight"] - off[f"0.model._model.{lin[0]}.weight"] if n > 1 else flat.numel()

        def v(f, key):
            key = f"0.model._model.{key}"
            return None if f is None else stacked(f, off[key], n, stride, shapes[key])

        def linear(i):
            return Linear(v(flat, f"{i}.weight"), v(flat, f"{i}.bias"), v(grad, f"{i}.weight"), v(grad, f"{i}.bias"))

        blocks = [self._critic_block(j, lambda key: (v(flat, key), v(grad, key))) for j in range(2)] + [Act("none")]
        return Stack(self.ops, [(linear(i), blk) for i, blk in zip(lin, blocks)])

    def _critic_linears(self):
        """indices of the critic MLP's Linears in `model._model`"""
        return 0, 2, 4

    def _critic_block(self, j: int, views):
        """what follows the critics' hidden Linear j; views(key) -> (parameter, gradient) [n, ...] views"""
        return Act("relu")

    # ------------------------------------------------------------------ buffers
    def _alloc(self):
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        B, O, A, n = self.B, self.O, self.A, self.n
        self.x_next, self.x_cur, self.x_pi = f(B, O + A), f(B, O + A), f(B, O + A)
        self.pi_acts, self.head, self.q_acts, self.q = self.pi.acts(B), f(1, B, 2 * A), self.q_online.acts(B), f(n, B, 1)
        self.logp, self.tanh_y, self.y = f(B), f(B, A), f(B)
        self.dq, self.dact, self.dhead = f(n, B, 1), f(n, B, A), f(1, B, 2 * A)
        self.eps_next, self.eps_cur = f(B, A), f(B, A)
        self.norm_out = f(1)
        self.zero_normsq = torch.zeros(1, dtype=torch.float64, device=self.device)

    # ------------------------------------------------------------------ networks
    def _actor_fwd(self, obs: torch.Tensor, eps: torch.Tensor, action_out: torch.Tensor, save_tanh: bool):
        self.pi.forward(obs.unsqueeze(0), self.pi_acts, self.head)
        self.ops.sac_sample_fwd(self.head[0], eps, self.scale, self.abias, action_out, self.logp,
                                self.tanh_y if save_tanh else None)

    def _adam(self, group: FlatGroup, opt: dict, name: str):
        if self.allreduce is not None:
            self.allreduce(group.grad, name)
        self.ops.increment(group.step_t)
        group.step += 1
        handle = getattr(group, "optimizer", None)          # B200Adam built by main / make_optimizers (schedulers edit it)
        lr = handle.lr if handle is not None else opt["lr"]
        self.ops.adam_step(group.flat, group.grad, group.exp_avg, group.exp_avg_sq, self.zero_normsq, 0.0, lr,
                           opt["betas"][0], opt["betas"][1], opt["eps"], group.step_t, self.norm_out,
                           **group.adam_kwargs(opt.get("weight_decay", 0.0)))

    # ------------------------------------------------------------------ the update
    def train_step(self, data: Dict[str, torch.Tensor], do_ema: bool, noise: Optional[Dict[str, torch.Tensor]] = None):
        """data: observations / next_observations [B,O], actions [B,A], rewards / terminated [B,1] (float32, on the
        device).  noise (parity tests): {"eps_next", "eps_cur"} N(0,1) draws of the two rsample calls."""
        o, O = self.ops, self.O
        obs, nobs = data["observations"], data["next_observations"]
        assert obs.shape == (self.B, O) and data["actions"].shape == (self.B, self.A), (obs.shape, data["actions"].shape)
        if noise is None:
            o.increment(self.noise_counter)
            o.fill_normal(self.eps_next, self.rng_seed, 1, self.noise_counter)
            o.fill_normal(self.eps_cur, self.rng_seed, 2, self.noise_counter)
            eps_next, eps_cur = self.eps_next, self.eps_cur
        else:
            eps_next, eps_cur = noise["eps_next"], noise["eps_cur"]
        o.copy(nobs, self.x_next[:, :O])
        o.copy(obs, self.x_cur[:, :O])
        o.copy(obs, self.x_pi[:, :O])
        o.copy(data["actions"], self.x_cur[:, O:])
        la = self.alpha.views["log_alpha"]
        # ---- soft-critic update (sac.py:45-53)
        self._actor_fwd(nobs, eps_next, self.x_next[:, O:], save_tanh=False)
        self.q_target.forward(self.x_next.unsqueeze(0), self.q_acts, self.q)
        o.sac_target(self.q[:, :, 0], self.logp, data["rewards"].reshape(-1), data["terminated"].reshape(-1), la,
                     self.gamma, self.y)
        self.q_online.forward(self.x_cur.unsqueeze(0), self.q_acts, self.q)
        o.sac_critic_loss(self.q[:, :, 0], self.y, self.dq[:, :, 0], self.metrics[0:1])
        self.q_online.backward(self.dq, self.x_cur.unsqueeze(0), self.q_acts)
        self._adam(self.qf, self.opt["qf"], "qf")
        # ---- target EMA (sac.py:55-57)
        if do_ema:
            o.ema(self.qf_target.flat, self.qf.flat, self.tau)
        # ---- actor update (sac.py:59-66) and temperature (sac.py:68-73)
        self._actor_update(obs, eps_cur)

    def _actor_update(self, obs: torch.Tensor, eps_cur: torch.Tensor, masks: Optional[torch.Tensor] = None):
        """one actor and one temperature step on `obs` (whose copy already sits in x_pi's observation columns): the
        policy and temperature losses on the critics' q of x_pi, then the critics' input gradient w.r.t. the action
        columns only (dact; no critic parameter gradients) and the actor's backward.  masks: the critics' dropout masks"""
        o, x_pi = self.ops, self.x_pi.unsqueeze(0)
        la = self.alpha.views["log_alpha"]
        self._actor_fwd(obs, eps_cur, self.x_pi[:, self.O:], save_tanh=True)
        self.q_online.forward(x_pi, self.q_acts, self.q, masks)
        getattr(o, self.ACTOR_LOSS)(self.q[:, :, 0], self.logp, la, self.target_entropy, self.dq[:, :, 0],
                                    self.metrics[1:2], self.metrics[2:3], self.alpha.grad[0:1])
        self.q_online.backward(self.dq, x_pi, self.q_acts, [(self.dact, slice(self.O, None), "none", None)], wgrad=False,
                               masks=masks)
        o.sac_sample_bwd(self.head[0], eps_cur, self.tanh_y, self.scale, self.dact, la, self.dhead[0])
        self.pi.backward(self.dhead, obs.unsqueeze(0), self.pi_acts)
        self._adam(self.actor, self.opt["actor"], "actor")
        # temperature: gradient written by the policy loss kernel
        self._adam(self.alpha, self.opt["alpha"], "alpha")

    # ------------------------------------------------------------------ state
    def metrics_dict(self) -> Dict[str, torch.Tensor]:
        return {"Loss/value_loss": self.metrics[0], "Loss/policy_loss": self.metrics[1], "Loss/alpha_loss": self.metrics[2]}

    def load_reference_state(self, actor: dict, qf: dict, qf_target: dict, log_alpha):
        """actor keys as SACActor.state_dict() (fc_mean / fc_logstd separate), critics keyed '{i}.model._model.k.*'"""
        a = dict(actor)
        a["head.weight"] = torch.cat([a.pop("fc_mean.weight"), a.pop("fc_logstd.weight")], 0)
        a["head.bias"] = torch.cat([a.pop("fc_mean.bias"), a.pop("fc_logstd.bias")], 0)
        a.pop("action_scale", None), a.pop("action_bias", None)
        self.actor.load(a)
        self.qf.load(qf)
        self.qf_target.load(qf_target)
        with torch.no_grad():
            self.alpha.views["log_alpha"].copy_(torch.as_tensor(log_alpha).reshape(1))

    def export_reference_state(self):
        a = self.actor.state_dict()
        hw, hb = a.pop("head.weight"), a.pop("head.bias")
        a["fc_mean.weight"], a["fc_logstd.weight"] = hw[: self.A].clone(), hw[self.A:].clone()
        a["fc_mean.bias"], a["fc_logstd.bias"] = hb[: self.A].clone(), hb[self.A:].clone()
        return {"actor": a, "qf": self.qf.state_dict(), "qf_target": self.qf_target.state_dict(),
                "log_alpha": {"log_alpha": self.alpha.views["log_alpha"].detach().clone()}}
