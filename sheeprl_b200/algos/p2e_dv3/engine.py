"""Kernel schedule of one Plan2Explore (Dreamer-V3) exploration update — SURVEY §8f-4.

Reference being replaced: `train` sheeprl/algos/p2e_dv3/p2e_dv3_exploration.py:41-520 (discrete or continuous
`scaled_normal` actions).  The world
model, the rollout machinery, the actor / critic updates and every kernel are the Dreamer-V3 engine's
(`sheeprl_b200/engine.py`); this class adds what Plan2Explore adds:

  * ensemble learning (:212-240): N MLPs [z_t, h_t, a_t] -> z_{t+1}, squared error, ONE flat Adam group for the
    members the reference leaves unclipped and one for the last member — the reference's `clip_gradients(module=ens)`
    after the loop clips the last member only, and parity keeps that;
  * the exploration behaviour (:242-392): rollout with the exploration actor; per critic of `critics_exploration` its
    values, its reward (intrinsic = variance of the ensemble's next-state predictions, mean over the state, times
    `intrinsic_reward_multiplier`; or the task reward head), its lambda-values and Moments; the advantages are mixed
    by weight — the policy loss is linear in the advantage, so the fused policy kernel runs once per critic with
    scale = weight share and the entropy bonus folded into the first call.  Continuous actions (objective = advantage,
    :314-315): each critic's lambda-values and baseline (and the reward head, for task-reward critics) send their
    weight share of the gradient into the imagined states, and ONE backward through the rollout carries the sum into
    the exploration actor; the ensembles see the detached trajectory (:279-283), so the intrinsic reward is a constant;
  * the task behaviour (:397-474): the plain Dreamer-V3 behaviour step on the task actor / critic.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional, Sequence

import torch

from sheeprl_b200.engine import TWOHOT_HIGH, TWOHOT_LOW, DV3Engine, _MLP, dv3_param_shapes
from sheeprl_b200.lib import sync_deterministic
from sheeprl_b200.params import FlatGroup


def ensemble_param_shapes(cfg, actions_dim: Sequence[int], members: Sequence[int]) -> "OrderedDict[str, tuple]":
    """keys of `nn.ModuleList([MLP(...)])` (p2e_dv3/agent.py:174-200) restricted to `members`"""
    a, w = cfg.algo, cfg.algo.world_model
    Z = w.stochastic_size * w.discrete_size
    d_in = Z + w.recurrent_model.recurrent_state_size + int(sum(actions_dim))
    hid, nh = a.ensembles.dense_units, a.ensembles.mlp_layers
    out = OrderedDict()
    for i in members:
        for k in range(nh):
            out[f"{i}._model.{3 * k}.weight"] = (hid, d_in if k == 0 else hid)
            out[f"{i}._model.{3 * k + 1}.weight"] = (hid,)
            out[f"{i}._model.{3 * k + 1}.bias"] = (hid,)
        out[f"{i}._model.{3 * nh}.weight"] = (Z, hid)
        out[f"{i}._model.{3 * nh}.bias"] = (Z,)
    return out


class P2EDV3Engine(DV3Engine):
    METRIC_NAMES_P2E = ("Loss/ensemble_loss", "Loss/policy_loss_exploration")

    def __init__(self, cfg, actions_dim: Sequence[int], in_channels: int = 3, device="cuda", ops=None,
                 is_continuous: bool = False, mlp_dims=None, cnn_dims=None):
        if cfg.algo.world_model.decoupled_rssm:
            raise NotImplementedError(
                "Plan2Explore cannot run with decoupled_rssm: the reference's exploration train() calls the five-argument "
                "RSSM.dynamic (p2e_dv3_exploration.py:136), which DecoupledRSSM does not have")
        super().__init__(cfg, actions_dim, in_channels, device, ops, is_continuous=is_continuous, mlp_dims=mlp_dims,
                         cnn_dims=cnn_dims)
        a = cfg.algo
        N, H, L, A, Z = self.N, self.H, self.L, self.A, self.Z
        M1, M0 = (H + 1) * N, H * N
        b = self._buf
        _, ac_s, cr_s, _ = dv3_param_shapes(cfg, self.actions_dim, in_channels, self.is_continuous,
                                            dict(zip(self.vec_keys, self.vec_dims)), self.cnn_dims)
        # ---- exploration actor and critics
        self.actor_expl = FlatGroup(ac_s, device)
        self.actor_expl_mlp = _MLP(self, self.actor_expl, "model._model.", L, self.du, self.nh, None, M1, self.eps,
                                   "actor_expl", True)
        self.critics_expl: "OrderedDict[str, dict]" = OrderedDict()
        for k, v in a.critics_exploration.items():
            if v.weight > 0:
                grp, tgt = FlatGroup(cr_s, device), FlatGroup(cr_s, device, with_optimizer=False)
                self.critics_expl[k] = dict(
                    weight=float(v.weight), reward_type=str(v.reward_type), group=grp, target=tgt,
                    mlp=_MLP(self, grp, "_model.", L, self.du, self.nh, self.bins_c, M1, self.eps, f"critic_expl_{k}", True),
                    target_mlp=_MLP(self, tgt, "_model.", L, self.du, self.nh, self.bins_c, M0, self.eps, f"target_expl_{k}", False),
                    moments_state=b(f"moments_state_{k}", 2), moments_out=b(f"moments_out_{k}", 2),
                    values=b(f"values_{k}", H + 1, N), lam=b(f"lam_{k}", H, N), reward_mean=b(f"reward_mean_{k}", 1),
                    values_mean=b(f"values_mean_{k}", 1), lam_mean=b(f"lam_mean_{k}", 1), value_loss=b(f"value_loss_{k}", 1),
                    policy_rows=b(f"policy_rows_{k}", M0) if self.is_continuous else None)
        if not any(c["reward_type"] == "intrinsic" for c in self.critics_expl.values()):
            raise RuntimeError("You must specify at least one intrinsic critic (`reward_type='intrinsic'`)")
        # ---- ensembles
        self.n_ens = int(a.ensembles.n)
        rest = list(range(self.n_ens - 1))
        self.ens_rest = FlatGroup(ensemble_param_shapes(cfg, self.actions_dim, rest), device) if rest else None
        self.ens_last = FlatGroup(ensemble_param_shapes(cfg, self.actions_dim, [self.n_ens - 1]), device)
        eh, el = a.ensembles.dense_units, a.ensembles.mlp_layers
        self.ens_mlps = [_MLP(self, self.ens_last if i == self.n_ens - 1 else self.ens_rest, f"{i}._model.", L + A, eh, el, Z,
                              M1, self.eps, f"ens{i}", True) for i in range(self.n_ens)]
        self.ens_in = b("ens_in", M1, L + A)
        self.z_next = b("z_next", N, Z)
        self.ens_rows = b("ens_rows", M1)
        self.d_ens_out = b("d_ens_out", N, Z)
        self.ens_mean = b("ens_mean", M1, Z)
        self.ens_scratch = b("ens_scratch", M1, Z)
        self.intr_reward = b("intr_reward", H + 1, N)
        self.d_actor_raw_k = b("d_actor_raw_k", M0, self.AW)
        self.policy_rows_k = b("policy_rows_k", M0)
        self.p2e_metrics = b("p2e_metrics", 4)          # ensemble loss, exploration policy loss, scratch x2
        self.unit_moments = b("unit_moments", 2)
        self.unit_moments[1] = 1.0
        # norms: wm, actor_task, critic_task (base slots 0-2), ens(last member), actor_expl, critics_expl...
        self.norms = b("norms_p2e", 6 + len(self.critics_expl))       # last slot: scratch (norm of the unclipped members)
        for name in ["ens_rest", "ens_last", "actor_expl"] + [f"critic_expl_{k}" for k in self.critics_expl]:
            self.normsq[name] = self._buf(f"normsq_{name}", (), dtype=torch.float64)
        # per-phase noise (parity mode) / Philox streams (production)
        self.noise_img_state_expl = b("noise_img_state_expl", H, N, Z)
        self.noise_img_action_expl = b("noise_img_action_expl", H + 1, N, A)

    # ------------------------------------------------------------------ state access used by agent.py / tests
    def extra_groups(self):
        """flat groups beyond wm / actor / critic (the optimizer handles of the reference's main attach to these)"""
        d = {"actor_expl": self.actor_expl, "ens_last": self.ens_last}
        if self.ens_rest is not None:
            d["ens_rest"] = self.ens_rest
        for k, c in self.critics_expl.items():
            d[f"critic_expl_{k}"] = c["group"]
        return d

    def optimizer_groups(self):
        return super().optimizer_groups() + list(self.extra_groups().values())

    def groups(self) -> "OrderedDict[str, FlatGroup]":
        out = OrderedDict(wm=self.wm, actor_task=self.actor, critic_task=self.critic, target_task=self.target,
                          actor_expl=self.actor_expl)
        for k, c in self.critics_expl.items():
            out[f"critic_expl_{k}"], out[f"target_expl_{k}"] = c["group"], c["target"]
        return out

    def load_ensembles(self, state: Dict[str, torch.Tensor]):
        last = f"{self.n_ens - 1}."
        if self.ens_rest is not None:
            self.ens_rest.load({k: v for k, v in state.items() if not k.startswith(last)})
        self.ens_last.load({k: v for k, v in state.items() if k.startswith(last)})

    def ensembles_state_dict(self) -> "OrderedDict[str, torch.Tensor]":
        out = OrderedDict()
        if self.ens_rest is not None:
            out.update(self.ens_rest.state_dict())
        out.update(self.ens_last.state_dict())
        return out

    # ------------------------------------------------------------------ the step
    def train_step(self, data: Dict[str, torch.Tensor], noise: Optional[Dict[str, torch.Tensor]] = None):
        """noise (parity mode): {"post", "img_state_expl", "img_action_expl", "img_state_task", "img_action_task"}"""
        ops = self.ops
        sync_deterministic(ops)
        N, H, Z = self.N, self.H, self.Z
        if noise is None:
            self._draw_noise(None)                                                   # post / task rollout streams 0-2
            ops.fill_exponential(self.noise_img_state_expl.view(-1), self.rng_seed, 3, self.rng_t)
            fill = ops.fill_normal if self.is_continuous else ops.fill_exponential
            if not self.minedojo:                                     # the MineDojo actors imagine mode actions
                fill(self.noise_img_action_expl.view(-1), self.rng_seed, 4, self.rng_t)
        else:
            self._draw_noise({"post": noise["post"], "img_state": noise["img_state_task"],
                              "img_action": noise.get("img_action_task")})
            self.noise_img_state_expl.copy_(noise["img_state_expl"].reshape(H, N, Z))
            if not self.minedojo:
                self.noise_img_action_expl.copy_(torch.cat([x for x in noise["img_action_expl"]], -1))
        self._world_model_phase(data, heads_detached=True)
        self._ensemble_learning(data)
        # the exploration rollout and its losses (the continuous backward re-reads the action noise) use their own noise;
        # the task rollout afterwards the base buffers.  The exploration losses finish before the task rollout
        # overwrites the kept rollout activations.
        task_noise = (self.noise_img_state, self.noise_img_action)
        self.noise_img_state, self.noise_img_action = self.noise_img_state_expl, self.noise_img_action_expl
        try:
            self._imagine(self.actor_expl, self.actor_expl_mlp)
            self._exploration_losses()
        finally:
            self.noise_img_state, self.noise_img_action = task_noise
        self._imagine()
        self._behaviour_losses()
        return self.metrics

    # ------------------------------------------------------------------ ensembles
    def _ensemble_learning(self, data: Dict[str, torch.Tensor]):
        ops, N, B, L, A, Z = self.ops, self.N, self.B, self.L, self.A, self.Z
        a = self.cfg.algo
        M = N - B                                                    # (T-1)*B transitions
        x = self.ens_in[:N]
        ops.copy(self.latent, x[:, :L])
        ops.copy(data["actions"].reshape(N, A), x[:, L:])            # the action taken AT step t (not the shifted one)
        ops.copy(self.latent[B:, :Z], self.z_next[:M])
        ops.zero(self.ens_last.grad)
        if self.ens_rest is not None:
            ops.zero(self.ens_rest.grad)
        ops.zero(self.p2e_metrics[0:1])
        x = x[:M]                                                    # the last step has no successor
        for m in self.ens_mlps:
            out = m.forward(x, M=M)
            ops.mse_loss_grad(out, self.z_next[:M], 1.0 / M, self.ens_rows[:M], self.d_ens_out[:M])
            ops.sum_rows(self.ens_rows[:M].view(M, 1), self.p2e_metrics[2:3], 1.0 / M)
            ops.axpy(self.p2e_metrics[2:3], self.p2e_metrics[0:1])
            m.backward(x, self.d_ens_out[:M], None, False, M=M)
        o = a.ensembles.optimizer
        if self.ens_rest is not None:
            self._optimizer_step("ens_rest", self.ens_rest, 0.0, o, self.norms.numel() - 1)
        self._optimizer_step("ens_last", self.ens_last, float(a.ensembles.clip_gradients or 0.0), o, 3)

    def _intrinsic_reward(self):
        """reward[t, n] = multiplier * mean_z Var_i(ens_i([traj, actions]))  (unbiased variance over the members)"""
        ops, N, H, L, Z = self.ops, self.N, self.H, self.L, self.Z
        M1 = (H + 1) * N
        n = self.n_ens
        x = self.ens_in
        ops.copy(self.traj.view(M1, L), x[:, :L])
        ops.copy(self.actions.view(M1, self.A), x[:, L:])
        outs = [m.forward(x) for m in self.ens_mlps]
        ops.zero(self.ens_mean)
        for o in outs:
            ops.axpy(o, self.ens_mean, 1.0 / n)
        ops.zero(self.intr_reward)
        scale = float(self.cfg.algo.intrinsic_reward_multiplier) / (Z * max(n - 1, 1))
        for o in outs:
            ops.mse_loss_grad(o, self.ens_mean, 0.0, self.ens_rows, self.ens_scratch)     # row sums of (x_i - mean)^2
            ops.axpy(self.ens_rows, self.intr_reward.view(-1), scale)

    # ------------------------------------------------------------------ exploration behaviour
    def _exploration_losses(self):
        ops, N, H, L = self.ops, self.N, self.H, self.L
        a = self.cfg.algo
        M1, M0 = (H + 1) * N, H * N
        traj2 = self.traj.view(M1, L)
        c_logit = self.cont_img.forward(traj2)
        mo = a.actor.moments
        weights_sum = sum(c["weight"] for c in self.critics_expl.values())
        v_logits, r_logits = {}, None
        for k, c in self.critics_expl.items():
            v_logits[k] = c["mlp"].forward(traj2)
            ops.twohot_mean(v_logits[k], TWOHOT_LOW, TWOHOT_HIGH, c["values"].view(-1))
            if c["reward_type"] == "intrinsic":
                self._intrinsic_reward()
                rew = self.intr_reward
            else:
                r_logits = self.rew_img.forward(traj2)
                ops.twohot_mean(r_logits, TWOHOT_LOW, TWOHOT_HIGH, self.rew_pred.view(-1))
                rew = self.rew_pred
            ops.sum_rows(rew.view(M1, 1), c["reward_mean"], 1.0 / M1)
            ops.lambda_returns(rew, c["values"], c_logit.view(H + 1, N), self.true_cont, float(a.gamma), float(a.lmbda),
                               c["lam"], self.discount)
            lam_all = c["lam"] if self.allgather is None else self.allgather(c["lam"])
            ops.moments_update(lam_all.view(-1), c["moments_state"], float(mo.decay), float(mo.max),
                               float(mo.percentile.low), float(mo.percentile.high), c["moments_out"])
            ops.sum_rows(c["values"].view(M1, 1), c["values_mean"], 1.0 / M1)
            ops.sum_rows(c["lam"].view(M0, 1), c["lam_mean"], 1.0 / M0)
        ops.zero(self.p2e_metrics[1:2])
        if self.is_continuous:
            # ---- policy: loss = -mean(D * (sum_k share_k * adv_k + ent_coef * ent)), differentiated through the rollout
            self._continuous_policy_gradient(c_logit, [
                (c["mlp"], v_logits[k], c["values"], c["lam"], c["moments_out"], c["weight"] / weights_sum,
                 None if c["reward_type"] == "intrinsic" else r_logits, c["policy_rows"])
                for k, c in self.critics_expl.items()])
            for c in self.critics_expl.values():
                ops.sum_rows(c["policy_rows"].view(M0, 1), self.p2e_metrics[2:3], -c["weight"] / weights_sum / M0)
                ops.axpy(self.p2e_metrics[2:3], self.p2e_metrics[1:2])
        else:
            # ---- policy: loss = -mean(D * (logp * sum_k share_k * adv_k + ent_coef * ent)); linear in the advantage
            for j, (k, c) in enumerate(self.critics_expl.items()):
                share = c["weight"] / weights_sum
                rows, draw = (self.policy_rows, self.d_actor_raw) if j == 0 else (self.policy_rows_k, self.d_actor_raw_k)
                ops.actor_loss_grad(self.actor_raw[:M0], self.actions.view(M1, self.A)[:M0], c["lam"].view(-1),
                                    c["values"].view(-1)[:M0], self.discount.view(-1)[:M0], c["moments_out"],
                                    self.actions_dim, self.unimix, float(a.actor.ent_coef) / share if j == 0 else 0.0,
                                    share / M0, rows, draw)
                ops.sum_rows(rows.view(M0, 1), self.p2e_metrics[2:3], -share / M0)
                ops.axpy(self.p2e_metrics[2:3], self.p2e_metrics[1:2])
                if j > 0:
                    ops.axpy(self.d_actor_raw_k, self.d_actor_raw)
        self._actor_update(self.actor_expl, self.actor_expl_mlp, "actor_expl", 4)
        for j, (k, c) in enumerate(self.critics_expl.items()):
            self._critic_update(c["group"], c["mlp"], c["target_mlp"], v_logits[k], c["lam"], c["value_loss"],
                                f"critic_expl_{k}", 5 + j)

    # ------------------------------------------------------------------ metrics / targets
    def metrics_dict(self) -> Dict[str, torch.Tensor]:
        d = {n: self.metrics[i] for i, n in enumerate(self.METRIC_NAMES[:8])}
        d["Loss/policy_loss_task"], d["Loss/value_loss_task"] = self.metrics[8], self.metrics[9]
        d["Loss/ensemble_loss"], d["Loss/policy_loss_exploration"] = self.p2e_metrics[0], self.p2e_metrics[1]
        d["Grads/world_model"], d["Grads/actor_task"], d["Grads/critic_task"] = self.norms[0], self.norms[1], self.norms[2]
        d["Grads/ensemble"], d["Grads/actor_exploration"] = self.norms[3], self.norms[4]
        for j, (k, c) in enumerate(self.critics_expl.items()):
            d[f"Loss/value_loss_exploration_{k}"] = c["value_loss"][0]
            d[f"Grads/critic_exploration_{k}"] = self.norms[5 + j]
            d[f"Values_exploration/predicted_values_{k}"] = c["values_mean"][0]
            d[f"Values_exploration/lambda_values_{k}"] = c["lam_mean"][0]
            if c["reward_type"] == "intrinsic":
                d[f"Rewards/intrinsic_{k}"] = c["reward_mean"][0]
        return d

    def update_targets(self, tau: float):
        """EMA of the task target critic and of every exploration target critic (p2e_dv3_exploration.py:866-880)"""
        self.update_target(tau)
        for c in self.critics_expl.values():
            if tau >= 1.0:
                self.ops.copy(c["group"].flat, c["target"].flat)
            else:
                self.ops.ema(c["target"].flat, c["group"].flat, float(tau))
