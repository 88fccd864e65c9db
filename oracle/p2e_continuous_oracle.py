"""TEST INFRASTRUCTURE (oracle) — CPU restatement of one Plan2Explore / Dreamer-V3 exploration update with CONTINUOUS
`scaled_normal` actions (`sheeprl/algos/p2e_dv3/p2e_dv3_exploration.py:41-520` with is_continuous=True), on top of the
Dreamer-V3 and discrete Plan2Explore oracles' pieces.

Phases as in oracle/p2e_oracle.py; what differs is behaviour learning.  The objective is the advantage itself (:314-315,
:429-430), so the policy gradient flows from every critic's lambda-values and baseline (and the reward head, for
task-reward critics) through the imagined states, back through the rollout's dynamics into each step's action and the
actor head.  The world model, critics and ensembles act as constants; the ensembles see the detached trajectory and
actions (:279-283), so the intrinsic reward carries no gradient.

Parity PINNED: tests/golden/p2e_tiny_c.pt is written by oracle/make_golden_p2e_continuous.py from the EXECUTED
reference train().  Only tests/ may import this module.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle.dv3_oracle import (AdamState, clip_grad_norm, continuous_action, dense_stack, recurrent_step,
                               reference_normal_order, st_sample, transition_logits, twohot_mean, world_model_phase)
from oracle.p2e_oracle import _critic_update, _lambda_values, _moments, ensemble_forward


def draw_noise(T: int, B: int, H: int, S: int, D: int, actions_dim: Sequence[int], seed: int) -> Dict[str, Tensor]:
    """one update's draws: Exp(1) for the scan's posterior samples and, per behaviour phase (`_expl`, `_task`), the
    imagined states; one N(0,1) tensor [H+1, N, sum(A)] per phase for the actions"""
    g = torch.Generator().manual_seed(seed)
    N = T * B

    def exp1(*shape):
        return torch.empty(*shape).exponential_(1.0, generator=g)

    out = {"prior": exp1(T, B, S, D), "post": exp1(T, B, S, D)}
    for ph in ("expl", "task"):
        out[f"img_state_{ph}"] = exp1(H, N, S, D)
        out[f"img_action_{ph}"] = [torch.randn(H + 1, N, int(sum(actions_dim)), generator=g)]
    return out


def reference_noise_order(noise: Dict[str, Tensor], T: int, H: int) -> Tuple[List[Tensor], List[Tensor]]:
    """(torch.multinomial draws, Normal.rsample draws) in the reference's call order.  Categorical: the scan (prior then
    posterior per step), then the imagined states of each phase.  Normal, per phase: one per rollout step and one
    (discarded) for the actor's re-evaluation on the whole trajectory (:313 / :422)."""
    cat, normal = [], []
    for t in range(T):
        cat += [noise["prior"][t], noise["post"][t]]
    for ph in ("expl", "task"):
        cat += [noise[f"img_state_{ph}"][i] for i in range(H)]
        normal += reference_normal_order({"img_action": noise[f"img_action_{ph}"]}, H)
    return cat, normal


def _rollout(cfg, wm_c, actor, zs, hs, img_state, img_action, condition_margin):
    """H imagined steps with the graph kept: each action carries the gradient of the actor head and feeds the next
    dynamics step; the actor itself sees the detached state (:249, :258).
    Returns (traj [H+1,N,L], actions [H+1,N,A], entropy [H+1,N])."""
    a, w = cfg.algo, cfg.algo.world_model
    S, D = w.stochastic_size, w.discrete_size
    eps, um, n_hid, H = a.mlp_layer_norm.kw.eps, a.unimix, a.mlp_layers, a.horizon
    N = zs.shape[0] * zs.shape[1]
    zi, hi = zs.detach().reshape(N, -1), hs.detach().reshape(N, -1)
    ents = []

    def act(state, i):
        hdn = dense_stack(actor, "model._model.", state.detach(), n_hid, eps, False)
        head = F.linear(hdn, actor["mlp_heads.0.weight"], actor["mlp_heads.0.bias"])
        x, ent = continuous_action(head, img_action[0][i], a.actor)
        ents.append(ent)
        return x

    traj, acts = [torch.cat((zi, hi), -1)], []
    acts.append(act(traj[0], 0))
    for i in range(1, H + 1):
        hi = recurrent_step(wm_c, zi, acts[-1], hi, eps)
        zi = st_sample(transition_logits(wm_c, hi, S, D, um, eps), S, D, img_state[i - 1], condition_margin)
        traj.append(torch.cat((zi, hi), -1))
        acts.append(act(traj[-1], i))
    return torch.stack(traj), torch.stack(acts), torch.stack(ents)


def _behaviour(cfg, wm_c, ens_c, actor, critics, zs, hs, img_state, img_action, continues, condition_margin):
    """one behaviour phase; critics: [(weight, reward_type, params, moments)].
    Returns (detached trajectory, discount, policy loss, [(values, reward, lambda-values) per critic, detached])."""
    a = cfg.algo
    eps, n_hid = a.mlp_layer_norm.kw.eps, a.mlp_layers
    traj, acts, ent = _rollout(cfg, wm_c, actor, zs, hs, img_state, img_action, condition_margin)
    with torch.no_grad():
        cont = continues(traj)
        discount = torch.cumprod(cont * a.gamma, 0) / a.gamma
    weights_sum = sum(c[0] for c in critics)
    advantage, parts = 0.0, []
    for weight, reward_type, params, moments in critics:
        values = twohot_mean(dense_stack({k: v.detach() for k, v in params.items()}, "_model.", traj, n_hid, eps, True))
        if reward_type == "intrinsic":
            with torch.no_grad():
                x = torch.cat((traj, acts), -1)
                emb = torch.stack([ensemble_forward(ens_c, i, x, a.ensembles.mlp_layers, eps) for i in range(a.ensembles.n)])
                rew = emb.var(0).mean(-1, keepdim=True) * a.intrinsic_reward_multiplier
        else:
            rew = twohot_mean(dense_stack(wm_c, "reward_model._model.", traj, n_hid, eps, True))
        lam = _lambda_values(rew, values, cont, a.gamma, a.lmbda)
        offset, invscale = _moments(moments, lam, a.actor.moments)
        advantage = advantage + ((lam - offset) / invscale - (values[:-1] - offset) / invscale) * weight / weights_sum
        parts.append((values.detach(), rew.detach(), lam.detach()))
    policy_loss = -torch.mean(discount[:-1] * (advantage + a.actor.ent_coef * ent.unsqueeze(-1)[:-1]))
    return traj.detach(), discount, policy_loss, parts


def p2e_continuous_train_step(cfg, wm, ensembles, actor_task, critic_task, target_task, actor_expl, critics_expl,
                              opts: Dict[str, AdamState], data, noise, moments_task, actions_dim,
                              condition_margin: float = 0.0):
    """One exploration update; arguments and side effects as `oracle.p2e_oracle.p2e_train_step`."""
    a = cfg.algo
    T, B = a.per_rank_sequence_length, a.per_rank_batch_size
    N = T * B
    eps, n_hid = a.mlp_layer_norm.kw.eps, a.mlp_layers
    out: Dict[str, Tensor] = {}
    trainable = [wm, ensembles, actor_task, critic_task, actor_expl] + [c["module"] for c in critics_expl.values()]
    for d in trainable:
        for v in d.values():
            v.requires_grad_(True)
            v.grad = None

    # ---- 1. dynamic learning
    zs, hs, cont_target = world_model_phase(cfg, wm, opts["wm"], data, noise, condition_margin, False, out,
                                            detach_heads=True)
    zs, hs = zs.detach(), hs.detach()

    # ---- 2. ensemble learning (:212-240).  NB the clip covers the LAST member only (`module=ens` after the loop)
    n_ens = a.ensembles.n
    ens_in = torch.cat((zs, hs, data["actions"].float()), -1)
    loss = 0.0
    for i in range(n_ens):
        pred = ensemble_forward(ensembles, i, ens_in, a.ensembles.mlp_layers, eps)[:-1]
        loss = loss + ((pred - zs[1:]) ** 2).sum(-1).mean()
    loss.backward()
    with torch.no_grad():
        last = [v.grad for k, v in ensembles.items() if k.startswith(f"{n_ens - 1}.")]
        out["Grads/ensemble"] = clip_grad_norm(last, a.ensembles.clip_gradients)
        opts["ens"].step(ensembles, {k: v.grad for k, v in ensembles.items()})
    out["Loss/ensemble_loss"] = loss.detach()

    wm_c = {k: v.detach() for k, v in wm.items()}
    ens_c = {k: v.detach() for k, v in ensembles.items()}
    true_cont = cont_target.reshape(1, N, 1)

    def continues(traj):
        c = (torch.sigmoid(dense_stack(wm_c, "continue_model._model.", traj, n_hid, eps, True)) > 0.5).float()
        return torch.cat((true_cont, c[1:]), 0)

    # ---- 3. behaviour learning: exploration (:242-392)
    crit = [(c["weight"], c["reward_type"], c["module"], c["moments"]) for c in critics_expl.values()]
    traj, discount, policy_loss, parts = _behaviour(cfg, wm_c, ens_c, actor_expl, crit, zs, hs, noise["img_state_expl"],
                                                    noise["img_action_expl"], continues, condition_margin)
    for (name, c), (values, rew, lam) in zip(critics_expl.items(), parts):
        if c["reward_type"] == "intrinsic":
            out[f"Rewards/intrinsic_{name}"] = rew.mean()
        out[f"Values_exploration/predicted_values_{name}"] = values.mean()
        out[f"Values_exploration/lambda_values_{name}"] = lam.mean()
    policy_loss.backward()
    with torch.no_grad():
        out["Grads/actor_exploration"] = clip_grad_norm([v.grad for v in actor_expl.values()], a.actor.clip_gradients)
        opts["actor_expl"].step(actor_expl, {k: v.grad for k, v in actor_expl.items()})
    out["Loss/policy_loss_exploration"] = policy_loss.detach()
    for (name, c), (_, _, lam) in zip(critics_expl.items(), parts):
        vl, norm = _critic_update(cfg, c["module"], c["target_module"], opts[f"critic_expl_{name}"], traj, lam, discount)
        out[f"Loss/value_loss_exploration_{name}"], out[f"Grads/critic_exploration_{name}"] = vl, norm

    # ---- 4. behaviour learning: task (:397-474)
    traj, discount, policy_loss, [(_, _, lam)] = _behaviour(
        cfg, wm_c, None, actor_task, [(1.0, "task", critic_task, moments_task)], zs, hs, noise["img_state_task"],
        noise["img_action_task"], continues, condition_margin)
    policy_loss.backward()
    with torch.no_grad():
        out["Grads/actor_task"] = clip_grad_norm([v.grad for v in actor_task.values()], a.actor.clip_gradients)
        opts["actor_task"].step(actor_task, {k: v.grad for k, v in actor_task.items()})
    out["Loss/policy_loss_task"] = policy_loss.detach()
    out["Loss/value_loss_task"], out["Grads/critic_task"] = _critic_update(cfg, critic_task, target_task, opts["critic_task"],
                                                                           traj, lam, discount)
    for d in trainable:
        for v in d.values():
            v.grad = None
            v.requires_grad_(False)
    return out
