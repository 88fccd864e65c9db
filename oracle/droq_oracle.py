"""TEST INFRASTRUCTURE (oracle) — functional fp32 restatement of one DroQ `train()` call on the CPU.

Follows: `train` sheeprl/algos/droq/droq.py:32-164; `DROQCritic` droq/agent.py:19-47 (MLP of miniblocks
Linear -> Dropout(p) -> LayerNorm(H) -> ReLU, sheeprl/utils/model.py:34-88, then Linear); `DROQAgent`
droq/agent.py:50-267; the actor, losses and Adam as oracle/sac_oracle.py.

Noise is injected: `eps_next[g]` / `eps_cur` for the two kinds of `Normal.rsample` calls and the dropout keep masks as
bool tensors [4G+2, n, B, H] in the reference's call order (per minibatch g: slots 4g, 4g+1 the target critics' two
layers, 4g+2, 4g+3 the online critics'; slots 4G, 4G+1 the policy loss's), each slot holding all n critics.
Parity PINNED: tests/golden/droq_*.pt come from the executed reference (oracle/make_golden_droq.py).  The
`exp=droq`-sized fixture starts from `init_params` (a seed) and keeps each parameter tensor at the fixed entries
`sample_index` names (`sample_state`), so it stays small.
"""
from __future__ import annotations

import zlib
from typing import Dict, List

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle.sac_oracle import actor_forward

LN_EPS = 1e-5


def layout(p: float):
    return ((0, 4, 8), (2, 6)) if p > 0 else ((0, 3, 6), (1, 4))


def init_params(obs_dim: int, act_dim: int, hidden: int, n_critics: int, p: float, seed: int, alpha: float = 1.0):
    """torch.nn.Linear default init (uniform +-1/sqrt(fan_in)), LayerNorm (1, 0); reference key names"""
    from oracle.sac_oracle import init_params as sac_init

    P = sac_init(obs_dim, act_dim, hidden, 0, seed, alpha)
    g = torch.Generator().manual_seed(seed + 1)
    lin, ln = layout(p)
    qf: Dict[str, Tensor] = {}
    for i in range(n_critics):
        for j, (fan_in, fan_out) in enumerate(((obs_dim + act_dim, hidden), (hidden, hidden), (hidden, 1))):
            b = fan_in ** -0.5
            qf[f"{i}.model._model.{lin[j]}.weight"] = (torch.rand(fan_out, fan_in, generator=g) * 2 - 1) * b
            qf[f"{i}.model._model.{lin[j]}.bias"] = (torch.rand(fan_out, generator=g) * 2 - 1) * b
            if j < 2:
                qf[f"{i}.model._model.{ln[j]}.weight"] = torch.ones(hidden)
                qf[f"{i}.model._model.{ln[j]}.bias"] = torch.zeros(hidden)
    P["qf"], P["qf_target"] = qf, {k: v.clone() for k, v in qf.items()}
    return P


def critic_forward(P: Dict[str, Tensor], i: int, x: Tensor, p: float, keep: List[Tensor]) -> Tensor:
    """critic i on x = [obs | act]; keep = the bool masks [B, H] of its two dropout layers"""
    lin, ln = layout(p)
    m = f"{i}.model._model"
    for j in range(2):
        x = x @ P[f"{m}.{lin[j]}.weight"].t() + P[f"{m}.{lin[j]}.bias"]
        if p > 0:
            x = x * (keep[j].to(x.dtype) * (torch.tensor(1.0) / (1.0 - p)))
        x = torch.relu(F.layer_norm(x, (x.shape[-1],), P[f"{m}.{ln[j]}.weight"], P[f"{m}.{ln[j]}.bias"], LN_EPS))
    return x @ P[f"{m}.{lin[2]}.weight"].t() + P[f"{m}.{lin[2]}.bias"]


def _q_all(P, x, n, p, keep2):
    """[B, n] from a [2, n, B, H] slot pair"""
    return torch.cat([critic_forward(P, i, x, p, [keep2[0, i], keep2[1, i]] if p > 0 else []) for i in range(n)], -1)


def droq_train(P, opt_qf, opt_actor, opt_alpha, critic_data: Dict[str, Tensor], actor_obs: Tensor, eps_next: Tensor,
               eps_cur: Tensor, keep: Tensor, gamma: float, tau: float, n: int, p: float, scale: Tensor, bias: Tensor,
               target_entropy: float):
    """One `train()` call; P mutated in place.  Returns the G*n value losses (reference order), policy and alpha loss."""
    actor, qf, tgt, la = P["actor"], P["qf"], P["qf_target"], P["log_alpha"]
    B = actor_obs.shape[0]
    G = critic_data["observations"].shape[0] // B
    value_losses = []
    for g in range(G):
        d = {k: v[g * B:(g + 1) * B] for k, v in critic_data.items()}
        alpha = float(la["log_alpha"].exp())
        with torch.no_grad():
            a2, logp2 = actor_forward(actor, d["next_observations"], eps_next[g], scale, bias)
            q2 = _q_all(tgt, torch.cat([d["next_observations"], a2], -1), n, p, keep[4 * g:4 * g + 2])
            y = d["rewards"] + (1 - d["terminated"]) * gamma * (q2.min(-1, keepdim=True)[0] - alpha * logp2)
        qp = {k: v.detach().requires_grad_(True) for k, v in qf.items()}
        q = _q_all(qp, torch.cat([d["observations"], d["actions"]], -1), n, p, keep[4 * g + 2:4 * g + 4])
        losses = [F.mse_loss(q[:, i:i + 1], y) for i in range(n)]
        grads = torch.autograd.grad(sum(losses), list(qp.values()))
        opt_qf.step(qf, dict(zip(qp.keys(), grads)))
        value_losses += [float(v.detach()) for v in losses]
        with torch.no_grad():
            for k in tgt:
                tgt[k].copy_(tau * qf[k] + (1 - tau) * tgt[k])
    alpha = float(la["log_alpha"].exp())
    ap = {k: v.detach().requires_grad_(True) for k, v in actor.items()}
    act, logp = actor_forward(ap, actor_obs, eps_cur, scale, bias)
    qn = _q_all(qf, torch.cat([actor_obs, act], -1), n, p, keep[4 * G:4 * G + 2])
    actor_loss = (alpha * logp - qn.mean(-1, keepdim=True)).mean()
    grads = torch.autograd.grad(actor_loss, list(ap.values()))
    opt_actor.step(actor, dict(zip(ap.keys(), grads)))
    lp = la["log_alpha"].detach().requires_grad_(True)
    alpha_loss = (-lp * (logp.detach() + target_entropy)).mean()
    (ga,) = torch.autograd.grad(alpha_loss, [lp])
    opt_alpha.step(la, {"log_alpha": ga})
    return {"Loss/value_loss": value_losses, "Loss/policy_loss": float(actor_loss.detach()),
            "Loss/alpha_loss": float(alpha_loss.detach())}


def draw_noise(G: int, B: int, A: int, n: int, H: int, p: float, seed: int):
    """eps_next [G, B, A], eps_cur [B, A], keep [4G+2, n, B, H] (bool) from one seeded generator"""
    g = torch.Generator().manual_seed(seed)
    eps_next = torch.randn(G, B, A, generator=g)
    eps_cur = torch.randn(B, A, generator=g)
    keep = torch.rand(4 * G + 2, n, B, H, generator=g) >= p
    return eps_next, eps_cur, keep


def reference_call_order(keep: Tensor, G: int, n: int) -> List[Tensor]:
    """the [B, H] masks of `keep` in the order the reference calls F.dropout"""
    out = []
    for g in range(G):
        for base in (4 * g, 4 * g + 2):
            for i in range(n):
                out += [keep[base, i], keep[base + 1, i]]
    for i in range(n):
        out += [keep[4 * G, i], keep[4 * G + 1, i]]
    return out


SAMPLE = 2048                  # entries kept per parameter tensor by the large fixture


def sample_index(name: str, numel: int, k: int = SAMPLE) -> Tensor:
    """the fixed entries of a parameter tensor (all of them when it has at most k) that a large fixture keeps"""
    if numel <= k:
        return torch.arange(numel)
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    return torch.randperm(numel, generator=g)[:k].sort().values


def sample_state(state: Dict[str, Dict[str, Tensor]]) -> Dict[str, Dict[str, Tensor]]:
    """{group: {key: tensor}} -> the same keys holding the 1-D sampled entries (sample_index of "group/key")"""
    return {g: {k: v.detach().cpu().reshape(-1)[sample_index(f"{g}/{k}", v.numel())].clone() for k, v in d.items()}
            for g, d in state.items()}
