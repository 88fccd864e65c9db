"""TEST INFRASTRUCTURE (oracle) — a functional fp32 torch restatement of A2C's `train()` (sheeprl/algos/a2c/a2c.py:26-114):
one epoch of minibatches, each minibatch's loss back-propagated into the same gradients, one clip and one optimizer
step at the end.  The model is PPO's (`oracle/ppo_oracle.py::ppo_forward`); the optimizer is torch's own RMSprop / Adam
over the parameter tensors (single-tensor path, as the reference runs on the CPU).
Parity PINNED: tests/golden/a2c_*.pt come from the executed reference train() (oracle/make_golden_a2c.py).
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch

from oracle import ppo_oracle as PO


def init_params(spec, seed: int) -> Dict[str, torch.Tensor]:
    """Deterministic initial parameters (CPU torch.Generator draws, identical on every host), so the fixtures store a
    seed: weights and biases U(-1/sqrt(fan_in), 1/sqrt(fan_in)), LayerNorm weights 1 + N(0, 0.1) and biases N(0, 0.1)."""
    g = torch.Generator().manual_seed(seed)
    out, shapes = {}, PO.ppo_param_shapes(spec)
    ln = {k for k, s in shapes.items() if k.endswith(".weight") and len(s) == 1}
    ln |= {k[:-6] + "bias" for k in ln}
    fan = 1
    for k, s in shapes.items():
        if k in ln:
            out[k] = (1.0 if k.endswith(".weight") else 0.0) + 0.1 * torch.randn(*s, generator=g)
            continue
        if k.endswith(".weight"):
            fan = 1
            for d in s[1:]:
                fan *= d
        out[k] = (torch.rand(*s, generator=g) * 2 - 1) / fan ** 0.5
    return out


def make_optimizer(p: Dict[str, torch.Tensor], opt_cfg: dict) -> torch.optim.Optimizer:
    """torch's RMSprop / Adam over the oracle's parameter tensors (made leaves that require grad) from an optimizer
    config ({"_target_": ..., lr, ...} as configs/optim/*.yaml writes it)"""
    for v in p.values():
        v.requires_grad_(True)
    kw = {k: v for k, v in opt_cfg.items() if not k.startswith("_")}
    cls = torch.optim.Adam if opt_cfg.get("_target_", "").endswith("Adam") else torch.optim.RMSprop
    return cls(list(p.values()), foreach=False, **kw)


def replay_updates(init: Dict[str, torch.Tensor], opt_cfg: dict, grads: Sequence[Dict[str, torch.Tensor]]):
    """the parameters after one optimizer step per recorded gradient, from `init`, with torch's own optimizer on the
    CPU: what the reference's optimizer.step() computed from those gradients (make_golden_a2c.py checks the two are
    bit-identical), so the fixtures store the gradients and not the parameters as well"""
    p = {k: v.clone() for k, v in init.items()}
    opt = make_optimizer(p, opt_cfg)
    for g in grads:
        for k, t in p.items():
            t.grad = g[k].clone()
        opt.step()
    return {k: v.detach() for k, v in p.items()}


def a2c_losses(lp, ent, values, batch, hp):
    """policy_loss (a2c/loss.py), value_loss (mse) and entropy_loss (ppo/loss.py:66-75) with loss_reduction"""
    adv = batch["advantages"]
    if hp["normalize_advantages"]:
        adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    red = (lambda x: x.sum()) if hp["loss_reduction"] == "sum" else (lambda x: x.mean())
    return red(-(lp * adv)), red((values - batch["returns"]) ** 2), red(-ent)


def a2c_train(p: Dict[str, torch.Tensor], opt: torch.optim.Optimizer, spec, data: Dict[str, torch.Tensor],
              index_batches: Sequence[Sequence[int]], hp, grads_out: Dict[str, torch.Tensor] = None) -> List[Dict[str, float]]:
    """one train() call over the given minibatch index lists; mutates p / opt.  data: flat [N, ...] float tensors (rgb
    raw 0..255 as float).  `grads_out` (optional) receives the accumulated, clipped gradient the optimizer stepped with."""
    logs = []
    opt.zero_grad(set_to_none=True)
    for idx in index_batches:
        idx = torch.as_tensor(idx)
        batch = {k: v[idx] for k, v in data.items()}
        obs = {}
        if spec["cnn_channels"]:
            obs["rgb"] = batch["rgb"] / 255 - 0.5
        if spec["mlp_dim"]:
            obs["state"] = batch["state"]
        lp, ent, values = PO.ppo_forward(p, spec, obs, batch["actions"])
        pg, v, e = a2c_losses(lp, ent, values, batch, hp)
        (pg + hp["vf_coef"] * v + hp["ent_coef"] * e).backward()
        logs.append({"Loss/policy_loss": float(pg.detach()), "Loss/value_loss": float(v.detach()),
                     "Loss/entropy_loss": float(e.detach())})
    if hp["max_grad_norm"] > 0:
        torch.nn.utils.clip_grad_norm_(list(p.values()), hp["max_grad_norm"])
    if grads_out is not None:
        grads_out.update({k: t.grad.detach().clone() for k, t in p.items()})
    opt.step()
    return logs
