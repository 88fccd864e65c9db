"""TEST INFRASTRUCTURE — executable specification (plain fp32 torch, CPU) of the A2C C-ABI ops in `include/b200rl.h`
(`b200rl_a2c_loss`, `b200rl_rmsprop_step`), on top of the `oracle/ops_emul.py::EmulOps` specification of every other
op.  Same two uses: `-m gpu` tests compare each CUDA kernel against the method of the same name, and `-m "not gpu"`
tests inject this object into `A2CEngine` (test double) to walk the engine's schedule on a GPU-less host.  The product
never constructs it.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.ops_emul import EmulOps
from oracle.ppo_oracle import SAFE_LIM


def logp_entropy(head, actions, head_dims, is_continuous):
    """log-prob of the taken action and entropy per row (ppo/agent.py:179-239), differentiable in `head`"""
    if is_continuous:
        mean, ls = head.chunk(2, -1)
        sd = ls.exp()
        corr = 0.0
        if int(is_continuous) == 2:          # tanh_normal: stored actions are squashed (ppo/agent.py:194-206)
            corr = 2.0 * (math.log(2.0) - actions - F.softplus(-2.0 * actions)).sum(-1)
            actions = torch.atanh(actions.clamp(-SAFE_LIM, SAFE_LIM))
        lp = (-((actions - mean) ** 2) / (2 * sd * sd) - ls - math.log(math.sqrt(2 * math.pi))).sum(-1) - corr
        return lp, (0.5 + 0.5 * math.log(2 * math.pi) + ls).sum(-1)
    lp, ent, off = 0.0, 0.0, 0
    for n in head_dims:
        logp = torch.log_softmax(head[:, off:off + n], -1)
        lp = lp + (logp * actions[:, off:off + n]).sum(-1)
        ent = ent - (logp.exp() * logp).sum(-1)
        off += n
    return lp, ent


class A2CEmulOps(EmulOps):
    def a2c_loss(self, head, actions, adv, values, returns, dhead, dvalues, losses, seg, head_dims, is_continuous,
                 normalize_adv, reduce_sum, vf_coef, ent_coef):
        """per minibatch i (rows [i*seg, min(N, (i+1)*seg))): a2c/a2c.py:79-100 with loss_reduction sum / mean"""
        N = head.shape[0]
        red = (lambda x: x.sum()) if reduce_sum else (lambda x: x.mean())
        for i, r0 in enumerate(range(0, N, seg)):
            rows = slice(r0, min(N, r0 + seg))
            if normalize_adv and rows.stop - rows.start < 2:
                raise ValueError("advantage normalisation needs at least two rows in every minibatch")
            h = head[rows].detach().clone().requires_grad_(True)
            v = values[rows].detach().clone().requires_grad_(True)
            lp, ent = logp_entropy(h, actions[rows], head_dims, is_continuous)
            a = adv[rows]
            if normalize_adv:
                a = (a - a.mean()) / (a.std() + 1e-8)
            pg, vl, el = red(-(lp * a)), red((v - returns[rows]) ** 2), red(-ent)
            gh, gv = torch.autograd.grad(pg + vf_coef * vl + ent_coef * el, [h, v])
            dhead[rows], dvalues[rows] = gh, gv
            losses[i] = torch.stack([pg, vl, el]).detach()

    def rmsprop_step(self, p, g, square_avg, momentum_buf, grad_avg, normsq, max_norm, lr, alpha, eps, weight_decay,
                     momentum, norm_out):
        """clip_grad_norm_(max_norm) folded into torch.optim.RMSprop's single-tensor update"""
        total = torch.sqrt(normsq).float()
        norm_out.copy_(total)
        coef = torch.clamp(max_norm / (total + 1e-6), max=1.0) if max_norm > 0 else torch.tensor(1.0)
        grad = g * coef
        if weight_decay != 0:
            grad = grad.add(p, alpha=weight_decay)
        square_avg.mul_(alpha).addcmul_(grad, grad, value=1 - alpha)
        if grad_avg is not None:
            grad_avg.lerp_(grad, 1 - alpha)
            avg = square_avg.addcmul(grad_avg, grad_avg, value=-1).sqrt_()
        else:
            avg = square_avg.sqrt()
        avg = avg.add_(eps)
        if momentum > 0:
            momentum_buf.mul_(momentum).addcdiv_(grad, avg)
            p.add_(momentum_buf, alpha=-lr)
        else:
            p.addcdiv_(grad, avg, value=-lr)
