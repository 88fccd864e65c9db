"""TEST INFRASTRUCTURE — executable specification (plain fp32 torch, CPU) of the C-ABI ops Dreamer-V2's update adds to
`include/b200rl.h` (`b200rl_adam_step_wd`), on top of the `oracle/ops_emul.py::EmulOps` specification of every other
op.  Same two uses: `-m gpu` tests compare each CUDA kernel against the method of the same name, and `-m "not gpu"`
tests inject this object into an engine (test double) to walk its schedule on a GPU-less host.  The product never
constructs it.
"""
from __future__ import annotations

from oracle.ops_emul import EmulOps


class DV2EmulOps(EmulOps):
    def adam_step(self, p, g, m, v, normsq, max_norm, lr, b1, b2, eps, step_t, norm_out, weight_decay=0.0):
        """clip_grad_norm_(max_norm) folded into torch.optim.Adam(weight_decay=...)'s single-tensor update: the L2 term
        is added to the clipped gradient (torch/optim/adam.py `grad = grad.add(param, alpha=weight_decay)`), so it
        enters both moments"""
        if weight_decay == 0:
            return super().adam_step(p, g, m, v, normsq, max_norm, lr, b1, b2, eps, step_t, norm_out)
        step = int(step_t.item())
        total = normsq.sqrt().float()
        norm_out.copy_(total)
        coef = (max_norm / (total + 1e-6)).clamp(max=1.0) if max_norm > 0 else 1.0
        gg = (g * coef).add(p, alpha=weight_decay)
        m.lerp_(gg, 1 - b1)
        v.mul_(b2).addcmul_(gg, gg, value=1 - b2)
        denom = (v.sqrt() / (1 - b2 ** step) ** 0.5).add_(eps)
        p.addcdiv_(m, denom, value=-lr / (1 - b1 ** step))
