"""Kernel schedule of the A2C update: the whole accumulated update of one `train()` call in one pass.

Reference being replaced: `train` sheeprl/algos/a2c/a2c.py:26-114.  It runs ONE epoch of minibatches, back-propagates
each minibatch's loss into the same `.grad` buffers (`no_backward_sync` while accumulating) and takes one clip +
`optimizer.step()` at the end.  The update is therefore the gradient of a sum of per-minibatch losses, and every
weight gradient is a product that reduces over rows: one forward, one loss launch and one backward over all N rows of
the rollout give that sum directly.  The minibatch structure only decides which rows share a reduction scale and the
advantage-normalisation statistics, which is a per-segment detail of `a2c_loss` (one CTA per minibatch).

The model is PPO's (a2c.py:14 imports `PPOAgent` / `build_agent` from ppo/agent.py), so the parameters, buffers,
forward and backward are `PPOEngine`'s; only the objective, the schedule and the optimizer differ.
"""
from __future__ import annotations

from typing import Dict, Sequence

import torch

from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import B200Adam
from sheeprl_b200.algos.ppo.engine import PPOEngine

INT32_MAX = 2 ** 31 - 1


class A2CEngine(PPOEngine):
    """hp: vf_coef, ent_coef, normalize_advantages, max_grad_norm, loss_reduction ("mean" | "sum").  opt: the update
    used when no optimizer handle is attached: {"name": "rmsprop", lr, alpha, eps, weight_decay, momentum, centered}
    or {"name": "adam", lr, eps, betas}.  With a handle (`B200RMSprop` / `B200Adam`), its param_groups[0] is read
    before every step, so schedulers that edit it take effect."""

    def _check_rows(self, sizes: Sequence[int]):
        if not sizes or min(sizes) < 1:
            raise ValueError("train() needs at least one non-empty minibatch")
        B = sizes[0]
        if any(n != B for n in sizes[:-1]) or sizes[-1] > B:
            raise ValueError(f"minibatches must share one size (the last may be shorter), got {list(sizes)}")
        if self.hp["normalize_advantages"] and sizes[-1] < 2:
            raise ValueError("normalize_advantages with a one-row minibatch: the unbiased std of one advantage is NaN "
                             "(the reference's parameters become NaN); choose per_rank_batch_size so that no minibatch "
                             "has a single row")
        N = sum(sizes)
        for (H, W, C, k, st, Ho, Wo, Co) in self.geo:
            if N * Ho * Wo * k * k * C > INT32_MAX - 1 or N * H * W * C > INT32_MAX - 1:
                raise ValueError(f"a rollout of {N} rows of {self.geo[0][0]}x{self.geo[0][1]}x{self.geo[0][2]} images "
                                 "exceeds the 32-bit indexing of the convolution patch matrix; A2C's one-pass update "
                                 "needs the whole rollout's patch matrix (use fewer envs x rollout steps)")
        return B, N

    def train(self, data: Dict[str, torch.Tensor], index_batches: Sequence[Sequence[int]], on_minibatch=None):
        """data: flat [N, ...] device tensors (rgb uint8 or float32 raw 0..255; everything else float32);
        index_batches: the row indices of each minibatch, in sampler order.  `on_minibatch(losses[3])` is called once
        per minibatch with its (policy, value, entropy) losses."""
        o, s, hp = self.ops, self.spec, self.hp
        batches = [list(ib) for ib in index_batches]
        B, N = self._check_rows([len(ib) for ib in batches])
        idx = torch.as_tensor([i for ib in batches for i in ib], dtype=torch.int64).to(self.device, non_blocking=True)
        b = self._buffers(N)

        def rows(key):
            v = data[key]
            out = torch.empty((N, *v.shape[1:]), dtype=v.dtype, device=v.device)
            o.replay_gather(v.reshape(v.shape[0], -1), idx, out, 1, N, 1)
            return out

        x_state = rows("state").unsqueeze(0) if s["mlp_dim"] else None
        self.forward(b, rows("rgb") if self.geo else None, x_state)
        losses = torch.empty(len(batches), 3, dtype=torch.float32, device=self.device)
        o.a2c_loss(b["head"][0], rows("actions"), rows("advantages").reshape(-1), b["values"].reshape(-1),
                   rows("returns").reshape(-1), b["dhead"][0], b["dvalues"].reshape(-1), losses, B, self.head_dims,
                   self.dist_mode, hp["normalize_advantages"], hp["loss_reduction"] == "sum", hp["vf_coef"],
                   hp["ent_coef"])
        self._backward(b, x_state)
        self._optimizer_step()
        self.losses = losses
        if on_minibatch is not None:
            for i in range(len(batches)):
                on_minibatch(losses[i])

    def _apply_update(self, lr: float):
        g = self.group
        handle = getattr(g, "optimizer", None)
        if handle is None:
            o = dict(self.opt)
        else:
            o = dict(handle.param_groups[0], name="adam" if isinstance(handle, B200Adam) else "rmsprop")
        clip = float(self.hp["max_grad_norm"])
        if o["name"] == "adam":
            b1, b2 = o["betas"]
            self.ops.adam_step(g.flat, g.grad, g.exp_avg, g.exp_avg_sq, self.normsq, clip, lr, b1, b2, o["eps"],
                               g.step_t, self.norm_out, **g.adam_kwargs(o.get("weight_decay", 0.0)))
            return
        # RMSprop state in the group's buffers: square_avg -> exp_avg_sq, momentum_buffer -> exp_avg
        momentum = float(o["momentum"])
        self.ops.rmsprop_step(g.flat, g.grad, g.exp_avg_sq, g.exp_avg if momentum > 0 else None,
                              g.alloc_grad_avg() if o["centered"] else None, self.normsq, clip, lr, float(o["alpha"]),
                              float(o["eps"]), float(o["weight_decay"]), momentum, self.norm_out)
