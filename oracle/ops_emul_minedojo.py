"""TEST INFRASTRUCTURE — executable specification (plain torch, CPU) of the MineDojo actor's masked, chained sample in
`include/b200rl.h` (`b200rl_minedojo_sample` / `_supported`), on top of the `oracle/ops_emul.py::EmulOps`
specification of every other op.  Same two uses: `-m gpu` tests compare the CUDA kernel against it (in float64), and
`-m "not gpu"` tests inject `MinedojoEmulOps` into `DV3Engine` / `PlayerDV3` (test double).  The product never
constructs it.

The rule is MinedojoActor.forward with a mask dict (sheeprl/algos/dreamer_v3/agent.py:898-932): unimix each head, set
the disallowed log-probs to -inf (head 0: mask_action_type; head 1: mask_craft_smelt where head 0 drew 15; head 2:
mask_equip_place where head 0 drew 16 or 17, mask_destroy where it drew 18), normalise like torch's Categorical and
draw argmax(probs / q) (q None: the mode).  One deviation: a mask row that allows no class leaves its head unmasked.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle.ops_emul import FP32_EPS, EmulOps

Tensor = torch.Tensor

CRAFT, EQUIP, PLACE, DESTROY = 15, 16, 17, 18
MASK_KEYS = ("mask_action_type", "mask_craft_smelt", "mask_equip_place", "mask_destroy")


def minedojo_sample_spec(raw: Tensor, noise: Optional[Tensor], unimix: float, actions_dim: Sequence[int],
                         masks: Sequence[Optional[Tensor]] = (None, None, None, None)) -> Tuple[Tensor, List[Tensor]]:
    """(one-hot rows [M, K0+K1+K2], per-head normalised probs [M, K_h]) in raw's dtype.  masks: mask_action_type,
    mask_craft_smelt, mask_equip_place, mask_destroy as [M, K_h] rows (nonzero = allowed) or None (all allowed)."""
    dims = [int(k) for k in actions_dim]
    heads = torch.split(raw, dims, -1)
    qs = torch.split(noise, dims, -1) if noise is not None else (None,) * len(dims)
    m_type, m_craft, m_equip, m_destroy = masks
    hots, probs, a0 = [], [], None
    for i, (x, q, K) in enumerate(zip(heads, qs, dims)):
        if unimix > 0:
            pr = (1 - unimix) * torch.softmax(x, -1) + unimix / K
            lg = torch.log(pr.clamp(FP32_EPS, 1 - FP32_EPS))
        else:
            lg = x.clone()
        allow = torch.ones_like(lg, dtype=torch.bool)
        if i == 0 and m_type is not None:
            allow = m_type != 0
        elif i == 1 and m_craft is not None:
            allow = torch.where((a0 == CRAFT).unsqueeze(-1), m_craft != 0, allow)
        elif i == 2:
            if m_equip is not None:
                allow = torch.where(((a0 == EQUIP) | (a0 == PLACE)).unsqueeze(-1), m_equip != 0, allow)
            if m_destroy is not None:
                allow = torch.where((a0 == DESTROY).unsqueeze(-1), m_destroy != 0, allow)
        allow = allow | ~allow.any(-1, keepdim=True)            # nothing allowed: the head's unmasked distribution
        lg = lg.masked_fill(~allow, float("-inf"))
        p = torch.softmax(lg - torch.logsumexp(lg, -1, keepdim=True), -1)
        idx = (p / q if q is not None else p).argmax(-1)
        hots.append(F.one_hot(idx, K).to(raw.dtype))
        probs.append(p)
        if i == 0:
            a0 = idx
    return torch.cat(hots, -1), probs


class MinedojoEmulOps(EmulOps):
    def minedojo_sample_supported(self, actions_dim) -> bool:
        return len(actions_dim) == 3 and all(1 <= int(k) <= 2048 for k in actions_dim)

    def minedojo_sample(self, raw: Tensor, noise: Optional[Tensor], unimix: float, actions_dim, onehot: Tensor,
                        mask_action_type: Optional[Tensor] = None, mask_craft_smelt: Optional[Tensor] = None,
                        mask_equip_place: Optional[Tensor] = None, mask_destroy: Optional[Tensor] = None):
        hot, _ = minedojo_sample_spec(raw, noise, unimix, actions_dim,
                                      (mask_action_type, mask_craft_smelt, mask_equip_place, mask_destroy))
        onehot.copy_(hot)
