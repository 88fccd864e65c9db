"""TEST INFRASTRUCTURE (oracle) — NOT part of the product path.

The Dreamer-V3 oracle (`oracle/dv3_oracle.py`) for `algo.world_model.decoupled_rssm=True`.  The reference's
`DecoupledRSSM` (agent.py:501-593) differs from `RSSM` in one function: `_representation` takes the embedding alone
(:582-593).  `train()` then computes the posterior of every step in front of the loop (dreamer_v3.py:115-129), which is
the same arithmetic row by row as computing it inside the loop, so the decoupled oracle is the coupled oracle's code with
`representation_logits` replaced for the duration of a `with decoupled():` block.  What does change is the order of the
reference's sampling calls, `reference_noise_order` below.
"""
from __future__ import annotations

import contextlib
from typing import Dict, List, Sequence

from oracle import dv3_oracle as O

Tensor = O.Tensor


def representation_logits(wm, h, e, S, D, unimix, eps):  # agent.py:582-593: no recurrent state in the input
    raw = O.dense_stack(wm, "rssm.representation_model._model.", e, 1, eps, True)
    return O.unimix_logits(raw, S, D, unimix)


@contextlib.contextmanager
def decoupled():
    """inside the block `O.world_model_phase` / `O.dv3_train_step` compute the decoupled model"""
    orig = O.representation_logits
    O.representation_logits = representation_logits
    try:
        yield
    finally:
        O.representation_logits = orig


def reference_noise_order(noise: Dict[str, Tensor], T: int, H: int, n_heads: int) -> List[Tensor]:
    """`noise` in the order the reference's train() calls torch.multinomial with `decoupled_rssm`: ONE posterior draw over
    [T,B,S,D] in front of the loop (dreamer_v3.py:116), then the discarded prior draw of every step (agent.py:579), then
    the behaviour draws in the coupled order."""
    return [noise["post"]] + [noise["prior"][t] for t in range(T)] + O.reference_noise_order(noise, 0, H, n_heads)


def init_params(cfg, actions_dim: Sequence[int], **kw):
    """`O.init_params` with the narrower representation model: its first layer has no recurrent-state columns"""
    wm, actor, critic, target = O.init_params(cfg, actions_dim, **kw)
    R = cfg.algo.world_model.recurrent_model.recurrent_state_size
    k = "rssm.representation_model._model.0.weight"
    wm[k] = wm[k][:, R:].clone()
    return wm, actor, critic, target
