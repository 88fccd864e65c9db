"""`sheeprl-eval` entry for A2C checkpoints on the CUDA player (reference: sheeprl/algos/a2c/evaluate.py).  The evaluation
loop is the reference's (`evaluate_a2c` -> `ppo.utils.test`); only `build_agent` is substituted, so the player that
acts is `PPOPlayer` on the CUDA kernels, loaded from the checkpoint's `agent` state dict."""
from __future__ import annotations

from typing import Any, Dict

from sheeprl_b200.utils.delegate import import_reference, substituted


def evaluate_a2c(fabric, cfg: Dict[str, Any], state: Dict[str, Any]):
    from sheeprl_b200.algos.a2c import agent as A

    ref = import_reference("sheeprl.algos.a2c.evaluate")
    with substituted(ref, {"build_agent": A.build_agent}):
        return ref.evaluate_a2c(fabric, cfg, state)


try:  # register under the reference's evaluation registry when it is importable (sheeprl/utils/registry.py:111-120)
    from sheeprl.utils.registry import register_evaluation  # type: ignore

    evaluate_a2c = register_evaluation(algorithms="a2c")(evaluate_a2c)
except Exception:  # pragma: no cover - real sheeprl not installed
    pass
