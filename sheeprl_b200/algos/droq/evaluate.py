"""`sheeprl-eval` entry for DroQ checkpoints on the CUDA player (reference: sheeprl/algos/droq/evaluate.py).  The
evaluation loop is the reference's (`evaluate` -> `sac.utils.test`); only `build_agent` is substituted, so the player
that acts is `SACPlayer` on the CUDA kernels, loaded from the checkpoint's `agent` state dict."""
from __future__ import annotations

from typing import Any, Dict

from sheeprl_b200.utils.delegate import import_reference, substituted


def evaluate_droq(fabric, cfg: Dict[str, Any], state: Dict[str, Any]):
    from sheeprl_b200.algos.droq import agent as A

    ref = import_reference("sheeprl.algos.droq.evaluate")
    with substituted(ref, {"build_agent": A.build_agent}):
        return ref.evaluate(fabric, cfg, state)


try:  # register under the reference's evaluation registry when it is importable (sheeprl/utils/registry.py:111-120)
    from sheeprl.utils.registry import register_evaluation  # type: ignore

    evaluate_droq = register_evaluation(algorithms="droq")(evaluate_droq)
except Exception:  # pragma: no cover - real sheeprl not installed
    pass
