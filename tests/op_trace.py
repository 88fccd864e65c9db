"""Digests of the op sequence every engine and player issues on the CPU test double, per scenario: each `ops.*` call
and each torch op the engines issue outside them, recorded by tools/trace_dense_ops.py's recorder (method, scalar
arguments, tensor storages / offsets / shapes / strides / dtypes), over the dense-engine scenarios of that tool plus
every Dreamer-V3 and Plan2Explore fixture configuration and player.

    python tests/op_trace.py OUT.json        -> {scenario: [lines, sha256 of the lines]}

tests/golden/op_trace_default.json holds the digests recorded before the deterministic mode existed; with torch's
deterministic switch off, the engines must still issue exactly that sequence (tests/test_deterministic_cpu.py)."""
from __future__ import annotations

import contextlib
import hashlib
import importlib.util
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _tool():
    spec = importlib.util.spec_from_file_location("trace_dense_ops", os.path.join(ROOT, "tools", "trace_dense_ops.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def dv3_scenarios():
    from tests import test_dv3_decoder_keys_cpu as DK
    from tests import test_dv3_decoupled_cpu as DC
    from tests import test_engine_emul as EE
    from tests import test_p2e_continuous_cpu as P2C
    from tests import test_p2e_cpu as P2E
    from tests import test_p2e_decoder_keys_cpu as P2K
    from tests import test_player_cpu as PL

    for name in ("dv3_tiny_a", "dv3_tiny_b", "dv3_tiny_c", "dv3_tiny_v", "dv3_tiny_vo", "dv3_tiny_mk", "dv3_tiny_h0"):
        yield f"dv3 engine {name}", lambda name=name: EE.test_engine_matches_oracle_and_reference(name)
    for name in ("dv3_tiny_v", "dv3_tiny_vo", "dv3_tiny_mk"):
        yield f"dv3 public {name}", lambda name=name: EE.test_public_api_with_vector_observations(name)
    for name in DC.FIXTURES:
        yield f"dv3 decoupled engine {name}", lambda name=name: DC.test_engine_schedule_matches_oracle_and_reference(name)
    yield "dv3 decoupled player", DC.test_player_matches_reference
    for name in DK.FIXTURES:
        yield f"dv3 decoder keys engine {name}", lambda name=name: DK.test_engine_schedule_matches_oracle_and_reference(name)
    yield "dv3 decoder keys player", DK.test_player_resizes_to_num_envs_and_ignores_masks
    for name in PL.PLAYER_FIXTURES:
        yield f"dv3 player {name}", lambda name=name: PL.test_player_matches_reference(name)
    yield "p2e engine", P2E.test_engine_schedule_matches_reference
    yield "p2e public", P2E.test_public_api_matches_reference
    yield "p2e finetuning", P2E.test_finetuning_update_is_the_task_behaviour_step
    yield "p2e player", P2E.test_player_acts_with_the_exploration_actor
    yield "p2e continuous engine", P2C.test_engine_schedule_matches_reference
    yield "p2e continuous public", P2C.test_public_api_matches_reference
    yield "p2e continuous finetuning", P2C.test_continuous_finetuning_update_is_the_task_behaviour_step
    yield "p2e continuous player", P2C.test_player_acts_with_the_continuous_exploration_actor
    yield "p2e decoder keys engine", P2K.test_engine_schedule_matches_reference


@contextlib.contextmanager
def _traced(T):
    """wraps every test-double ops class for the recorder, and puts the classes back afterwards"""
    from oracle import ops_emul

    mods = [ops_emul] + [importlib.import_module(f"oracle.{m}") for m in ("ops_emul_a2c", "ops_emul_droq", "ops_emul_recurrent")]
    classes = {v for m in mods for v in vars(m).values() if isinstance(v, type) and v.__name__.endswith("EmulOps")}
    saved = {c: dict(vars(c)) for c in classes}
    try:
        for c in classes:
            T.wrap_ops(c)
        yield
    finally:
        for c, d in saved.items():
            for k in list(vars(c)):
                if k not in d:
                    delattr(c, k)
            for k, v in d.items():
                if k not in ("__dict__", "__weakref__") and vars(c).get(k) is not v:
                    setattr(c, k, v)


def digests(only=None):
    T = _tool()
    out = {}
    torch.manual_seed(0)
    with _traced(T):
        for title, run in list(T.scenarios()) + list(dv3_scenarios()):
            if only is not None and title not in only:
                continue
            T.LINES.clear(), T.STORAGES.clear(), T.ALLOCATED.clear()
            with T.AtenRecorder():
                try:
                    run()
                except Exception as e:                                   # a failing scenario is part of the trace
                    T.LINES.append(f"EXCEPTION {type(e).__name__}: {e}")
            lines = T.LINES + ["--- allocations"] + sorted(T.ALLOCATED)
            out[title] = [len(lines), hashlib.sha256("\n".join(lines).encode()).hexdigest()]
    return out


if __name__ == "__main__":
    with open(sys.argv[1], "w") as f:
        json.dump(digests(), f, indent=1, sort_keys=True)
