"""DroQ train() calls on one GPU (eager), next to the reference's own train() (torch eager) on the same GPU when the
reference package is present under oracle/_ref (placed there by build()):

    python tests/perf/bench_droq.py [--calls 20]        -> one JSON line per workload, with the card and power limit

Workloads: `exp=droq` (obs 8 as in its default env, act 2, hidden 256, 2 critics, batch 256, dropout 0.01, replay ratio
20 on 4 envs = 80 critic steps per call) and the same recipe at a MuJoCo size (obs 17, act 6).  Both sides read the same
data from a buffer stand-in, so the time is the update alone.
(lives under tests/: it uses the oracle's data generator and the reference harness, which only tests/, smoke() and
bench.py may import)
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.perf.bench_a2c import card, timed_eager  # noqa: E402

WORKLOADS = {
    "exp=droq (obs 8, act 2, H 256, n 2, B 256, p 0.01, G 80)": dict(obs_dim=8, act_dim=2, hidden=256, n_critics=2,
                                                                      B=256, p=0.01, G=80, seed=1),
    "exp=droq at a MuJoCo size (obs 17, act 6)": dict(obs_dim=17, act_dim=6, hidden=256, n_critics=2, B=256, p=0.01,
                                                       G=80, seed=2),
}


class Replay:
    """sample_tensors(n) -> the first n rows of a fixed draw, as [1, n, ...] on the device"""

    def __init__(self, rows):
        self.rows = rows

    def sample_tensors(self, n, **kw):
        return {k: v[:n].unsqueeze(0) for k, v in self.rows.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    from oracle import ref_harness
    from oracle import sac_oracle as SO
    from oracle.make_golden_droq import droq_cfg
    from sheeprl_b200.algos.droq.agent import build_agent
    from sheeprl_b200.algos.droq.droq import make_optimizers, train
    from sheeprl_b200.lib import CudaOps

    cu = CudaOps()
    gpu = card()
    ref_ok = ref_harness.reference_available()
    if ref_ok:
        ref_harness.install()

    class Fab:
        device, world_size, global_rank = torch.device("cuda"), 1, 0

    for name, sp in WORKLOADS.items():
        cfg = droq_cfg(sp)

        class Box:
            shape = (sp["act_dim"],)
            low, high = np.full(sp["act_dim"], -1.0, np.float32), np.full(sp["act_dim"], 1.0, np.float32)

        class Space:
            shape = (sp["obs_dim"],)

        G, B = sp["G"], sp["B"]
        rows = {k: v.cuda() for k, v in SO.make_batch(G * B, sp["obs_dim"], sp["act_dim"], seed=sp["seed"]).items()}
        rb = Replay(rows)
        agent, _ = build_agent(Fab, cfg, {"state": Space}, Box, ops=cu)
        opts = make_optimizers(agent, cfg)
        step = lambda: train(Fab, agent, *opts, rb, None, cfg, G)  # noqa: E731
        step()
        l0 = cu.launches
        step()
        launches = cu.launches - l0
        ms = timed_eager(step, args.calls)
        eng = agent._b200_engine
        assert torch.isfinite(eng.qf.flat).all() and torch.isfinite(eng.actor.flat).all()
        ref = None
        if ref_ok:
            import sheeprl.algos.droq.agent as RA
            import sheeprl.algos.droq.droq as RD
            from sheeprl.utils.timer import timer

            timer.disabled = True
            RA.get_single_device_fabric = lambda f: f
            fab = ref_harness.FakeFabric("cuda")
            fab.all_reduce = lambda x, group=None: x
            ragent, _ = RA.build_agent(fab, cfg, {"state": Space}, Box)
            qf = torch.optim.Adam(ragent.qfs.parameters(), lr=3e-4, eps=1e-4)
            ac = torch.optim.Adam(ragent.actor.parameters(), lr=3e-4, eps=1e-4)
            al = torch.optim.Adam([ragent.log_alpha], lr=3e-4, eps=1e-4)
            f = lambda: RD.train(fab, ragent, ac, qf, al, rb, None, cfg, G)  # noqa: E731
            f()
            ref = {"ms_per_train_call": timed_eager(f, max(3, args.calls // 4)),
                   "kind": "reference train(), torch eager, same GPU"}
        print(json.dumps({"metric": f"DroQ train() [{name}]", "value": ms, "unit": "ms/train call",
                          "gpu_launches_per_train_call": launches, "launches_per_critic_step": launches / G,
                          "critic_steps_per_train_call": G, "reference": ref, "gpu": gpu}))


if __name__ == "__main__":
    main()
