"""A2C train() calls on one GPU (eager), next to the reference's own train() (torch eager) on the same GPU when the
reference package is present under oracle/_ref (placed there by build()):

    python tests/perf/bench_a2c.py [--calls 200]        -> one JSON line per workload, with the card and power limit

(lives under tests/: it uses the oracle's rollout generator and the reference harness, which only tests/, smoke() and
bench.py may import)
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

HP = dict(vf_coef=1.0, ent_coef=0.0, normalize_advantages=False, max_grad_norm=0.0, loss_reduction="sum")
RMSPROP = {"_target_": "torch.optim.RMSprop", "lr": 1e-3, "eps": 1e-4, "weight_decay": 0}
VECTOR = dict(cnn_channels=0, screen=0, mlp_dim=4, dense=64, layers=2, cnn_features=512, mlp_features=64,
              actions_dim=(2,), is_continuous=False, act="tanh")
# (spec, hp, optimizer, rows, minibatch): the three shapes the reference's A2C experiments train at
WORKLOADS = {
    "exp=a2c (4 envs x 5 steps, minibatch 5, vector)": (VECTOR, HP, RMSPROP, 20, 5),
    "algo=a2c (16 envs x 128 steps, minibatch 64, vector)": (VECTOR, HP, RMSPROP, 2048, 64),
    "exp=a2c_atari (1 env x 40 steps of 84x84x4, minibatch 40)": (
        dict(cnn_channels=4, screen=84, mlp_dim=0, dense=512, layers=1, cnn_features=512, mlp_features=0,
             actions_dim=(6,), is_continuous=False, act="relu"),
        dict(vf_coef=0.25, ent_coef=0.01, normalize_advantages=True, max_grad_norm=0.5, loss_reduction="mean"),
        dict(RMSPROP, lr=1e-4, eps=1e-8), 40, 40),
}


def timed_eager(step, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    args = ap.parse_args()
    from oracle import a2c_oracle as AO
    from oracle import ppo_oracle as PO
    from oracle import ref_harness
    from oracle.make_golden_a2c import a2c_cfg
    from oracle.make_golden_ppo import obs_space, split_obs
    from sheeprl_b200.algos.a2c.a2c import _optimizer_factory
    from sheeprl_b200.algos.a2c.agent import build_agent
    from sheeprl_b200.lib import CudaOps

    cu = CudaOps()
    gpu = card()
    ref_ok = ref_harness.reference_available()
    if ref_ok:
        ref_harness.install()

    class Fab:
        device, world_size, global_rank = torch.device("cuda"), 1, 0

    class RefFabric(ref_harness.FakeFabric):
        @contextlib.contextmanager
        def no_backward_sync(self, module, enabled=True):
            yield

    for name, (spec, hp, opt_cfg, N, B) in WORKLOADS.items():
        cfg = a2c_cfg(spec, hp, B, opt_cfg)
        init = AO.init_params(spec, 1)
        agent, _ = build_agent(Fab, spec["actions_dim"], False, cfg, obs_space(spec), agent_state=init, ops=cu)
        _optimizer_factory([agent])(dict(opt_cfg), list(agent.parameters()))
        eng = agent._b200_engine
        data = PO.make_rollout(spec, N, 2)
        dev = {k: v.cuda() for k, v in data.items()}
        if "rgb" in dev:
            dev["rgb"] = dev["rgb"].to(torch.uint8)
        plan = torch.randperm(N, generator=torch.Generator().manual_seed(3)).split(B)
        plan = [p.tolist() for p in plan]
        eng.train(dev, plan)
        l0 = cu.launches
        eng.train(dev, plan)
        launches = cu.launches - l0
        ms = timed_eager(lambda: eng.train(dev, plan), args.calls)
        assert torch.isfinite(eng.losses).all() and torch.isfinite(eng.group.flat).all()
        ref = None
        if ref_ok:
            import sheeprl.algos.a2c.a2c as RA
            import sheeprl.algos.ppo.agent as PA

            PA.get_single_device_fabric = lambda f: f
            fab = RefFabric("cuda")
            ragent, _ = PA.build_agent(fab, spec["actions_dim"], False, cfg, obs_space(spec), None)
            ropt = torch.optim.RMSprop(ragent.parameters(), **{k: v for k, v in opt_cfg.items() if k != "_target_"})
            rdata = split_obs(spec, {k: v.cuda() for k, v in data.items()})
            f = lambda: RA.train(fab, ragent, ropt, rdata, None, cfg)  # noqa: E731
            f()
            ref = {"ms_per_train_call": timed_eager(f, max(5, args.calls // 4)),
                   "kind": "reference train(), torch eager, same GPU"}
        print(json.dumps({"metric": f"A2C train() [{name}]", "value": ms, "unit": "ms/train call",
                          "gpu_launches_per_train_call": launches, "minibatches_per_train_call": len(plan),
                          "reference": ref, "gpu": gpu}))


if __name__ == "__main__":
    main()
