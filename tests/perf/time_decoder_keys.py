"""Cost of decoding a subset of the encoded keys at the BASELINE S config (B16 T64 H15) on one GPU, through the public
build_agent() + train():

    python tests/perf/time_decoder_keys.py [--calls 50] [--warmup 10]     -> one JSON line, with the card and power limit

Three configurations over an image + `own` (12) + `opp` (12) + `reward` (1) observation, 9 + 4 discrete actions:
decoder = encoder (every key decoded), the DIAMBRA subset (`reward` encoded only, `[opp, own]` decoded) and the Crafter
shape (image + `reward`, `mlp_keys.decoder: []`).  Reports ms per train() (the replayed CUDA graph), the three arms
alternated in the same process, the kernel launches of one eager step, and us per `PlayerDV3.get_actions` at 2
environments with its launch count (host-bound: issued back to back without a per-call sync, so only the launch
count compares arms).  Fails without a GPU.

(lives under tests/: it uses the oracle's batch generator)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def timed(fn, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_decoder_keys.py measures on a GPU; none is visible")
    from oracle import dv3_oracle as O
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent
    from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import make_optimizers, train
    from sheeprl_b200.algos.dreamer_v3.utils import Moments
    from sheeprl_b200.configs import make_dv3_cfg

    class Fab:
        device = torch.device("cuda")

    class Space:
        def __init__(self, *shape):
            self.shape = shape

    class Agg:
        disabled = True

    adim = (9, 4)
    full = {"own": 12, "opp": 12, "reward": 1}
    configs = {
        "decoder_equals_encoder": dict(mlp_keys=full),
        "diambra_subset": dict(mlp_keys=full, algo__mlp_keys__decoder=["opp", "own"]),
        "crafter_shape": dict(mlp_keys={"reward": 1}, algo__mlp_keys__decoder=[]),
    }
    arms = {}
    for name, kw in configs.items():
        cfg = make_dv3_cfg("S", num_envs=2, **kw)
        space = {"rgb": Space(3, 64, 64), **{k: Space(d) for k, d in kw["mlp_keys"].items()}}
        wm, actor, critic, target, player = build_agent(Fab, adim, False, cfg, space)
        eng = wm._b200_engine
        mo = cfg.algo.actor.moments
        moments = Moments(mo.decay, mo.max, mo.percentile.low, mo.percentile.high)
        opts = make_optimizers(eng, cfg)
        data = {k: v.cuda() for k, v in O.make_batch(cfg, adim, seed=3, as_uint8=True).items()}

        def step(wm=wm, actor=actor, critic=critic, target=target, opts=opts, data=data, cfg=cfg, moments=moments):
            train(Fab, wm, actor, critic, target, *opts, data, Agg(), cfg, False, adim, moments)

        arms[name] = (eng, step, data, player, kw["mlp_keys"])
    for _, step, *_ in arms.values():
        for _ in range(max(args.warmup, 10)):
            step()
    train_ms = {k: [] for k in arms}
    rounds = 5
    for _ in range(rounds):                                   # alternate the settings
        for name, (_, step, *_) in arms.items():
            train_ms[name].append(timed(step, max(args.calls, 50) // rounds))
    out = {"gpu": card(), "config": "dreamer_v3 S, B16 T64 H15, actions (9, 4)", "calls": max(args.calls, 50), "rows": {}}
    for name, (eng, step, data, player, mlp) in arms.items():
        n0 = eng.ops.launches
        eng.train_step(dict(data), None)
        step_launches = eng.ops.launches - n0
        player.init_states()
        obs = {"rgb": torch.randint(0, 256, (1, 2, 3, 64, 64), dtype=torch.uint8, device="cuda")}
        obs.update({k: torch.randn(1, 2, d, device="cuda") for k, d in mlp.items()})
        act = lambda player=player, obs=obs: player.get_actions(obs, False, {})  # noqa: E731
        for _ in range(20):
            act()
        act_us = 1000.0 * timed(act, 200)
        n0 = eng.ops.launches
        act()
        act_launches = eng.ops.launches - n0
        torch.cuda.synchronize()
        ms = sorted(train_ms[name])
        out["rows"][name] = {
            "train_ms_median": round(ms[len(ms) // 2], 3), "train_ms_min": round(ms[0], 3), "train_ms_max": round(ms[-1], 3),
            "step_launches": step_launches, "get_actions_us_2envs": round(act_us, 1), "get_actions_launches": act_launches}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
