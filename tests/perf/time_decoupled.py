"""Cost of `algo.world_model.decoupled_rssm` at the BASELINE S config (B16 T64 H15) on one GPU, through the public
build_agent() + train():

    python tests/perf/time_decoupled.py [--calls 50] [--warmup 10]     -> one JSON line, with the card and power limit

ms per train() (the replayed CUDA graph) with the switch off and on, alternated in the same process; CUDA-event time of
the scan phase alone (coupled: `_scan_forward` + `_scan_backward` around rssm_scan_fwd / _bwd; decoupled: the batched
chain + gru_scan_fwd / _bwd), run eagerly on the saves of the last step; and the kernel launches of one eager step.  The
two settings are different models: this is a cost table for choosing the switch, not a speed-up.  Fails without a GPU.

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
        raise SystemExit("time_decoupled.py measures on a GPU; none is visible")
    from oracle import dv3_oracle as O
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent
    from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import make_optimizers, train
    from sheeprl_b200.algos.dreamer_v3.utils import Moments
    from sheeprl_b200.configs import make_dv3_cfg

    class Fab:
        device = torch.device("cuda")

    class Space:
        shape = (3, 64, 64)

    class Agg:
        disabled = True

    adim, arms = (2,), {}
    for dec in (False, True):
        cfg = make_dv3_cfg("S", algo__world_model__decoupled_rssm=dec)
        wm, actor, critic, target, _ = build_agent(Fab, adim, False, cfg, {"rgb": Space})
        eng = wm._b200_engine
        mo = cfg.algo.actor.moments
        moments = Moments(mo.decay, mo.max, mo.percentile.low, mo.percentile.high)
        opts = make_optimizers(eng, cfg)
        data = {k: v.cuda() for k, v in O.make_batch(cfg, adim, seed=3, as_uint8=True).items()}

        def step(wm=wm, actor=actor, critic=critic, target=target, opts=opts, data=data, cfg=cfg, moments=moments):
            train(Fab, wm, actor, critic, target, *opts, data, Agg(), cfg, False, adim, moments)

        arms[dec] = (eng, step, data)
    for _, step, _ in arms.values():
        for _ in range(max(args.warmup, 10)):
            step()
    train_ms = {False: [], True: []}
    rounds = 5
    for _ in range(rounds):                                   # alternate the two settings
        for dec, (_, step, _) in arms.items():
            train_ms[dec].append(timed(step, max(args.calls, 50) // rounds))
    out = {"gpu": card(), "config": "dreamer_v3 S, B16 T64 H15", "calls": max(args.calls, 50), "rows": {}}
    for dec, (eng, step, data) in arms.items():
        first = data["is_first"].reshape(eng.N).float()

        def scan(eng=eng, first=first):
            eng._scan_forward(first)
            eng._scan_backward(first)

        for _ in range(5):
            scan()
        scan_ms = timed(scan, 20)
        n0 = eng.ops.launches
        scan()
        scan_launches = eng.ops.launches - n0
        n0 = eng.ops.launches
        eng.train_step(dict(data), None)
        step_launches = eng.ops.launches - n0
        torch.cuda.synchronize()
        assert eng.fused_scan and eng.fused_scan_bwd and eng.ops.rssm_scan_error(eng._scan_ws) == 0
        ms = sorted(train_ms[dec])
        out["rows"]["decoupled" if dec else "coupled"] = {
            "train_ms_median": round(ms[len(ms) // 2], 3), "train_ms_min": round(ms[0], 3), "train_ms_max": round(ms[-1], 3),
            "scan_fwd_bwd_ms": round(scan_ms, 3), "scan_launches": scan_launches, "step_launches": step_launches}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
