"""ms per train() call with torch's deterministic switch off and on, alternating in one process, for every engine:
Dreamer-V3 (BASELINE S config, CUDA-graph replay), Plan2Explore exploration (p2e_tiny fixture), PPO (ppo_pixel fixture),
recurrent PPO (ppo_rec_pixel fixture), A2C (a2c_pixel fixture), SAC (BASELINE config 3 shapes) and DroQ (droq_exp
fixture, one train() call of 20 gradient steps).  Prints the card's name and power limit first, then one JSON line per
engine.

    python tests/perf/time_deterministic.py [--calls 20] [--rounds 3]
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return q or torch.cuda.get_device_name()


def timed(step, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def dv3(cu):
    from oracle import dv3_oracle as O
    from sheeprl_b200.configs import make_dv3_cfg
    from sheeprl_b200.engine import DV3Engine

    cfg = make_dv3_cfg("S")
    adim = (6,)
    eng = DV3Engine(cfg, adim, in_channels=3, device="cuda:0", ops=cu)
    data = {k: v.float().cuda() for k, v in O.make_batch(cfg, adim, seed=2).items()}
    return lambda: eng.step_graph().run(lambda d: eng.train_step(d, None), data, key=eng.graph_key())


def sac(cu):
    from oracle import sac_oracle as SO
    from sheeprl_b200.algos.sac.engine import SACEngine

    O, A, H, B = 17, 6, 256, 256
    opt = {"lr": 3e-4, "eps": 1e-4, "betas": (0.9, 0.999)}
    eng = SACEngine(O, A, H, H, 2, B, 0.99, 0.005, 1.0, -1.0, 1.0, opt, opt, opt, "cuda", cu)
    P = SO.init_params(O, A, H, 2, seed=0)
    eng.load_reference_state(P["actor"], P["qf"], P["qf_target"], P["log_alpha"]["log_alpha"])
    data = {k: v.cuda() for k, v in SO.make_batch(B, O, A, seed=1).items()}
    return lambda: eng.train_step(data, True)


def p2e(cu):
    from tests.test_p2e_cpu import load, make_engine

    fx, cfg = load()
    eng = make_engine(fx, cfg, device="cuda", ops=cu)
    data = {k: v.clone().float().cuda() for k, v in fx["data"][0].items()}
    return lambda: eng.train_step(data, None)


def rec(cu):
    from tests.test_ppo_recurrent_cpu import load, make_engine

    fx = load("ppo_rec_pixel")
    eng = make_engine(fx, device="cuda", ops=cu)
    data = {k: v.cuda() for k, v in fx["data"].items()}
    return lambda: eng.train(data, fx["index_batches"])


def a2c(cu):
    from tests.test_a2c_cpu import build, load

    r = load("a2c_pixel")[0]
    c = r["calls"][0]
    eng = build(r, "cuda", cu)[0]._b200_engine
    data = {k: v.cuda() for k, v in c["data"].items()}
    return lambda: eng.train(data, c["index_batches"])


def droq(cu):
    from tests.test_droq_cpu import call_inputs, load, make_engine

    fx = load("droq_exp")
    critic, actor_obs = call_inputs(fx, 0)[:2]
    critic, actor_obs = {k: v.cuda() for k, v in critic.items()}, actor_obs.cuda()
    eng = make_engine(fx, device="cuda", ops=cu)
    return lambda: eng.train_call(critic, actor_obs)


def ppo(cu):
    from tests.test_ppo_cpu import load, make_engine

    fx = load("ppo_pixel")
    eng = make_engine(fx, device="cuda", ops=cu)
    data = {k: v.cuda() for k, v in fx["data"].items()}
    return lambda: eng.train(data, fx["index_batches"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from sheeprl_b200.lib import CudaOps

    print("card:", card(), flush=True)
    cu = CudaOps()
    for name, make in (("dreamer_v3_S", dv3), ("p2e_exploration", p2e), ("ppo_pixel", ppo), ("ppo_recurrent_pixel", rec),
                       ("a2c_pixel", a2c), ("sac", sac), ("droq_exp", droq)):
        step = make(cu)
        ms = {False: [], True: []}
        for mode in (False, True):                 # warm-up: graph capture and workspace growth of both modes
            torch.use_deterministic_algorithms(mode)
            for _ in range(3):
                step()
        for _ in range(args.rounds):
            for mode in (False, True):
                torch.use_deterministic_algorithms(mode)
                ms[mode].append(timed(step, args.calls))
        torch.use_deterministic_algorithms(False)
        print(json.dumps({"engine": name, "ms_default": [round(x, 4) for x in ms[False]],
                          "ms_deterministic": [round(x, 4) for x in ms[True]]}), flush=True)


if __name__ == "__main__":
    main()
