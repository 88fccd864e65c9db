"""Cost of the MineDojo actor on one GPU, through the public build_agent() + train() and PlayerDV3.get_actions:

    python tests/perf/time_minedojo.py [--calls 50] [--warmup 10]     -> one JSON line, with the card and power limit

Player: us per get_actions step (with a device synchronise per step), masked (the four mask keys, one
b200rl_minedojo_sample launch after the head products) against unmasked (three cat_sample launches), alternated in the
same process, at 2 environments (the dreamer_v3_minedojo recipe) and at 16.  Train: ms per train() (the replayed CUDA
graph) at the dreamer_v3_XS sizes with MineDojo-like head widths [19, 244, 640] and the four mask keys encoded and
decoded, next to the same configuration with the plain actor.  Also reports which RSSM scan route the envelope queries
picked at these shapes (the action vector is 903 wide).  Fails without a GPU.

(lives under tests/: it uses the oracle's batch generator)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

DIMS = (19, 244, 640)
MASKS = {"mask_action_type": 19, "mask_craft_smelt": 244, "mask_equip_place": 640, "mask_destroy": 640}
ACTOR = "sheeprl.algos.dreamer_v3.agent.MinedojoActor"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


class Fab:
    device = torch.device("cuda")


class Space:
    def __init__(self, *shape):
        self.shape = shape


class Agg:
    disabled = True


def build(actor_cls, num_envs):
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent
    from sheeprl_b200.configs import make_dv3_cfg

    cfg = make_dv3_cfg("XS", mlp_keys=MASKS, algo__actor__cls=actor_cls)
    cfg.env.num_envs = num_envs
    space = {"rgb": Space(3, 64, 64), **{k: Space(d) for k, d in MASKS.items()}}
    torch.manual_seed(0)
    return cfg, build_agent(Fab, DIMS, False, cfg, space)


def player_us(player, obs, mask, calls):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        player.get_actions(obs, False, mask)
        torch.cuda.synchronize()
    return 1e6 * (time.perf_counter() - t0) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_minedojo.py measures on a GPU; none is visible")
    from oracle import dv3_oracle as O
    from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import make_optimizers, train
    from sheeprl_b200.algos.dreamer_v3.utils import Moments

    out = {"card": card(), "head_widths": list(DIMS)}
    g = torch.Generator().manual_seed(1)
    for E in (2, 16):
        _, (*_, player) = build(ACTOR, E)
        obs = {"rgb": torch.randint(0, 256, (1, E, 3, 64, 64), generator=g, dtype=torch.uint8).cuda()}
        mask = {k: (torch.rand(1, E, d, generator=g) < 0.5).cuda() for k, d in MASKS.items()}
        obs.update(mask)
        player.init_states()
        for m in (mask, None):
            player_us(player, obs, m, args.warmup)
        t = {"masked": [], "unmasked": []}
        for _ in range(5):                                            # alternated arms
            t["masked"].append(player_us(player, obs, mask, args.calls))
            t["unmasked"].append(player_us(player, obs, None, args.calls))
        out[f"player_us_{E}envs"] = {k: round(sorted(v)[len(v) // 2], 1) for k, v in t.items()}
    for name, cls in (("minedojo", ACTOR), ("plain", "sheeprl.algos.dreamer_v3.agent.Actor")):
        cfg, (wm, actor, critic, target, _) = build(cls, 2)
        eng = wm._b200_engine
        data = O.make_batch(cfg, DIMS, seed=4)
        for k in MASKS:
            data[k] = (data[k] > 0).float()
        data = {k: v.cuda() for k, v in data.items()}
        opts = make_optimizers(eng, cfg)
        mo = cfg.algo.actor.moments
        moments = Moments(mo.decay, mo.max, mo.percentile.low, mo.percentile.high)

        def step():
            train(Fab, wm, actor, critic, target, *opts, data, Agg(), cfg, False, DIMS, moments)

        for _ in range(args.warmup):
            step()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.calls):
            step()
        e1.record()
        torch.cuda.synchronize()
        out[f"train_ms_xs_{name}"] = round(e0.elapsed_time(e1) / args.calls, 3)
        out[f"rssm_scan_{name}"] = {"fused_forward": bool(eng.fused_scan), "fused_backward": bool(eng.fused_scan_bwd)}
        if name == "minedojo":
            Win = eng._w("rssm.recurrent_model.mlp._model.0.weight")
            out["imagination_onehot_gather"] = bool(eng.ops.onehot_linear_supported(eng.S, eng.D, eng.A, Win.shape[0]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
