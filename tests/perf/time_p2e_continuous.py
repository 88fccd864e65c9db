"""Plan2Explore (Dreamer-V3 S, 8 ensemble members, intrinsic + extrinsic exploration critics) with a CONTINUOUS 6-dim
action (`scaled_normal`, the policy gradient through the imagined rollout in both behaviour phases) at the BASELINE
batch (bs16 seq64 h15, 64x64x3): finite-ness + step time (eager and CUDA graph).  The discrete counterpart is
time_p2e.py, the continuous Dreamer-V3 step time_cont.py.

    python tests/perf/time_p2e_continuous.py
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from oracle import dv3_oracle as O  # noqa: E402
from sheeprl_b200.algos.p2e_dv3.engine import P2EDV3Engine  # noqa: E402
from sheeprl_b200.configs import make_p2e_dv3_cfg  # noqa: E402


def timed(f, n=10):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    cfg, adim = make_p2e_dv3_cfg("S"), (6,)
    eng = P2EDV3Engine(cfg, adim, device="cuda", is_continuous=True)
    # oracle-side initialisation of every module (statistically the reference's)
    wm, actor, critic, target = O.init_params(cfg, adim, seed=0, is_continuous=True)
    _, actor_e, critic_i, _ = O.init_params(cfg, adim, seed=1, is_continuous=True)
    _, _, critic_x, _ = O.init_params(cfg, adim, seed=2, is_continuous=True)
    st = dict(wm=wm, actor_task=actor, critic_task=critic, target_task=target, actor_expl=actor_e,
              critic_expl_intrinsic=critic_i, target_expl_intrinsic={k: v.clone() for k, v in critic_i.items()},
              critic_expl_extrinsic=critic_x, target_expl_extrinsic={k: v.clone() for k, v in critic_x.items()})
    for name, g in eng.groups().items():
        g.load(st[name])
    gen = torch.Generator().manual_seed(3)
    ens = {}
    for grp in (eng.ens_rest, eng.ens_last):
        for k, shp in grp.shapes.items():
            ens[k] = (torch.ones(shp) if (len(shp) == 1 and k.endswith("weight")) else
                      torch.zeros(shp) if len(shp) == 1 else torch.randn(shp, generator=gen) / shp[1] ** 0.5)
    eng.load_ensembles(ens)
    data = {k: v.cuda() for k, v in O.make_batch(cfg, adim, seed=1, as_uint8=True, is_continuous=True).items()}
    for _ in range(3):
        eng.train_step(data, None)
    torch.cuda.synchronize()
    md = {k: float(v) for k, v in eng.metrics_dict().items()}
    assert all(map(lambda x: x == x and abs(x) < 1e30, md.values())), md
    eager = timed(lambda: eng.train_step(data, None))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.train_step(data, None)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.train_step(data, None)
    g.replay()
    graph = timed(g.replay)
    print(json.dumps({"metric": "Plan2Explore Dreamer-V3 S exploration train step (8 ensembles, 2 exploration critics, "
                                "continuous(6))", "ms_eager": eager, "ms_graph": graph, "steps_per_s": 1e3 / graph,
                      "bytes_allocated_GB": round(eng.bytes_allocated() / 1e9, 2),
                      "metrics": {k: round(v, 4) for k, v in md.items()}}))


if __name__ == "__main__":
    main()
