"""TEST INFRASTRUCTURE — writes tests/golden/p2e_dec_diambra.pt by EXECUTING THE REAL REFERENCE
`sheeprl.algos.p2e_dv3.p2e_dv3_exploration.train` on the DIAMBRA shape (container only):

    python -m oracle.make_golden_p2e_decoder_keys

Image + `own` / `opp` / `reward` vectors; `reward` is encoded only and the MLP decoder reconstructs `[opp, own]`, in
another order than the encoder's.  Same content and procedure as oracle/make_golden_p2e.py (perturbed reference
initialisation, two updates, noise conditioned by the oracle, the oracle checked against the reference before the file
is written); the oracle reconstructs the decoder keys (oracle/dv3_decoder_keys_oracle.py).
"""
from __future__ import annotations

import contextlib
import copy
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import dv3_oracle as O  # noqa: E402
from oracle import make_golden_p2e as MG  # noqa: E402
from oracle import p2e_oracle as P  # noqa: E402
from oracle import ref_harness, ref_run  # noqa: E402
from oracle.dv3_decoder_keys_oracle import decoder_keys  # noqa: E402
from sheeprl_b200.configs import make_p2e_dv3_cfg  # noqa: E402

CFG = dict(MG.CFG, per_rank_batch_size=2, per_rank_sequence_length=4, cnn_channels_multiplier=2, hidden_size=24, n_ensembles=2, horizon=3,
           mlp_keys={"own": 4, "opp": 3, "reward": 1}, algo__mlp_keys__decoder=["opp", "own"])
ACTIONS_DIM = MG.ACTIONS_DIM
STEPS = 2
NAME = "p2e_dec_diambra"


def obs_space(cfg):
    sz = cfg.env.screen_size
    space = {k: ref_harness.Shape((3, sz, sz)) for k in cfg.algo.cnn_keys.encoder}
    space.update({k: ref_harness.Shape((d,)) for k, d in O.vec_dims(cfg).items()})
    return space


def build_reference(cfg, seed=0):
    """`make_golden_p2e.build_reference` with the vector keys in the observation space"""
    ref_harness.install()
    import sheeprl.algos.p2e_dv3.agent as PA

    PA.get_single_device_fabric = lambda f: f
    PA.isolate_rng = contextlib.nullcontext
    rcfg = ref_run.to_ref_cfg(cfg)
    fab = ref_harness.FakeFabric()
    fab.seed_everything = lambda s: torch.manual_seed(s)
    torch.manual_seed(seed)
    wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl, _ = PA.build_agent(
        fab, ACTIONS_DIM, False, rcfg, obs_space(cfg))
    return fab, rcfg, wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl


@contextlib.contextmanager
def vector_keys():
    """inside the block the Plan2Explore generator's helpers build the reference with the vector keys"""
    orig = MG.build_reference
    MG.build_reference = build_reference
    try:
        yield
    finally:
        MG.build_reference = orig


def run_oracle(cfg, sd, data, noise, margin=0.0):
    with decoder_keys():
        return MG.run_oracle(cfg, sd, data, noise, margin)


def main():
    cfg = make_p2e_dv3_cfg(**CFG)
    sd = MG.export(*build_reference(cfg)[2:])
    g = torch.Generator().manual_seed(5)
    for name, d in sd.items():
        if name.startswith("target_"):
            continue
        for v in d.values():
            v.add_(torch.randn(v.shape, generator=g) * 0.05)
    sd["target_task"] = {k: v + 0.01 for k, v in sd["critic_task"].items()}
    for k in list(sd):
        if k.startswith("critic_expl_"):
            sd["target_expl_" + k[len("critic_expl_"):]] = {n: v - 0.01 for n, v in sd[k].items()}
    a, w = cfg.algo, cfg.algo.world_model
    T, B, H = a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon
    data = [O.make_batch(cfg, ACTIONS_DIM, seed=1 + s) for s in range(STEPS)]
    noise = [P.draw_noise(T, B, H, w.stochastic_size, w.discrete_size, ACTIONS_DIM, seed=10 + s) for s in range(STEPS)]
    run_oracle(cfg, copy.deepcopy(sd), data, noise, margin=1e-3)          # conditions `noise` in place
    with vector_keys():
        after, metrics, moments = MG.run_reference(cfg, sd, data, noise)
    _, om, _ = run_oracle(cfg, copy.deepcopy(sd), data, noise)
    worst = 0.0
    for s in range(STEPS):
        for k, v in metrics[s].items():
            if k in om[s]:
                err = abs(float(om[s][k]) - float(v)) / max(1.0, abs(float(v)))
                worst = max(worst, err)
                assert err < 2e-4, (s, k, float(om[s][k]), float(v))
    print("oracle vs reference: worst relative metric error", worst)
    for d in data:                                  # pixels are whole numbers: stored as uint8 (the file stays small)
        for k in cfg.algo.cnn_keys.encoder:
            d[k] = d[k].to(torch.uint8)
    out = {"cfg": CFG, "actions_dim": ACTIONS_DIM, "init": sd, "data": data, "noise": noise, "after": after,
           "metrics": [{k: float(v) for k, v in m.items()} for m in metrics], "moments": moments}
    path = os.path.join(ROOT, "tests", "golden", NAME + ".pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), sorted(metrics[-1]))


if __name__ == "__main__":
    main()
