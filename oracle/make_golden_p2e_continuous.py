"""TEST INFRASTRUCTURE — writes tests/golden/p2e_tiny_c.pt by EXECUTING THE REAL REFERENCE
`sheeprl.algos.p2e_dv3.p2e_dv3_exploration.train` with continuous actions (container only):

    python -m oracle.make_golden_p2e_continuous

Continuous control from state vectors (a 7-dim vector observation, no image) with a 3-dim `scaled_normal` action; the
Plan2Explore parts as in p2e_tiny.pt (oracle/make_golden_p2e.py).  Both exploration critics carry weights other than 1,
`ent_coef` is large enough for the entropy bonus to show in a 1e-4 comparison, and the default `action_clip` (1.0)
clips about a third of the action draws.  Fixture: config kwargs, initial parameters of every module (reference
`build_agent`, perturbed), two replay batches, the noise of both updates (Exp(1) conditioned by the oracle so no
categorical draw sits on a near-tie; one N(0,1) tensor per behaviour phase), the metrics the reference logged and every
trained module's parameters + the five Moments after two updates.
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
from oracle import p2e_continuous_oracle as PC  # noqa: E402
from oracle import ref_harness, ref_run  # noqa: E402
from oracle.make_golden_p2e import export, oracle_state  # noqa: E402
from sheeprl_b200.configs import make_p2e_dv3_cfg  # noqa: E402

CFG = dict(size="S", per_rank_batch_size=3, per_rank_sequence_length=5, horizon=4, dense_units=32, mlp_layers=1,
           recurrent_state_size=24, hidden_size=32, stochastic_size=6, discrete_size=5, bins=31, cnn_keys=(),
           mlp_keys={"state": 7}, n_ensembles=3, intrinsic_weight=0.7, extrinsic_weight=0.6,
           intrinsic_reward_multiplier=2.0, algo__world_model__kl_free_nats=0.05, algo__actor__ent_coef=0.05)
ACTIONS_DIM = (3,)
STEPS = 2


def build_reference(cfg, seed=0):
    ref_harness.install()
    import sheeprl.algos.p2e_dv3.agent as PA

    PA.get_single_device_fabric = lambda f: f
    PA.isolate_rng = contextlib.nullcontext
    rcfg = ref_run.to_ref_cfg(cfg)
    fab = ref_harness.FakeFabric()
    fab.seed_everything = lambda s: torch.manual_seed(s)
    space = {k: ref_harness.Shape((d,)) for k, d in O.vec_dims(cfg).items()}
    torch.manual_seed(seed)
    wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl, _ = PA.build_agent(
        fab, ACTIONS_DIM, True, rcfg, space)
    return fab, rcfg, wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl


def run_oracle(cfg, sd, data, noise, margin=0.0):
    p, critics, opts, mt = oracle_state(cfg, sd)
    metrics = []
    for s in range(len(data)):
        metrics.append(PC.p2e_continuous_train_step(cfg, p["wm"], p["ens"], p["actor_task"], p["critic_task"],
                                                    p["target_task"], p["actor_expl"], critics, opts, data[s], noise[s],
                                                    mt, ACTIONS_DIM, margin))
    moments = {"task": mt, **{k: c["moments"] for k, c in critics.items()}}
    return p, metrics, moments


def run_reference(cfg, sd, data, noise):
    ref_harness.install()
    import torch.distributions.normal as TN
    from sheeprl.algos.dreamer_v3.utils import Moments
    from sheeprl.algos.p2e_dv3 import p2e_dv3_exploration as X

    fab, rcfg, wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl = build_reference(cfg)
    mods = {"wm": wm, "ens": ens, "actor_task": actor_task, "critic_task": critic_task, "target_task": target_task,
            "actor_expl": actor_expl}
    for k, c in critics_expl.items():
        mods[f"critic_expl_{k}"], mods[f"target_expl_{k}"] = c["module"], c["target_module"]
    for k, m in mods.items():
        ref_run._load(m, sd[k])
    a = cfg.algo

    def adam(params, o):
        return torch.optim.Adam(params, lr=o.lr, eps=o.eps, weight_decay=o.weight_decay, betas=tuple(o.betas))

    wo, eo = adam(wm.parameters(), a.world_model.optimizer), adam(ens.parameters(), a.ensembles.optimizer)
    ato, cto = adam(actor_task.parameters(), a.actor.optimizer), adam(critic_task.parameters(), a.critic.optimizer)
    aeo = adam(actor_expl.parameters(), a.actor.optimizer)
    for c in critics_expl.values():
        c["optimizer"] = adam(c["module"].parameters(), a.critic.optimizer)
    mo = a.actor.moments
    new_m = lambda: Moments(mo.decay, mo.max, mo.percentile.low, mo.percentile.high)  # noqa: E731
    m_task, m_expl = new_m(), {k: new_m() for k in critics_expl}
    T, H = a.per_rank_sequence_length, a.horizon
    metrics = []
    for s in range(len(data)):
        agg = ref_harness.RecordingAggregator()
        batch = {k: v.clone().float() for k, v in data[s].items()}
        cat, normal = PC.reference_noise_order(noise[s], T, H)
        orig = TN._standard_normal
        TN._standard_normal = lambda shape, dtype, device: normal.pop(0).reshape(shape)
        try:
            with ref_harness.NoiseQueue(cat):
                X.train(fab, wm, actor_task, critic_task, target_task, wo, ato, cto, batch, agg, rcfg, ens, eo, actor_expl,
                        critics_expl, aeo, m_expl, m_task, True, ACTIONS_DIM)
        finally:
            TN._standard_normal = orig
        assert not normal, "the reference drew fewer Normal samples than expected"
        metrics.append(agg.values)
    moments = {"task": m_task, **m_expl}
    moments = {k: {"low": v.low.detach().clone(), "high": v.high.detach().clone()} for k, v in moments.items()}
    return export(wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl), metrics, moments


def main():
    cfg = make_p2e_dv3_cfg(**CFG)
    sd = export(*build_reference(cfg)[2:])
    g = torch.Generator().manual_seed(5)
    for group, d in sd.items():
        if group.startswith("target_"):
            continue
        for v in d.values():
            v.add_(torch.randn(v.shape, generator=g) * 0.05)
    sd["target_task"] = {k: v + 0.01 for k, v in sd["critic_task"].items()}
    for k in list(sd):
        if k.startswith("critic_expl_"):
            sd["target_expl_" + k[len("critic_expl_"):]] = {n: v - 0.01 for n, v in sd[k].items()}
    a, w = cfg.algo, cfg.algo.world_model
    T, B, H = a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon
    data = [O.make_batch(cfg, ACTIONS_DIM, seed=1 + s, is_continuous=True) for s in range(STEPS)]
    noise = [PC.draw_noise(T, B, H, w.stochastic_size, w.discrete_size, ACTIONS_DIM, seed=10 + s) for s in range(STEPS)]
    run_oracle(cfg, copy.deepcopy(sd), data, noise, margin=1e-3)          # conditions `noise` in place
    after, metrics, moments = run_reference(cfg, sd, data, noise)
    # the oracle must reproduce the executed reference before the fixture is written
    _, om, _ = run_oracle(cfg, copy.deepcopy(sd), data, noise)
    worst = 0.0
    for s in range(STEPS):
        for k, v in metrics[s].items():
            assert k in om[s], k
            err = abs(float(om[s][k]) - float(v)) / max(1.0, abs(float(v)))
            worst = max(worst, err)
            assert err < 2e-4, (s, k, float(om[s][k]), float(v))
    print("oracle vs reference: worst relative metric error", worst)
    # the target critics do not change inside train(): "after" keeps the trained groups only
    out = {"cfg": CFG, "actions_dim": ACTIONS_DIM, "is_continuous": True, "init": sd, "data": data, "noise": noise,
           "after": {k: v for k, v in after.items() if not k.startswith("target_")},
           "metrics": [{k: float(v) for k, v in m.items()} for m in metrics], "moments": moments}
    path = os.path.join(ROOT, "tests", "golden", "p2e_tiny_c.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), sorted(metrics[-1]))


if __name__ == "__main__":
    main()
