"""TEST INFRASTRUCTURE — writes tests/golden/dv3_tiny_{d,dv}.pt and dv3_player_decoupled.pt by EXECUTING THE REAL REFERENCE
`dreamer_v3.train` / `PlayerDV3` with `algo.world_model.decoupled_rssm=True` (container only):

    python -m oracle.make_golden_decoupled [names]

dv3_tiny_d: discrete actions, image key, `is_first` set mid-sequence in some rows, free nats low enough that both KL
branches are live;  dv3_tiny_dv: image + vector keys, continuous actions;  dv3_player_decoupled: the player script of
oracle/make_golden_player.py on dv3_tiny_d's weights.  Same content as the fixtures of oracle/make_golden.py.
"""
from __future__ import annotations

import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import dv3_decoupled_oracle as OD  # noqa: E402
from oracle import dv3_oracle as O  # noqa: E402
from oracle import ref_harness, ref_run  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402
from sheeprl_b200.configs import make_dv3_cfg  # noqa: E402

BASE = dict(size="S", per_rank_batch_size=2, horizon=4, dense_units=32, mlp_layers=2, cnn_channels_multiplier=2,
            recurrent_state_size=24, hidden_size=24, stochastic_size=6, discrete_size=5, bins=31,
            algo__world_model__decoupled_rssm=True)
FIXTURES = {
    "dv3_tiny_d": dict(cfg=dict(BASE, per_rank_sequence_length=5, algo__world_model__kl_free_nats=0.05),
                       actions_dim=(3, 2), perturb=0.05, steps=2, is_first=((2, 1), (3, 0), (4, 1))),
    "dv3_tiny_dv": dict(cfg=dict(BASE, per_rank_sequence_length=4, mlp_keys={"state": 5, "extra": 3}),
                        actions_dim=(3,), perturb=0.05, steps=2, is_continuous=True, is_first=((2, 1),)),
}


def run_reference_train(cfg, adim, data, noise, state, seed, cont):
    """`ref_run.run_reference_train` with the decoupled order of the sampling calls"""
    import torch.distributions.normal as TN
    from sheeprl.algos.dreamer_v3 import dreamer_v3 as D
    from sheeprl.algos.dreamer_v3.utils import Moments

    fab, rcfg, wm, actor, critic, target, _ = ref_run.build_reference_agent(cfg, adim, 3, seed, cont)
    for mod, name in ((wm, "wm"), (actor, "actor"), (critic, "critic"), (target, "target")):
        ref_run._load(mod, state[name])
    a = cfg.algo
    opts = [torch.optim.Adam(m.parameters(), lr=o.lr, eps=o.eps, weight_decay=o.weight_decay, betas=tuple(o.betas))
            for m, o in ((wm, a.world_model.optimizer), (actor, a.actor.optimizer), (critic, a.critic.optimizer))]
    mo = a.actor.moments
    moments = Moments(mo.decay, mo.max, mo.percentile.low, mo.percentile.high)
    T, H, metrics = a.per_rank_sequence_length, a.horizon, []
    for s in range(len(data)):
        agg = ref_harness.RecordingAggregator()
        batch = {k: v.clone().float() for k, v in data[s].items()}
        if cont:        # categorical draws: the scan and the imagined states; Normal.rsample: the actions
            cat = OD.reference_noise_order(noise[s], T, 0, 0) + [noise[s]["img_state"][i] for i in range(H)]
            normal = O.reference_normal_order(noise[s], H)
        else:
            cat, normal = OD.reference_noise_order(noise[s], T, H, len(adim)), []
        orig = TN._standard_normal
        TN._standard_normal = lambda shape, dtype, device: normal.pop(0).reshape(shape)
        try:
            with ref_harness.NoiseQueue(cat):
                D.train(fab, wm, actor, critic, target, *opts, batch, agg, rcfg, cont, tuple(adim), moments)
        finally:
            TN._standard_normal = orig
        assert not normal, "the reference drew fewer Normal samples than expected"
        metrics.append(agg.values)
    return (ref_run.reference_state_dicts(wm, actor, critic, target), metrics,
            {"low": moments.low.detach().clone(), "high": moments.high.detach().clone()})


def build_case(spec, seed=0):
    cfg = make_dv3_cfg(**spec["cfg"])
    adim, cont, steps = tuple(spec["actions_dim"]), bool(spec.get("is_continuous", False)), spec["steps"]
    _, _, wm, actor, critic, target, _ = ref_run.build_reference_agent(cfg, adim, seed=seed, is_continuous=cont)
    sd = ref_run.reference_state_dicts(wm, actor, critic, target)
    g = torch.Generator().manual_seed(5)
    for d in sd.values():
        for v in d.values():
            v.add_(torch.randn(v.shape, generator=g) * spec["perturb"])
    sd["target"] = {k: v + 0.01 for k, v in sd["critic"].items()}
    a, w = cfg.algo, cfg.algo.world_model
    T, B, H = a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon
    data = [O.make_batch(cfg, adim, seed=1 + s, is_continuous=cont) for s in range(steps)]
    for d in data:
        for t, b in spec.get("is_first", ()):
            d["is_first"][t, b] = 1.0
    noise = [O.draw_noise(T, B, H, w.stochastic_size, w.discrete_size, adim, seed=10 + s, is_continuous=cont)
             for s in range(steps)]
    # condition the noise with the oracle (in place), then run the reference on the conditioned noise
    cp = [{k: v.clone() for k, v in sd[n].items()} for n in ("wm", "actor", "critic", "target")]
    opts = [O.AdamState(cp[0], w.optimizer.lr, w.optimizer.eps), O.AdamState(cp[1], a.actor.optimizer.lr, a.actor.optimizer.eps),
            O.AdamState(cp[2], a.critic.optimizer.lr, a.critic.optimizer.eps)]
    ms = {"low": torch.zeros(()), "high": torch.zeros(())}
    with OD.decoupled():
        for s in range(steps):
            O.dv3_train_step(cfg, *cp, *opts, data[s], noise[s], ms, adim, condition_margin=1e-3, is_continuous=cont)
    after, metrics, moments = run_reference_train(cfg, adim, data, noise, sd, seed, cont)
    return cfg, adim, sd, data, noise, after, metrics, moments, (cp, ms)


def main():
    ref_harness.install()
    only = sys.argv[1:]
    for name, spec in FIXTURES.items():
        if only and name not in only:
            continue
        cfg, adim, sd, data, noise, after, metrics, moments, _ = build_case(spec)
        for d in data:
            for k in cfg.algo.cnn_keys.encoder:
                d[k] = d[k].to(torch.uint8)
        path = os.path.join(GOLDEN, name + ".pt")
        torch.save({"cfg_kwargs": spec["cfg"], "actions_dim": adim, "is_continuous": bool(spec.get("is_continuous", False)),
                    "init": sd, "data": data, "noise": noise, "after": after, "metrics": metrics, "moments": moments}, path)
        print("wrote", name, os.path.getsize(path), {k: round(v, 5) for k, v in metrics[-1].items()})
    if not only or "dv3_player_decoupled" in only:
        from oracle.make_golden_player import run

        path = os.path.join(GOLDEN, "dv3_player_decoupled.pt")
        torch.save(run("dv3_tiny_d"), path)
        print("wrote dv3_player_decoupled", os.path.getsize(path))


if __name__ == "__main__":
    main()
