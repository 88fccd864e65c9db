"""TEST INFRASTRUCTURE — writes tests/golden/dv3_minedojo.pt and tests/golden/p2e_minedojo.pt by EXECUTING THE REAL
REFERENCE `dreamer_v3.train` and `p2e_dv3_exploration.train` with `algo.actor.cls: MinedojoActor` (container only):

    python -m oracle.make_golden_minedojo [dv3] [p2e]

Both use the MineDojo layout at synthetic widths: three action heads [19, 40, 72] and the four action-mask keys as
vector observations in `mlp_keys.encoder` and `mlp_keys.decoder`, as the dreamer_v3_minedojo recipe lists them.
MinedojoActor.forward defaults to greedy=True and train() calls the actor without arguments, so every imagined action is
the mode of its head: the only torch.multinomial draws left are the RSSM's (prior / posterior per scan step, one per
imagined state).  The noise dicts therefore carry no action noise; their `img_action*` entries are lists of None per
head and step, which makes the oracle's `st_sample` take the mode.  Otherwise the procedure is
oracle/make_golden_decoder_keys.py's and oracle/make_golden_p2e_decoder_keys.py's: perturbed reference initialisation,
two updates, noise conditioned by the oracle, the oracle checked against the reference before the file is written.
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
from oracle.make_golden import GOLDEN  # noqa: E402
from sheeprl_b200.configs import make_dv3_cfg, make_p2e_dv3_cfg  # noqa: E402

ACTIONS_DIM = (19, 40, 72)
MASKS = {"mask_action_type": 19, "mask_craft_smelt": 40, "mask_equip_place": 72, "mask_destroy": 72}
DV3_ACTOR = "sheeprl.algos.dreamer_v3.agent.MinedojoActor"
P2E_ACTOR = "sheeprl.algos.p2e_dv3.agent.MinedojoActor"          # Plan2Explore's alias of the same class
DV3_CFG = dict(size="S", per_rank_batch_size=2, per_rank_sequence_length=4, horizon=4, dense_units=32, mlp_layers=2,
               cnn_channels_multiplier=2, recurrent_state_size=24, hidden_size=24, stochastic_size=6, discrete_size=5,
               bins=31, algo__world_model__kl_free_nats=0.05, mlp_keys=MASKS, algo__actor__cls=DV3_ACTOR)
P2E_CFG = dict(MG.CFG, per_rank_batch_size=2, per_rank_sequence_length=4, cnn_channels_multiplier=2, hidden_size=24,
               n_ensembles=2, horizon=3, mlp_keys=MASKS, cnn_keys=(), algo__actor__cls=P2E_ACTOR)   # vector-only: < 1 MB
STEPS = 2


def mode_noise(noise, H: int, keys=("img_action",)):
    """`noise` with every imagined-action entry replaced by None per head and step (the oracle then takes the mode)"""
    for k in keys:
        noise[k] = [[None] * (H + 1) for _ in ACTIONS_DIM]
    return noise


def make_data(cfg, seed: int):
    """O.make_batch with the mask keys as 0 / 1 rows, like the bool masks the environment returns"""
    d = O.make_batch(cfg, ACTIONS_DIM, seed=seed)
    for k in MASKS:
        d[k] = (d[k] > 0).float()
    return d


def dv3_reference_noise_order(noise, T: int, H: int):
    """torch.multinomial calls of dreamer_v3.train with MinedojoActor: prior then posterior per scan step
    (agent.py:433-434), then the transition of every imagined step (dreamer_v3.py:236); the actor draws nothing"""
    out = []
    for t in range(T):
        out += [noise["prior"][t], noise["post"][t]]
    return out + [noise["img_state"][i] for i in range(H)]


def p2e_reference_noise_order(noise, T: int, H: int, n_heads: int):
    """P.reference_noise_order without the actor's draws (both behaviour phases imagine mode actions)"""
    out = []
    for t in range(T):
        out += [noise["prior"][t], noise["post"][t]]
    for ph in ("expl", "task"):
        out += [noise[f"img_state_{ph}"][i] for i in range(H)]
    return out


def run_reference_dv3(cfg, data, noise, sd, seed: int = 0):
    """ref_run.run_reference_train (discrete branch) with the MineDojo actor's draw order"""
    ref_harness.install()
    from sheeprl.algos.dreamer_v3 import dreamer_v3 as D
    from sheeprl.algos.dreamer_v3.utils import Moments

    fab, rcfg, wm, actor, critic, target, _ = ref_run.build_reference_agent(cfg, ACTIONS_DIM, 3, seed)
    assert type(actor.module if hasattr(actor, "module") else actor).__name__ == "MinedojoActor"
    for mod, name in ((wm, "wm"), (actor, "actor"), (critic, "critic"), (target, "target")):
        ref_run._load(mod, sd[name])
    a = cfg.algo

    def adam(params, o):
        return torch.optim.Adam(params, lr=o.lr, eps=o.eps, weight_decay=o.weight_decay, betas=tuple(o.betas))

    wo, ao, co = (adam(m.parameters(), o) for m, o in ((wm, a.world_model.optimizer), (actor, a.actor.optimizer),
                                                       (critic, a.critic.optimizer)))
    mo = a.actor.moments
    moments = Moments(mo.decay, mo.max, mo.percentile.low, mo.percentile.high)
    metrics = []
    for s in range(len(data)):
        agg = ref_harness.RecordingAggregator()
        batch = {k: v.clone().float() for k, v in data[s].items()}
        with ref_harness.NoiseQueue(dv3_reference_noise_order(noise[s], a.per_rank_sequence_length, a.horizon)) as q:
            D.train(fab, wm, actor, critic, target, wo, ao, co, batch, agg, rcfg, False, ACTIONS_DIM, moments)
        assert q.i == len(q.noises), "the reference drew fewer categorical samples than expected"
        metrics.append(agg.values)
    return (ref_run.reference_state_dicts(wm, actor, critic, target), metrics,
            {"low": moments.low.detach().clone(), "high": moments.high.detach().clone()})


def build_dv3(seed: int = 0):
    cfg = make_dv3_cfg(**DV3_CFG)
    a, w = cfg.algo, cfg.algo.world_model
    T, B, H = a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon
    _, _, wm, actor, critic, target, _ = ref_run.build_reference_agent(cfg, ACTIONS_DIM, seed=seed)
    sd = ref_run.reference_state_dicts(wm, actor, critic, target)
    g = torch.Generator().manual_seed(5)
    for d in sd.values():
        for v in d.values():
            v.add_(torch.randn(v.shape, generator=g) * 0.05)
    sd["target"] = {k: v + 0.01 for k, v in sd["critic"].items()}
    data = [make_data(cfg, 1 + s) for s in range(STEPS)]
    data[0]["is_first"][2, 1] = 1.0
    noise = [mode_noise(O.draw_noise(T, B, H, w.stochastic_size, w.discrete_size, ACTIONS_DIM, seed=10 + s), H)
             for s in range(STEPS)]
    cp = [{k: v.clone() for k, v in sd[n].items()} for n in ("wm", "actor", "critic", "target")]
    opts = [O.AdamState(cp[0], w.optimizer.lr, w.optimizer.eps), O.AdamState(cp[1], a.actor.optimizer.lr, a.actor.optimizer.eps),
            O.AdamState(cp[2], a.critic.optimizer.lr, a.critic.optimizer.eps)]
    ms = {"low": torch.zeros(()), "high": torch.zeros(())}
    with decoder_keys():                       # conditions the RSSM noise in place
        for s in range(STEPS):
            O.dv3_train_step(cfg, *cp, *opts, data[s], noise[s], ms, ACTIONS_DIM, condition_margin=1e-3)
    after, metrics, moments = run_reference_dv3(cfg, data, noise, sd, seed)
    return cfg, sd, data, noise, after, metrics, moments


@contextlib.contextmanager
def p2e_minedojo():
    """inside the block the Plan2Explore generator's helpers run the MineDojo layout: its action heads, the mask keys
    in the observation space, and the reference's draw order without action draws"""
    saved = (MG.ACTIONS_DIM, MG.build_reference, P.reference_noise_order)

    def build_reference(cfg, seed=0):
        ref_harness.install()
        import sheeprl.algos.p2e_dv3.agent as PA

        PA.get_single_device_fabric = lambda f: f
        PA.isolate_rng = contextlib.nullcontext
        rcfg = ref_run.to_ref_cfg(cfg)
        fab = ref_harness.FakeFabric()
        fab.seed_everything = lambda s: torch.manual_seed(s)
        sz = cfg.env.screen_size
        space = {k: ref_harness.Shape((3, sz, sz)) for k in cfg.algo.cnn_keys.encoder}
        space.update({k: ref_harness.Shape((d,)) for k, d in O.vec_dims(cfg).items()})
        torch.manual_seed(seed)
        wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl, _ = PA.build_agent(
            fab, ACTIONS_DIM, False, rcfg, space)
        assert all(type(getattr(m, "module", m)).__name__ == "MinedojoActor" for m in (actor_task, actor_expl))
        return fab, rcfg, wm, ens, actor_task, critic_task, target_task, actor_expl, critics_expl

    MG.ACTIONS_DIM, MG.build_reference = ACTIONS_DIM, build_reference
    P.reference_noise_order = lambda noise, T, H, n_heads: p2e_reference_noise_order(noise, T, H, n_heads)
    try:
        yield
    finally:
        MG.ACTIONS_DIM, MG.build_reference, P.reference_noise_order = saved


def run_oracle_p2e(cfg, sd, data, noise, margin=0.0):
    with decoder_keys(), p2e_minedojo():
        return MG.run_oracle(cfg, sd, data, noise, margin)


def build_p2e():
    cfg = make_p2e_dv3_cfg(**P2E_CFG)
    with p2e_minedojo():
        sd = MG.export(*MG.build_reference(cfg)[2:])
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
    data = [make_data(cfg, 1 + s) for s in range(STEPS)]
    noise = [mode_noise(P.draw_noise(T, B, H, w.stochastic_size, w.discrete_size, ACTIONS_DIM, seed=10 + s), H,
                        ("img_action_expl", "img_action_task")) for s in range(STEPS)]
    run_oracle_p2e(cfg, copy.deepcopy(sd), data, noise, margin=1e-3)          # conditions `noise` in place
    with p2e_minedojo():
        after, metrics, moments = MG.run_reference(cfg, sd, data, noise)
    _, om, _ = run_oracle_p2e(cfg, copy.deepcopy(sd), data, noise)
    for s in range(STEPS):
        for k, v in metrics[s].items():
            if k in om[s]:
                err = abs(float(om[s][k]) - float(v)) / max(1.0, abs(float(v)))
                assert err < 2e-4, (s, k, float(om[s][k]), float(v))
    return cfg, sd, data, noise, after, metrics, moments


def _store(data, cfg):
    for d in data:                                  # pixels are whole numbers: stored as uint8 (the file stays small)
        for k in cfg.algo.cnn_keys.encoder:
            d[k] = d[k].to(torch.uint8)
    return data


def main():
    ref_harness.install()
    only = sys.argv[1:]
    if not only or "dv3" in only:
        cfg, sd, data, noise, after, metrics, moments = build_dv3()
        path = os.path.join(GOLDEN, "dv3_minedojo.pt")
        torch.save({"cfg_kwargs": DV3_CFG, "actions_dim": ACTIONS_DIM, "is_continuous": False, "init": sd,
                    "data": _store(data, cfg), "noise": noise, "after": after, "metrics": metrics, "moments": moments}, path)
        print("wrote", path, os.path.getsize(path), {k: round(v, 5) for k, v in metrics[-1].items()})
    if not only or "p2e" in only:
        cfg, sd, data, noise, after, metrics, moments = build_p2e()
        path = os.path.join(GOLDEN, "p2e_minedojo.pt")
        torch.save({"cfg": P2E_CFG, "actions_dim": ACTIONS_DIM, "init": sd, "data": _store(data, cfg), "noise": noise,
                    "after": after, "metrics": [{k: float(v) for k, v in m.items()} for m in metrics],
                    "moments": moments}, path)
        print("wrote", path, os.path.getsize(path), sorted(metrics[-1]))


if __name__ == "__main__":
    main()
