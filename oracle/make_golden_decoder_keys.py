"""TEST INFRASTRUCTURE — writes tests/golden/dv3_dec_*.pt by EXECUTING THE REAL REFERENCE `dreamer_v3.train` with decoders
over a subset of the encoded keys (container only):

    python -m oracle.make_golden_decoder_keys [names]

dv3_dec_diambra: image + three vector keys; `reward` is encoded only and the decoder's two keys come in another order
than the encoder's (the shape of the DIAMBRA recipes, `env.reward_as_observation: True`);
dv3_dec_crafter: image + `reward` vector, `mlp_keys.decoder: []` (the Crafter XL recipe);
dv3_dec_twoimg: two image keys (3 + 1 channels), a CNN decoder over the 1-channel one, plus two vector keys;
dv3_dec_nocnn: image in the encoder only (`cnn_keys.decoder: []`), vector decoder, continuous actions;
dv3_dec_crafter_d: dv3_dec_crafter with `decoupled_rssm: True`.
The noise is conditioned by the oracle (oracle/dv3_decoder_keys_oracle.py) and injected as oracle/make_golden.py does.
"""
from __future__ import annotations

import contextlib
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import dv3_decoupled_oracle as OD  # noqa: E402
from oracle import dv3_oracle as O  # noqa: E402
from oracle import ref_harness, ref_run  # noqa: E402
from oracle.dv3_decoder_keys_oracle import decoder_keys  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402
from sheeprl_b200.configs import make_dv3_cfg  # noqa: E402

BASE = dict(size="S", per_rank_batch_size=2, per_rank_sequence_length=4, horizon=4, dense_units=32, mlp_layers=2,
            cnn_channels_multiplier=2, recurrent_state_size=24, hidden_size=24, stochastic_size=6, discrete_size=5, bins=31,
            algo__world_model__kl_free_nats=0.05)
DIAMBRA = dict(BASE, mlp_keys={"own": 4, "opp": 3, "reward": 1}, algo__mlp_keys__decoder=["opp", "own"])
CRAFTER = dict(BASE, mlp_keys={"reward": 1}, algo__mlp_keys__decoder=[])
FIXTURES = {
    "dv3_dec_diambra": dict(cfg=DIAMBRA, actions_dim=(3, 2), perturb=0.05, steps=2, is_first=((2, 1),)),
    "dv3_dec_crafter": dict(cfg=CRAFTER, actions_dim=(4,), perturb=0.05, steps=2, is_first=((3, 0),)),
    "dv3_dec_twoimg": dict(cfg=dict(BASE, cnn_keys=("rgb", "depth"), cnn_channels={"rgb": 3, "depth": 1},
                                    mlp_keys={"state": 5, "extra": 3}, algo__cnn_keys__decoder=["depth"],
                                    algo__mlp_keys__decoder=["extra"]),
                           actions_dim=(3,), perturb=0.05, steps=2, is_first=((2, 0),)),
    "dv3_dec_nocnn": dict(cfg=dict(BASE, mlp_keys={"state": 5, "extra": 3}, algo__cnn_keys__decoder=[],
                                   algo__mlp_keys__decoder=["extra", "state"]),
                          actions_dim=(2,), perturb=0.05, steps=2, is_continuous=True, is_first=((2, 1),)),
    "dv3_dec_crafter_d": dict(cfg=dict(CRAFTER, algo__world_model__decoupled_rssm=True), actions_dim=(4,), perturb=0.05,
                              steps=2, is_first=((2, 1),)),
}


@contextlib.contextmanager
def oracle_for(cfg):
    """the decoder-keys oracle, decoupled when the config asks for it"""
    with decoder_keys(), (OD.decoupled() if cfg.algo.world_model.decoupled_rssm else contextlib.nullcontext()):
        yield


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
    with oracle_for(cfg):
        for s in range(steps):
            O.dv3_train_step(cfg, *cp, *opts, data[s], noise[s], ms, adim, condition_margin=1e-3, is_continuous=cont)
    if w.decoupled_rssm:
        from oracle.make_golden_decoupled import run_reference_train

        after, metrics, moments = run_reference_train(cfg, adim, data, noise, sd, seed, cont)
    else:
        after, metrics, moments = ref_run.run_reference_train(cfg, adim, data, noise, steps, seed=seed, state=sd,
                                                              is_continuous=cont)
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


if __name__ == "__main__":
    main()
