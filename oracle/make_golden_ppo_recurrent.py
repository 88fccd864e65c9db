"""TEST INFRASTRUCTURE — writes tests/golden/ppo_rec_*.pt by EXECUTING THE REAL REFERENCE `ppo_recurrent.train` and
`RecurrentPPOPlayer` (where the reference checkout is available):

    python -m oracle.make_golden_ppo_recurrent

Torch's distribution argument validation is OFF for the whole run
(`torch.distributions.Distribution.set_default_validate_args(False)`): padded steps leave all-zero action rows, which
`OneHotCategorical.log_prob` rejects under validation, so the reference's own `train()` raises on every padded
minibatch; with validation off it runs and the padded rows drop out through `[mask]`.  That is the behaviour
reproduced here.

Fixture: spec, hyper-parameters, initial parameters (reference `build_agent` under torch.manual_seed), the synthetic
padded rollout (lengths include 1 and T), the sequence-index lists the reference's RandomSampler/BatchSampler drew
(recorded), the three logged losses of every minibatch and the parameters after train().  To keep the files small the
initial parameters are stored as the seed of `ppo_recurrent_oracle.init_params` (loaded into the reference agent) and
the parameters after train() as their fp16 update (`pack_after`).  ppo_rec_player.pt: a few player steps with the
multinomial noise injected (images stored as uint8, normalised by `player_obs` as the rollout loop does).
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ppo_recurrent_oracle as RO  # noqa: E402
from oracle import ref_harness as H  # noqa: E402
from oracle.make_golden_ppo import obs_space  # noqa: E402
from sheeprl_b200.utils.utils import dotdict  # noqa: E402

HP = dict(clip_coef=0.2, vf_coef=0.2, ent_coef=0.0, clip_vloss=False, normalize_advantages=False, max_grad_norm=0.0)
FIXTURES = {
    # configs/algo/ppo_recurrent.yaml widths: 1 x 64 LayerNorm ReLU MLPs, LSTM 64; two discrete heads
    "ppo_rec_vector": dict(spec=dict(cnn_channels=0, screen=0, mlp_dim=4, dense=64, layers=1, layer_norm=True,
                                     cnn_features=512, mlp_features=64, actions_dim=(3, 2), is_continuous=False,
                                     act="relu", rnn=dict(hidden=64, pre=None, post=None)),
                           hp=dict(HP, ent_coef=0.001, max_grad_norm=0.5), T=6,
                           lengths=(6, 1, 4, 6, 2, 6, 3, 5), batches=2, epochs=2, seed=21),
    # every loss branch, pre- and post-RNN MLPs with LayerNorm (eps 1e-3), an LSTM width that is not a power of two
    "ppo_rec_branches": dict(spec=dict(cnn_channels=0, screen=0, mlp_dim=5, dense=32, layers=2, layer_norm=True,
                                       nets={"encoder": (24, 1), "actor": (32, 2), "critic": (16, 1)},
                                       cnn_features=512, mlp_features=16, actions_dim=(4,), is_continuous=False,
                                       act="tanh", rnn=dict(hidden=48, pre=(24, True), post=(48, True))),
                             hp=dict(HP, clip_vloss=True, normalize_advantages=True, ent_coef=0.01, vf_coef=0.5,
                                     max_grad_norm=0.5), T=5,
                             lengths=(5, 1, 3, 5, 2, 4, 1, 5, 5), batches=3, epochs=2, seed=22),
    # the full NatureCNN conv stack on 64x64 x 2 stacked frames plus a vector key (small frames and cnn_features keep
    # the file small)
    "ppo_rec_pixel": dict(spec=dict(cnn_channels=2, screen=64, mlp_dim=3, dense=64, layers=1, layer_norm=True,
                                    cnn_features=8, mlp_features=16, actions_dim=(4,), is_continuous=False,
                                    act="relu", rnn=dict(hidden=64, pre=None, post=None)),
                          hp=dict(HP, ent_coef=0.01), T=4, lengths=(4, 1, 3, 4), batches=2, epochs=1, seed=23),
}


def rec_cfg(spec, hp, batches, epochs, num_envs=1):
    def net(which):
        dense, layers, ln = RO.PO.net_cfg(spec, which)
        return {"dense_units": dense, "mlp_layers": layers, "layer_norm": ln, "ortho_init": False,
                "dense_act": "torch.nn.Tanh" if spec["act"] == "tanh" else "torch.nn.ReLU"}

    cnn = [k for k, _ in (spec.get("cnn_keys") or ([("rgb", spec["cnn_channels"])] if spec["cnn_channels"] else []))]
    mlp = [k for k, _ in (spec.get("mlp_keys") or ([("state", spec["mlp_dim"])] if spec["mlp_dim"] else []))]
    act = "torch.nn.Tanh" if spec["act"] == "tanh" else "torch.nn.ReLU"
    r = spec["rnn"]

    def side(c, default):
        return {"apply": bool(c), "bias": True, "activation": act, "layer_norm": bool(c and c[1]),
                "dense_units": int(c[0]) if c else default}

    rnn = {"lstm": {"hidden_size": r["hidden"]}, "pre_rnn_mlp": side(r.get("pre"), net("encoder")["dense_units"]),
           "post_rnn_mlp": side(r.get("post"), r["hidden"])}
    enc = dict(net("encoder"), cnn_features_dim=spec["cnn_features"], mlp_features_dim=spec["mlp_features"])
    return dotdict({"algo": dict(hp, cnn_keys={"encoder": cnn}, mlp_keys={"encoder": mlp}, encoder=enc, rnn=rnn,
                                 actor=net("actor"), critic=net("critic"), per_rank_num_batches=batches,
                                 update_epochs=epochs, loss_reduction="mean",
                                 optimizer={"_target_": "torch.optim.AdamW", "lr": 1e-3, "eps": 1e-4,
                                            "weight_decay": 0, "betas": [0.9, 0.999]}),
                    "env": {"screen_size": spec["screen"], "num_envs": num_envs}, "seed": 0,
                    "distribution": {"type": "auto"}})


def _export(agent):
    return {k.replace("_forward_module.", ""): v.detach().clone() for k, v in agent.state_dict().items()}


def run(fx):
    import sheeprl.algos.ppo_recurrent.agent as A
    import sheeprl.algos.ppo_recurrent.ppo_recurrent as P

    A.get_single_device_fabric = lambda f: f
    spec, hp = fx["spec"], fx["hp"]
    cfg = rec_cfg(spec, hp, fx["batches"], fx["epochs"])
    fab = H.FakeFabric()
    init = RO.init_params(spec, fx["seed"])
    agent, _ = A.build_agent(fab, spec["actions_dim"], False, cfg, obs_space(spec), init)
    assert all(torch.equal(v, init[k]) for k, v in _export(agent).items()), "key/shape layout drifted"
    opt = torch.optim.Adam(agent.parameters(), lr=1e-3, eps=1e-4)
    data = RO.make_rollout(spec, fx["T"], fx["lengths"], fx["seed"] + 1)
    drawn, orig = [], P.BatchSampler

    class Recording(orig):
        def __iter__(self):
            for b in super().__iter__():
                drawn.append(list(b))
                yield b

    class Agg:
        disabled = False

        def __init__(self):
            self.rows = []

        def update(self, k, v):
            if k == "Loss/policy_loss":
                self.rows.append({})
            self.rows[-1][k] = float(v)

    agg = Agg()
    P.BatchSampler = Recording
    try:
        torch.manual_seed(fx["seed"] + 2)
        ref_data = {k: v.clone() for k, v in data.items()}     # the fixtures' single keys are `rgb` / `state`
        P.train(fab, agent, opt, ref_data, agg, cfg)
    finally:
        P.BatchSampler = orig
    return {"spec": spec, "hp": hp, "batches": fx["batches"], "epochs": fx["epochs"], "init_seed": fx["seed"],
            "data": data, "index_batches": drawn, "losses": agg.rows,
            "after_delta": RO.pack_after(init, _export(agent)), "sampler_seed": fx["seed"] + 2}


def run_player(name, fx, E=5, steps=3):
    """A few RecurrentPPOPlayer steps on the fixture's initial parameters: forward (states carried), get_values on a
    subset of envs (the truncation path), greedy get_actions."""
    import sheeprl.algos.ppo_recurrent.agent as A

    spec = fx["spec"]
    cfg = rec_cfg(spec, fx["hp"], fx["batches"], fx["epochs"], num_envs=E)
    fab = H.FakeFabric()
    _, player = A.build_agent(fab, spec["actions_dim"], False, cfg, obs_space(spec), RO.init_params(spec, fx["init_seed"]))
    g = torch.Generator().manual_seed(99)
    Hs, nA = spec["rnn"]["hidden"], sum(spec["actions_dim"])
    states = (torch.randn(1, E, Hs, generator=g) * 0.3, torch.randn(1, E, Hs, generator=g) * 0.3)
    prev = torch.zeros(1, E, nA)
    rec = {"init_states": tuple(s.clone() for s in states), "init_prev": prev.clone(), "steps": []}
    for _ in range(steps):
        raw = {}                                       # images as the env gives them (uint8 in the fixture)
        if spec["cnn_channels"]:
            raw["rgb"] = torch.randint(0, 256, (1, E, spec["cnn_channels"], spec["screen"], spec["screen"]),
                                       generator=g).to(torch.uint8)
        if spec["mlp_dim"]:
            raw["state"] = torch.randn(1, E, spec["mlp_dim"], generator=g)
        obs = RO.player_obs(raw)
        noise = [torch.empty(E, a).exponential_(1.0, generator=g) for a in spec["actions_dim"]]
        with torch.no_grad(), H.NoiseQueue(noise):
            actions, logp, values, states = player(obs, prev_actions=prev, prev_states=states)
        rec["steps"].append({"obs": raw, "noise": torch.cat(noise, -1), "actions": [a.clone() for a in actions],
                             "logp": logp.clone(), "values": values.clone(),
                             "states": tuple(s.clone() for s in states)})
        prev = torch.cat(actions, -1)
    sub = [0, 2, 3]
    obs = RO.player_obs(rec["steps"][-1]["obs"])
    with torch.no_grad():
        vals, st2 = player.get_values({k: v[:, sub] for k, v in obs.items()}, prev[:, sub], tuple(s[:, sub] for s in states))
        greedy, st3 = player.get_actions(obs, prev, states, greedy=True)
    rec.update(sub=sub, sub_values=vals.clone(), sub_states=tuple(s.clone() for s in st2),
               greedy=[a.clone() for a in greedy], greedy_states=tuple(s.clone() for s in st3))
    return rec


def main():
    H.install()
    torch.distributions.Distribution.set_default_validate_args(False)
    players = {}
    for name, fx in FIXTURES.items():
        out = run(fx)
        players[name] = run_player(name, out)
        if "rgb" in out["data"]:                      # integer-valued pixels: keep the fixture small
            out["data"]["rgb"] = out["data"]["rgb"].to(torch.uint8)
        path = os.path.join(ROOT, "tests", "golden", f"{name}.pt")
        torch.save(out, path)
        print(name, os.path.getsize(path), out["index_batches"], out["losses"][-1])
    torch.save(players, os.path.join(ROOT, "tests", "golden", "ppo_rec_player.pt"))


if __name__ == "__main__":
    main()
