"""TEST INFRASTRUCTURE — writes tests/golden/a2c_*.pt by EXECUTING THE UNMODIFIED REFERENCE `a2c.train` (where the
reference checkout is available):

    python -m oracle.make_golden_a2c

Each run builds the reference PPOAgent (a2c.py:14) with the parameters `a2c_oracle.init_params(spec, seed)` and makes
two consecutive train() calls (one for the Adam run and for the pixel run) on synthetic rollouts, so the optimizer state
carries over.  The optimizer is a subclass of torch's RMSprop / Adam whose step() first records every `p.grad`: the
accumulated (and clipped) gradient, which the parameters after an RMSprop step alone do not pin (its first step moves
every element by about lr / sqrt(1 - alpha), whatever the gradient's size).  Recorded per call: the seed of the
rollout (`ppo_oracle.make_rollout`), the minibatch index lists the reference's RandomSampler / BatchSampler drew, the
logged losses of every minibatch (the entropy loss is not logged by the reference) and that gradient in fp32.  The
parameters after the run are not stored: `a2c_oracle.replay_updates` recomputes them from the initial parameters and
the recorded gradients, and this script checks that they are bit-identical to the reference agent's.  Seeds in place
of tensors keep every file well under 400 KB (the pixel run's one fp32 gradient of the NatureCNN stack is ~340 KB).
"""
from __future__ import annotations

import contextlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import a2c_oracle as AO  # noqa: E402
from oracle import ppo_oracle as PO  # noqa: E402
from oracle import ref_harness as H  # noqa: E402
from oracle.make_golden_ppo import obs_space, split_obs  # noqa: E402
from sheeprl_b200.utils.utils import dotdict  # noqa: E402

HP = dict(vf_coef=1.0, ent_coef=0.0, normalize_advantages=False, max_grad_norm=0.0, loss_reduction="sum")
RMSPROP = {"_target_": "torch.optim.RMSprop", "lr": 1e-3, "eps": 1e-4, "weight_decay": 0}   # algo/a2c.yaml over optim/rmsprop.yaml
VECTOR = dict(cnn_channels=0, screen=0, mlp_dim=4, dense=64, layers=2, cnn_features=512, mlp_features=64,
              actions_dim=(2,), is_continuous=False, act="tanh")
BRANCHES = dict(cnn_channels=0, screen=0, mlp_dim=6, dense=32, layers=2, layer_norm=True, cnn_features=512,
                mlp_features=16, actions_dim=(3, 2), is_continuous=False, act="relu")
CONT = dict(cnn_channels=0, screen=0, mlp_dim=5, dense=32, layers=2, cnn_features=512, mlp_features=16,
            actions_dim=(3,), is_continuous=True, act="tanh")
PIXEL = dict(cnn_channels=3, screen=64, mlp_dim=3, dense=32, layers=1, cnn_features=8, mlp_features=16,
             actions_dim=(4,), is_continuous=False, act="relu")
BR_HP = dict(HP, loss_reduction="mean", normalize_advantages=True, max_grad_norm=0.5, ent_coef=0.01, vf_coef=0.5)
FIXTURES = {
    # exp=a2c: 4 envs x 5 steps in minibatches of 5; the second call a ragged plan (6, 6, 6, 2)
    "a2c_vector": [dict(spec=VECTOR, hp=HP, opt=RMSPROP, calls=[(20, 5), (20, 6)], seed=31)],
    # every loss branch; RMSprop with momentum, centered, weight decay; then a run with an Adam optimizer config
    "a2c_branches": [
        dict(spec=BRANCHES, hp=BR_HP, calls=[(24, 8), (21, 8)], seed=32,
             opt=dict(RMSPROP, lr=3e-3, momentum=0.9, centered=True, weight_decay=1e-4, alpha=0.95)),
        dict(spec=BRANCHES, hp=BR_HP, calls=[(21, 8)], seed=33,
             opt={"_target_": "torch.optim.Adam", "lr": 1e-3, "eps": 1e-5, "betas": [0.9, 0.999]})],
    "a2c_continuous": [
        dict(spec=CONT, hp=dict(HP, ent_coef=0.01), opt=RMSPROP, calls=[(16, 5), (16, 5)], seed=34),
        dict(spec=dict(CONT, dist="tanh_normal"), hp=dict(HP, loss_reduction="mean", ent_coef=0.01), opt=RMSPROP,
             calls=[(16, 6), (16, 6)], seed=35)],
    # the full NatureCNN stack on 64x64x3 plus a vector key; ragged minibatches (4, 4, 2); one call (each fp32
    # gradient of the conv stack is ~340 KB)
    "a2c_pixel": [dict(spec=PIXEL, hp=dict(BR_HP, normalize_advantages=True), opt=RMSPROP, calls=[(10, 4)], seed=36)],
}


def a2c_cfg(spec, hp, batch, opt):
    def net(which):
        dense, layers, ln = PO.net_cfg(spec, which)
        return {"dense_units": dense, "mlp_layers": layers, "layer_norm": ln, "ortho_init": False,
                "dense_act": "torch.nn.Tanh" if spec["act"] == "tanh" else "torch.nn.ReLU"}

    cnn = ["rgb"] if spec["cnn_channels"] else []
    mlp = ["state"] if spec["mlp_dim"] else []
    enc = dict(net("encoder"), cnn_features_dim=spec["cnn_features"], mlp_features_dim=spec["mlp_features"])
    dist = spec.get("dist", "auto") if spec["is_continuous"] else "auto"
    return dotdict({"algo": dict(hp, name="a2c", cnn_keys={"encoder": cnn}, mlp_keys={"encoder": mlp}, encoder=enc,
                                 actor=net("actor"), critic=net("critic"), per_rank_batch_size=batch,
                                 optimizer=dict(opt)),
                    "buffer": {"share_data": False}, "env": {"screen_size": spec["screen"]}, "seed": 0,
                    "distribution": {"type": dist}})


class Fabric(H.FakeFabric):
    @contextlib.contextmanager
    def no_backward_sync(self, module, enabled=True):
        yield


def recording(cls, names, sink):
    class Recording(cls):
        def step(self, closure=None):
            sink.append({names[id(p)]: p.grad.detach().clone() for g in self.param_groups for p in g["params"]})
            return super().step(closure)

    return Recording


def run(r):
    import sheeprl.algos.a2c.a2c as R
    import sheeprl.algos.ppo.agent as A

    A.get_single_device_fabric = lambda f: f
    spec, hp = r["spec"], r["hp"]
    fab = Fabric()
    init = AO.init_params(spec, r["seed"])
    cfg = a2c_cfg(spec, hp, r["calls"][0][1], r["opt"])
    agent, _ = A.build_agent(fab, spec["actions_dim"], spec["is_continuous"], cfg, obs_space(spec), init)
    export = lambda: {k.replace("_forward_module.", ""): v.detach().clone() for k, v in agent.state_dict().items()}  # noqa: E731
    assert all(torch.equal(v, init[k]) for k, v in export().items()), "key/shape layout drifted"
    names = {id(p): k.replace("_forward_module.", "") for k, p in agent.named_parameters()}
    grads = []
    kw = {k: v for k, v in r["opt"].items() if not k.startswith("_")}
    cls = torch.optim.Adam if r["opt"]["_target_"].endswith("Adam") else torch.optim.RMSprop
    opt = recording(cls, names, grads)(agent.parameters(), **kw)
    orig, calls = R.BatchSampler, []
    for c, (N, batch) in enumerate(r["calls"]):
        drawn, rows = [], []

        class Sampler(orig):
            def __iter__(self):
                for b in super().__iter__():
                    drawn.append(list(b))
                    yield b

        class Agg:
            disabled = False

            def update(self, k, v):
                if k == "Loss/policy_loss":
                    rows.append({})
                rows[-1][k] = float(v)

        data = PO.make_rollout(spec, N, r["seed"] * 10 + c)
        cfg = a2c_cfg(spec, hp, batch, r["opt"])
        R.BatchSampler = Sampler
        try:
            torch.manual_seed(r["seed"] * 10 + 5 + c)
            R.train(fab, agent, opt, split_obs(spec, {k: v.clone() for k, v in data.items()}), Agg(), cfg)
        finally:
            R.BatchSampler = orig
        calls.append({"N": N, "batch": batch, "data_seed": r["seed"] * 10 + c, "index_batches": drawn, "losses": rows,
                      "grads": grads[-1], "sampler_seed": r["seed"] * 10 + 5 + c})
    after = AO.replay_updates(init, r["opt"], [c["grads"] for c in calls])
    assert all(torch.equal(after[k], v) for k, v in export().items()), "replayed parameters differ from the reference's"
    return {"spec": spec, "hp": hp, "opt": r["opt"], "init_seed": r["seed"], "calls": calls}


def main():
    H.install()
    for name, runs in FIXTURES.items():
        out = [run(r) for r in runs]
        path = os.path.join(ROOT, "tests", "golden", f"{name}.pt")
        torch.save(out, path)
        print(name, os.path.getsize(path), [[c["index_batches"] for c in r["calls"]] for r in out])


if __name__ == "__main__":
    main()
