"""TEST INFRASTRUCTURE — writes tests/golden/droq_*.pt by EXECUTING THE REAL REFERENCE `droq.train` (container only):

    python -m oracle.make_golden_droq [name ...]       (default: every fixture)

The unmodified reference `train()` runs with two functions patched to take pre-drawn values from queues, in the
reference's call order:
  * `torch.distributions.normal._standard_normal` (Normal.rsample): per critic minibatch g the target's action noise
    eps_next[g], then once the policy loss's eps_cur;
  * `torch.nn.functional.dropout` (nn.Dropout.forward): `x * keep * (1/(1-p))` with the next bool mask; per minibatch
    the target critics' (critic 0 layer 0, critic 0 layer 1, critic 1 layer 0, ...), then the online critics' in the
    same order, then after the last minibatch the policy loss's (oracle/droq_oracle.py::reference_call_order).
The tiny fixtures sample from a reference `ReplayBuffer` whose contents and `_rng` seed are stored, so a test can give
this project's buffer the same ones; the `exp=droq`-shaped fixture stores its data and noise as seeds and hands the
reference a buffer stand-in that returns that data.  It starts the reference agent from `droq_oracle.init_params`
(a seed) and keeps the parameters after minibatch 1 and after the call at the fixed entries of
`droq_oracle.sample_state`: 2048 per tensor, fp32, as the reference computed them.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import droq_oracle as DO  # noqa: E402
from oracle import ref_harness as H  # noqa: E402
from oracle import sac_oracle as SO  # noqa: E402
from sheeprl_b200.utils.utils import dotdict  # noqa: E402

FIXTURES = {
    "droq_tiny": dict(obs_dim=5, act_dim=3, hidden=16, n_critics=3, B=8, p=0.2, low=(-2.0, -1.0, 0.0),
                      high=(1.0, 1.0, 3.0), G=3, calls=2, seed=5, rb=dict(size=16, n_envs=2, rng=11)),
    "droq_tiny_p0": dict(obs_dim=4, act_dim=2, hidden=12, n_critics=2, B=6, p=0.0, low=(-1.0, -1.0), high=(1.0, 1.0),
                         G=2, calls=2, seed=6, rb=dict(size=12, n_envs=2, rng=12)),
    "droq_exp": dict(obs_dim=8, act_dim=2, hidden=256, n_critics=2, B=256, p=0.01, low=(-1.0, -1.0), high=(1.0, 1.0),
                     G=80, calls=1, seed=7, rb=None, sampled=True),
}
LR, EPS = 3e-4, 1e-4


def droq_cfg(spec):
    opt = {"_target_": "torch.optim.Adam", "lr": LR, "eps": EPS, "weight_decay": 0, "betas": [0.9, 0.999]}
    return dotdict({"algo": {"name": "droq", "mlp_keys": {"encoder": ["state"]}, "cnn_keys": {"encoder": []},
                             "gamma": 0.99, "tau": 0.005, "per_rank_batch_size": spec["B"],
                             "actor": {"hidden_size": spec["hidden"], "optimizer": dict(opt)},
                             "critic": {"hidden_size": spec["hidden"], "n": spec["n_critics"], "dropout": spec["p"],
                                        "optimizer": dict(opt)},
                             "alpha": {"alpha": 1.0, "optimizer": dict(opt)}},
                    "buffer": {"sample_next_obs": False, "from_numpy": False}, "metric": {"sync_on_compute": False},
                    "distribution": {}, "seed": spec["seed"]})


def export(agent):
    out = {"actor": {k: v.detach().clone() for k, v in agent.actor.module.state_dict().items()
                     if k not in ("action_scale", "action_bias")}, "qf": {}, "qf_target": {},
           "log_alpha": {"log_alpha": agent.log_alpha.detach().clone()}}
    for i, (q, t) in enumerate(zip(agent.qfs, agent.qfs_target)):
        for k, v in q.module.state_dict().items():
            out["qf"][f"{i}.{k}"] = v.detach().clone()
        for k, v in t.module.state_dict().items():
            out["qf_target"][f"{i}.{k}"] = v.detach().clone()
    return out


def load_params(agent, P):
    """reference-keyed parameters (droq_oracle.init_params) into the reference agent's modules"""
    with torch.no_grad():
        agent.actor.module.load_state_dict(P["actor"], strict=False)     # action_scale / action_bias stay
        agent.log_alpha.copy_(P["log_alpha"]["log_alpha"])
        for group, mods in (("qf", agent.qfs), ("qf_target", agent.qfs_target)):
            for i, m in enumerate(mods):
                pre = f"{i}."
                m.module.load_state_dict({k[len(pre):]: v for k, v in P[group].items() if k.startswith(pre)})


def rb_contents(spec):
    """[size, n_envs, ...] float32 arrays of a full ring (reference main's step_data keys)"""
    r = spec["rb"]
    g = np.random.default_rng(spec["seed"])
    T, E = r["size"], r["n_envs"]
    return {"observations": g.standard_normal((T, E, spec["obs_dim"])).astype(np.float32),
            "next_observations": g.standard_normal((T, E, spec["obs_dim"])).astype(np.float32),
            "actions": g.uniform(-1, 1, (T, E, spec["act_dim"])).astype(np.float32),
            "rewards": g.standard_normal((T, E, 1)).astype(np.float32),
            "terminated": (g.uniform(size=(T, E, 1)) < 0.1).astype(np.float32),
            "truncated": np.zeros((T, E, 1), np.float32)}


class DataStandIn:
    """returns the given critic rows, then the actor rows, as `sample_tensors` would ([1, rows, ...])"""

    def __init__(self, critic, actor):
        self.queue = [critic, actor]

    def sample_tensors(self, n, **kw):
        d = self.queue.pop(0)
        assert next(iter(d.values())).shape[0] == n
        return {k: v.unsqueeze(0).clone() for k, v in d.items()}


def exp_data(spec):
    G, B = spec["G"], spec["B"]
    critic = SO.make_batch(G * B, spec["obs_dim"], spec["act_dim"], seed=spec["seed"] * 10 + 1)
    actor = SO.make_batch(B, spec["obs_dim"], spec["act_dim"], seed=spec["seed"] * 10 + 2)
    return critic, actor


def run(spec):
    import sheeprl.algos.droq.agent as A
    import sheeprl.algos.droq.droq as D
    import torch.distributions.normal as TN
    import torch.nn.functional as F
    from sheeprl.data.buffers import ReplayBuffer
    from sheeprl.utils.timer import timer

    timer.disabled = True
    A.get_single_device_fabric = lambda f: f
    cfg = droq_cfg(spec)
    n, G, B, p = spec["n_critics"], spec["G"], spec["B"], spec["p"]

    class Box:
        shape = (spec["act_dim"],)
        low = np.asarray(spec["low"], np.float32)
        high = np.asarray(spec["high"], np.float32)

    fab = H.FakeFabric()
    fab.all_reduce = lambda x, group=None: x
    torch.manual_seed(spec["seed"])
    agent, _ = A.build_agent(fab, cfg, {"state": H.Shape((spec["obs_dim"],))}, Box)
    sampled = spec.get("sampled", False)
    if sampled:
        load_params(agent, DO.init_params(spec["obs_dim"], spec["act_dim"], spec["hidden"], n, p, spec["seed"]))
    keep_state = DO.sample_state if sampled else (lambda s: s)
    out = {"spec": spec, "state_dict_keys": list(agent.state_dict().keys()), "calls": []}
    if not sampled:
        out["init"] = export(agent)
    qf_opt = torch.optim.Adam(agent.qfs.parameters(), lr=LR, eps=EPS)
    actor_opt = torch.optim.Adam(agent.actor.parameters(), lr=LR, eps=EPS)
    alpha_opt = torch.optim.Adam([agent.log_alpha], lr=LR, eps=EPS)
    if spec["rb"] is not None:
        r = spec["rb"]
        rb = ReplayBuffer(r["size"], r["n_envs"])
        rb.add(rb_contents(spec))
        rb._rng = np.random.default_rng(r["rng"])
    orig_normal, orig_dropout, orig_ema = TN._standard_normal, F.dropout, agent.qfs_target_ema
    for c in range(spec["calls"]):
        nseed = spec["seed"] * 100 + c
        eps_next, eps_cur, keep = DO.draw_noise(G, B, spec["act_dim"], n, spec["hidden"], p, nseed)
        nq, dq = [*eps_next, eps_cur], DO.reference_call_order(keep, G, n) if p > 0 else []
        TN._standard_normal = lambda shape, dtype, device: nq.pop(0).reshape(shape)

        def dropout(x, p_=0.5, training=True, inplace=False):
            assert training and p_ == p
            return x * (dq.pop(0).to(x.dtype) * (torch.tensor(1.0) / (1.0 - p_)))

        F.dropout = dropout
        emas, after1 = [0], {}

        def ema(critic_idx, _orig=orig_ema):
            _orig(critic_idx=critic_idx)
            emas[0] += 1
            if emas[0] == n:
                e = export(agent)
                after1.update(keep_state({"qf": e["qf"], "qf_target": e["qf_target"]}))

        agent.qfs_target_ema = ema
        if spec["rb"] is not None:
            src = rb
        else:
            src = DataStandIn(*exp_data(spec))
        seen = []

        class Recording:
            def sample_tensors(self, *a, **k):
                d = src.sample_tensors(*a, **k)
                seen.append({key: v.reshape(-1, *v.shape[2:]).float().clone() for key, v in d.items()})
                return d

        agg = H.RecordingAggregator()
        values = []
        agg.update = lambda name, v, _u=agg.update: (values.append(float(v.detach())) if name == "Loss/value_loss" else _u(name, v))
        try:
            D.train(fab, agent, actor_opt, qf_opt, alpha_opt, Recording(), agg, cfg, G)
        finally:
            TN._standard_normal, F.dropout = orig_normal, orig_dropout
            agent.qfs_target_ema = orig_ema
        assert not nq and not dq
        call = {"losses": dict(agg.values, **{"Loss/value_loss": values}), "after": keep_state(export(agent)),
                "qf_opt_steps": [int(s["step"]) for s in qf_opt.state_dict()["state"].values()],
                "qf_opt_state_len": len(qf_opt.state_dict()["state"])}
        if spec["rb"] is not None:
            call.update(eps_next=eps_next, eps_cur=eps_cur, keep=keep, critic_data=seen[0],
                        actor_obs=seen[1]["observations"])
        else:
            call.update(noise_seed=nseed, after_minibatch1=after1)
        out["calls"].append(call)
    if spec["rb"] is not None:
        out["rb"] = dict(spec["rb"], contents={k: torch.from_numpy(v) for k, v in rb_contents(spec).items()})
        out["qf_opt_state"] = qf_opt.state_dict()
    return out


def main():
    H.install()
    for name, spec in FIXTURES.items():
        if len(sys.argv) > 1 and name not in sys.argv[1:]:
            continue
        fx = run(spec)
        path = os.path.join(ROOT, "tests", "golden", f"{name}.pt")
        torch.save(fx, path)
        print(name, os.path.getsize(path), fx["calls"][-1]["losses"]["Loss/policy_loss"])


if __name__ == "__main__":
    main()
