"""Record the op sequence the PPO, A2C, recurrent PPO, SAC and DroQ engines and their players issue on the CPU test
double, so that two revisions can be diffed: `python tools/trace_dense_ops.py > a.txt` on each, then `diff`.

Every `ops.*` call is one line: method name, scalar arguments, and per tensor (storage id in order of first appearance,
storage offset, shape, stride, dtype).  The torch ops the engines issue outside `ops` calls are recorded the same way
through a `TorchDispatchMode`; view ops are left out, since they launch nothing (binding a transpose once instead of
per call changes no launch).  The scenarios are the committed fixtures' configurations driven through the tests'
entry points, plus a few configurations no fixture has."""
from __future__ import annotations

import functools
import inspect
import os
import re
import sys

import torch
from torch.utils._python_dispatch import TorchDispatchMode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LINES: list = []
STORAGES: dict = {}
DEPTH = [0]


def desc(v):
    if isinstance(v, torch.Tensor):
        st = v.untyped_storage()
        if st.data_ptr() not in STORAGES:                  # holding the storage keeps its address from being reused
            STORAGES[st.data_ptr()] = (len(STORAGES), st)
        return f"T(s{STORAGES[st.data_ptr()][0]}+{v.storage_offset()},{tuple(v.shape)},{v.stride()},{str(v.dtype)[6:]})"
    if isinstance(v, (torch.UntypedStorage, torch.TypedStorage)):
        return f"S({v.nbytes()})"
    if isinstance(v, (list, tuple)):
        return "[" + ",".join(desc(x) for x in v) + "]"
    if isinstance(v, float):
        return repr(float(v))
    return re.sub(r" at 0x[0-9a-f]+", "", repr(v))           # generators, record-function handles


def record(name, args, kwargs, out=None):
    items = [desc(a) for a in args] + [f"{k}={desc(v)}" for k, v in kwargs.items()]
    line = f"{name}(" + ", ".join(items) + ")"
    if out is not None:
        line += " -> " + desc(out)
    LINES.append(line)


def wrap_ops(cls):
    """record every public method of an ops class (and its subclasses, which inherit or override them)"""
    for name, fn in list(vars(cls).items()):
        if name.startswith("_") or not inspect.isfunction(fn) or getattr(fn, "_traced", False):
            continue

        def make(fn, name):
            sig = inspect.signature(fn)

            @functools.wraps(fn)
            def w(self, *a, **k):
                if DEPTH[0] == 0:                          # bound with defaults: `epi="none"` and no `epi` are one call
                    bound = sig.bind(self, *a, **k)
                    bound.apply_defaults()
                    record("ops." + name, [], dict(list(bound.arguments.items())[1:]))
                DEPTH[0] += 1
                try:
                    return fn(self, *a, **k)
                finally:
                    DEPTH[0] -= 1
            w._traced = True
            return w

        setattr(cls, name, make(fn, name))


ALLOCS = ("empty.memory_format", "empty_strided.default", "empty_like.default", "zeros.default", "zeros_like.default")
ALLOCATED: list = []


class AtenRecorder(TorchDispatchMode):
    """Allocations are not part of the sequence (the order in which buffers are created launches nothing on a step);
    each scenario ends with the sorted list of every allocation it made instead, so a new or missing buffer shows."""

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        out = func(*args, **kwargs)
        if DEPTH[0] == 0 and not func.is_view and func.__name__ not in ("detach.default", "alias.default"):
            if func.__name__ in ALLOCS:
                ALLOCATED.append(f"{func.__name__} {tuple(out.shape)} {str(out.dtype)[6:]}")
            else:
                record("aten." + func.__name__, args, kwargs, out if isinstance(out, torch.Tensor) else None)
        return out


# ---------------------------------------------------------------------------------------------------------------------
def scenarios():
    from oracle.make_golden_ppo import obs_space, ppo_cfg, split_obs
    from tests import test_a2c_cpu as A2C
    from tests import test_droq_cpu as DQ
    from tests import test_ppo_cpu as PPO
    from tests import test_ppo_recurrent_cpu as REC
    from tests import test_sac_cpu as SAC

    for name in PPO.NAMES:
        yield f"ppo engine {name}", lambda name=name: PPO.check_engine(PPO.load(name), PPO.make_engine(PPO.load(name)), name)
    for name in PPO.PLAYER_NAMES:
        yield f"ppo player {name}", lambda name=name: PPO.check_player(name)

    def ppo_public(name, spec_edit=None):
        from oracle.ops_emul import EmulOps
        from sheeprl_b200.algos.ppo.agent import build_agent
        from sheeprl_b200.algos.ppo.ppo import make_optimizer, train

        fx = PPO.load(name)
        spec = dict(fx["spec"])
        if spec_edit:
            spec_edit(spec)
        cfg = ppo_cfg(spec, fx["hp"], fx["batch"], fx["epochs"])
        agent, player = build_agent(_Fab, spec["actions_dim"], spec["is_continuous"], cfg, obs_space(spec), ops=EmulOps())
        opt = make_optimizer(agent, cfg)
        torch.manual_seed(0)
        train(_Fab, agent, opt, split_obs(spec, fx["data"]), None, cfg)
        obs = split_obs(spec, {k: v[:3] for k, v in fx["data"].items()})
        player(obs), player.get_values(obs), player.get_actions(obs, greedy=True), player.get_actions(obs)

    yield "ppo public tanh_ln", lambda: ppo_public("ppo_tanh_ln")
    yield "ppo public multikey", lambda: ppo_public("ppo_multikey")

    def no_actor_layers(spec):
        spec["nets"] = {"actor": (spec["mlp_features"], 0)}

    yield "ppo public actor.mlp_layers=0", lambda: ppo_public("ppo_vector", no_actor_layers)

    for name in A2C.NAMES:
        yield f"a2c engine {name}", lambda name=name: A2C.check_engine(name)

    for name in REC.NAMES:
        yield f"rec engine {name}", lambda name=name: REC.check_engine(REC.load(name), REC.make_engine(REC.load(name)), name)

    def rec_variant(name, rnn):
        fx = REC.load(name)
        fx["spec"] = dict(fx["spec"], rnn=rnn)
        from oracle import ppo_recurrent_oracle as RO

        fx["init"] = RO.init_params(fx["spec"], 0)
        eng = REC.make_engine(fx)
        eng.train({k: v for k, v in fx["data"].items()}, fx["index_batches"])

    yield "rec pre/post no LN", lambda: rec_variant("ppo_rec_branches", {"hidden": 48, "pre": (24, False), "post": (48, False)})
    yield "rec pre LN, post none", lambda: rec_variant("ppo_rec_branches", {"hidden": 48, "pre": (24, True), "post": None})
    yield "rec pre none, post plain", lambda: rec_variant("ppo_rec_pixel", {"hidden": 64, "pre": None, "post": (64, False)})
    for name in REC.NAMES:
        yield f"rec public {name}", lambda name=name: rec_public(REC, name)
        yield f"rec player {name}", lambda name=name: REC.check_player(name)

    for name in ("sac_tiny", "sac_c4"):
        yield f"sac engine {name}", lambda name=name: SAC.check_engine(SAC.load(name), SAC.make_engine(SAC.load(name)), name)
    yield "sac engine 3 critics", sac_three_critics
    yield "sac public + batch change", lambda: sac_public(SAC)
    yield "sac player", SAC.test_player_greedy_and_sampled_actions

    for name in DQ.NAMES:
        yield f"droq engine {name}", lambda name=name: DQ.check_engine(DQ.load(name), DQ.make_engine(DQ.load(name)), name)
    yield "droq exp first minibatch", lambda: DQ.check_engine_first_minibatch(DQ.load("droq_exp"), DQ.make_engine(DQ.load("droq_exp")))
    yield "droq public", lambda: droq_public(DQ)


class _Fab:
    device, world_size, global_rank = torch.device("cpu"), 1, 0


def rec_public(REC, name):
    from sheeprl_b200.algos.ppo_recurrent.ppo_recurrent import make_optimizer, train

    fx = REC.load(name)
    cfg = REC._cfg(fx, num_envs=2)
    agent, player = REC._build(fx, cfg)
    opt = make_optimizer(agent, cfg)
    torch.manual_seed(fx["sampler_seed"])
    train(_Fab, agent, opt, {k: v.clone() for k, v in fx["data"].items()}, None, cfg)


def sac_public(SAC):
    import numpy as np

    from oracle.make_golden_sac import sac_cfg
    from oracle.ops_emul import EmulOps
    from sheeprl_b200.algos.sac.agent import build_agent
    from sheeprl_b200.algos.sac.sac import make_optimizers, train

    class Space:
        def __init__(self, shape):
            self.shape = shape

    class Box:
        shape, low, high = (3,), np.full(3, -2.0, np.float32), np.full(3, 1.0, np.float32)

    cfg = sac_cfg(16, 2)
    cfg.algo.per_rank_batch_size = 8
    agent, player = build_agent(_Fab, cfg, {"state": Space((5,))}, Box, ops=EmulOps())
    opts = make_optimizers(agent, cfg)
    g = torch.Generator().manual_seed(1)
    for u, B in enumerate((8, 8, 5, 8)):
        data = {"observations": torch.randn(B, 5, generator=g), "next_observations": torch.randn(B, 5, generator=g),
                "actions": torch.rand(B, 3, generator=g), "rewards": torch.randn(B, 1, generator=g),
                "terminated": torch.zeros(B, 1)}
        train(_Fab, agent, *opts, data, None, u + 1, cfg, 1)
    obs = torch.randn(4, 5, generator=g)
    player.get_actions(obs, greedy=True), player.get_actions(obs), player(obs[:2])


def sac_three_critics():
    from oracle.ops_emul import EmulOps
    from sheeprl_b200.algos.sac.agent import _default_linear_init
    from sheeprl_b200.algos.sac.engine import SACEngine

    opt = {"lr": 3e-4, "eps": 1e-4, "betas": (0.9, 0.999)}
    eng = SACEngine(5, 3, 16, 12, 3, 8, 0.99, 0.005, 1.0, -1.0, 1.0, opt, opt, opt, "cpu", EmulOps(), seed=3)
    g = torch.Generator().manual_seed(2)
    eng.actor.load(_default_linear_init(eng.actor.shapes, g))
    eng.qf.load(_default_linear_init(eng.qf.shapes, g))
    eng.qf_target.load(eng.qf.state_dict())
    for u in range(3):
        data = {"observations": torch.randn(8, 5, generator=g), "next_observations": torch.randn(8, 5, generator=g),
                "actions": torch.rand(8, 3, generator=g), "rewards": torch.randn(8, 1, generator=g),
                "terminated": torch.zeros(8, 1)}
        eng.train_step(data, u % 2 == 0)


def droq_public(DQ):
    from sheeprl_b200.algos.droq.droq import make_optimizers

    fx = DQ.load("droq_tiny")
    sp = fx["spec"]
    agent, player = DQ.build(sp)
    agent.load_state_dict(DQ.reference_state_dict(fx))
    make_optimizers(agent, DQ.make_cfg(sp))
    critic, actor_obs = DQ.call_inputs(fx, 0)[:2]
    eng = agent._b200_engine
    eng.train_call(critic, actor_obs)                                            # device-drawn noise and masks
    eng.train_call({k: v[:sp["B"]] for k, v in critic.items()}, actor_obs)      # G changes between calls
    player.get_actions(actor_obs[:3], greedy=True), player.get_actions(actor_obs[:3])


def main():
    from oracle import ops_emul

    mods = [ops_emul]
    for m in ("ops_emul_a2c", "ops_emul_droq", "ops_emul_recurrent"):
        mods.append(__import__(f"oracle.{m}", fromlist=["x"]))
    seen = set()
    for m in mods:
        for v in vars(m).values():
            if isinstance(v, type) and v.__name__.endswith("EmulOps") and v not in seen:
                seen.add(v)
                wrap_ops(v)
    torch.manual_seed(0)
    for title, run in scenarios():
        LINES.clear(), STORAGES.clear(), ALLOCATED.clear()
        with AtenRecorder():
            try:
                run()
            except Exception as e:                                   # a failing scenario is part of the trace
                LINES.append(f"EXCEPTION {type(e).__name__}: {e}")
        print(f"=== {title}: {len(LINES)} lines")
        for line in LINES:
            print(line)
        print(f"--- {title}: {len(ALLOCATED)} allocations")
        for line in sorted(ALLOCATED):
            print(line)


if __name__ == "__main__":
    main()
