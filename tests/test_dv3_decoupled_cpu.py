"""Decoupled RSSM (`algo.world_model.decoupled_rssm=True`; reference DecoupledRSSM, agent.py:501-593) on the CPU: the
oracle against the executed-reference fixtures, the engine's kernel schedule on the torch test double against the oracle,
the persistent-scan schedule against the per-step one, the public surface and Plan2Explore's refusal."""
import os

import pytest
import torch

from oracle import dv3_decoupled_oracle as OD
from oracle import ref_harness
from oracle.ops_emul_decoupled import DecoupledEmulOps
from sheeprl_b200.engine import DV3Engine
from tests.helpers import GOLDEN, assert_params_close, image_channels, load_fixture
from tests.helpers import oracle_run as coupled_oracle_run

FIXTURES = ["dv3_tiny_d", "dv3_tiny_dv"]
LRS = {"wm": 1e-4, "actor": 8e-5, "critic": 8e-5}


def oracle_run(*a, **k):
    with OD.decoupled():
        return coupled_oracle_run(*a, **k)


class TraceOps(DecoupledEmulOps):
    """records the name of every op the engine issues"""

    def __init__(self):
        self.trace = []

    def __getattribute__(self, name):
        attr = object.__getattribute__(self, name)
        if callable(attr) and not name.startswith("_"):
            object.__getattribute__(self, "trace").append(name)
        return attr


def make_engine(cfg, adim, init, cont, ops):
    eng = DV3Engine(cfg, adim, in_channels=image_channels(cfg), device="cpu", ops=ops, is_continuous=cont)
    eng.wm.load(init["wm"]), eng.actor.load(init["actor"]), eng.critic.load(init["critic"]), eng.target.load(init["target"])
    return eng


def fixture_case(name):
    fx, cfg = load_fixture(name)
    fdata = [{k: v.float() for k, v in d.items()} for d in fx["data"]]
    return fx, cfg, fx["actions_dim"], len(fx["data"]), fx["is_continuous"], fdata


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_matches_the_executed_reference(name):
    """post-step parameters of all three optimisers, the 13 metrics and Moments of the unmodified reference train()"""
    fx, cfg, adim, steps, cont, fdata = fixture_case(name)
    assert cfg.algo.world_model.decoupled_rssm
    assert any(float(d["is_first"][1:].sum()) > 0 for d in fx["data"]), "no is_first mid-sequence"
    st, outs, ms, _ = oracle_run(cfg, adim, fx["init"], fdata, fx["noise"], steps, is_continuous=cont)
    for s in range(steps):
        assert len(fx["metrics"][s]) == 13
        for k, v in fx["metrics"][s].items():
            assert float(outs[s][k]) == pytest.approx(v, rel=3e-5, abs=1e-6), (s, k)
    for n in ("wm", "actor", "critic"):
        assert_params_close(st[n], fx["after"][n], LRS[n], steps, tol=2e-6, label=n)
    assert float(ms["low"]) == pytest.approx(float(fx["moments"]["low"]), rel=1e-4, abs=1e-7)
    assert float(ms["high"]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


@pytest.mark.skipif(not ref_harness.reference_available(), reason="the reference package is not installed")
def test_oracle_pinned_to_the_live_reference():
    """a fresh seed through the reference's own train() (one posterior draw over [T,B,S,D], then one discarded prior
    draw per step) and through the oracle"""
    from oracle.make_golden_decoupled import FIXTURES as SPECS, build_case

    cfg, adim, sd, data, noise, after, metrics, moments, (cp, ms) = build_case(dict(SPECS["dv3_tiny_d"], steps=1), seed=3)
    for n, got in zip(("wm", "actor", "critic"), cp):
        assert_params_close(got, after[n], LRS[n], 1, tol=2e-6, label=n)
    assert float(ms["high"]) == pytest.approx(float(moments["high"]), rel=1e-4, abs=1e-7)


@pytest.mark.parametrize("name", FIXTURES)
def test_engine_schedule_matches_oracle_and_reference(name):
    fx, cfg, adim, steps, cont, fdata = fixture_case(name)
    st, o_outs, ms, _ = oracle_run(cfg, adim, fx["init"], fdata, fx["noise"], steps, keep=True, is_continuous=cont)
    eng = make_engine(cfg, adim, fx["init"], cont, DecoupledEmulOps())
    assert eng.decoupled and eng.fused_scan and eng.fused_scan_bwd
    e_outs, e_grads = [], []
    for s in range(steps):
        eng.train_step({k: v.clone().float() for k, v in fx["data"][s].items()}, fx["noise"][s])
        e_outs.append({k: float(v) for k, v in eng.metrics_dict().items()})
        e_grads.append({g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")})
    for grp, max_norm in (("wm", cfg.algo.world_model.clip_gradients), ("actor", cfg.algo.actor.clip_gradients),
                          ("critic", cfg.algo.critic.clip_gradients)):
        og = o_outs[0][f"grads/{grp}"]
        coef = min(1.0, max_norm / (float(o_outs[0]["Grads/" + {"wm": "world_model"}.get(grp, grp)]) + 1e-6))
        gnorm = float(torch.sqrt(sum((v.double() ** 2).sum() for v in og.values())))
        for k, v in og.items():
            diff = e_grads[0][grp][k] * coef - v
            rel = float(diff.double().norm()) / (float(v.double().norm()) + 1e-6 * gnorm + 1e-30)
            assert rel <= 1e-4, (grp, k, "per-tensor relative gradient error", rel)
    for s in range(steps):
        for k, v in fx["metrics"][s].items():
            assert e_outs[s][k] == pytest.approx(v, rel=3e-5, abs=1e-6), (s, k)
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        assert_params_close(g.views, fx["after"][n], LRS[n], steps, tol=2e-6, label=n)
    assert float(eng.moments_state[1]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


@pytest.mark.parametrize("name", FIXTURES)
def test_persistent_scan_schedule_equals_per_step_schedule(name):
    """what the envelope query selects is the only difference between the two schedules: same saves, same gradients"""
    fx, cfg, adim, steps, cont, fdata = fixture_case(name)
    outs = []
    for fused in (True, False):
        eng = make_engine(cfg, adim, fx["init"], cont, TraceOps())
        eng.fused_scan = fused
        eng.ops.trace.clear()
        eng.train_step({k: v.clone().float() for k, v in fx["data"][0].items()}, fx["noise"][0])
        assert ("gru_scan_fwd" in eng.ops.trace) == fused and ("gru_scan_bwd" in eng.ops.trace) == fused
        outs.append({k: getattr(eng, k).clone() for k in ("latent", "h_in", "g_pre", "g_ln", "d_g_ln", "d_g_pre", "d_x_pre",
                                                          "d_post_raw", "d_h0")} | {"grad": eng.wm.grad.clone()})
    for k in outs[0]:
        err = float((outs[0][k] - outs[1][k]).abs().max())
        assert err <= 1e-5 * max(1e-3, float(outs[0][k].abs().max())), (k, err)


def test_state_dict_keys_and_shapes_are_the_reference_ones():
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent

    fx, cfg = load_fixture("dv3_tiny_d")

    class Fab:
        device = torch.device("cpu")

    class Space:
        shape = (3, 64, 64)

    wm, actor, critic, target, player = build_agent(Fab, fx["actions_dim"], False, cfg, {"rgb": Space}, ops=DecoupledEmulOps())
    for mod, n in ((wm, "wm"), (actor, "actor"), (critic, "critic"), (target, "target")):
        sd = mod.state_dict()
        assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in fx["init"][n].items()}, n
    E = wm._b200_engine.E
    assert wm.state_dict()["rssm.representation_model._model.0.weight"].shape[1] == E     # no h columns
    wm.load_state_dict(fx["init"]["wm"])                                          # a reference state dict loads
    assert torch.equal(wm._b200_engine.wm.views["rssm.representation_model._model.0.weight"],
                       fx["init"]["wm"]["rssm.representation_model._model.0.weight"])


def test_player_matches_reference():
    from tests.test_player_cpu import check, run_player

    assert os.path.exists(os.path.join(GOLDEN, "dv3_player_decoupled.pt"))
    fx, got, cont = run_player("dv3_player_decoupled", ops=DecoupledEmulOps())
    check(fx, got, cont)


def test_plan2explore_refuses_decoupled_rssm():
    from sheeprl_b200.algos.p2e_dv3.agent import build_agent
    from sheeprl_b200.configs import make_p2e_dv3_cfg

    fx, _ = load_fixture("dv3_tiny_d")
    cfg = make_p2e_dv3_cfg(n_ensembles=2, **fx["cfg_kwargs"])

    class Fab:
        device = torch.device("cpu")

    class Space:
        shape = (3, 64, 64)

    with pytest.raises(NotImplementedError, match="five-argument"):
        build_agent(Fab, (3,), False, cfg, {"rgb": Space}, ops=DecoupledEmulOps())


@pytest.mark.skipif(not ref_harness.reference_available(), reason="the reference package is not installed")
def test_delegated_main_runs_with_decoupled_rssm(tmp_path):
    """the reference's own `main` (DecoupledRSSM player, ratio governor, checkpoint) around this package's build_agent /
    train with the switch on"""
    import sheeprl_b200.algos.dreamer_v3.agent as A
    import sheeprl_b200.algos.dreamer_v3.dreamer_v3 as B
    from sheeprl_b200.data import buffers as Bf
    from tests.test_main_delegation_cpu import Fabric, _harness, _loop_cfg

    _harness(tmp_path)
    os.makedirs(tmp_path / "run" / "checkpoint", exist_ok=True)
    cfg, fab = _loop_cfg(tmp_path), Fabric(tmp_path)
    cfg.algo.world_model.decoupled_rssm = True
    engines, orig_train = [], B.train

    def counting_train(*a, **k):
        engines.append(a[1]._b200_engine)
        return orig_train(*a, **k)

    A.DEFAULT_OPS, Bf.DEFAULTS["ops"] = DecoupledEmulOps(), DecoupledEmulOps()
    B.train = counting_train
    try:
        B.main(fab, cfg)
    finally:
        B.train = orig_train
        A.DEFAULT_OPS, Bf.DEFAULTS["ops"], Bf.DEFAULTS["device"] = None, None, "cuda"
    assert len(engines) >= 3 and engines[0].decoupled
    (ck,) = fab.checkpoints
    wm = ck["state"]["world_model"]
    assert wm["rssm.representation_model._model.0.weight"].shape[1] == engines[0].E
    assert all(torch.isfinite(v).all() for v in wm.values())
