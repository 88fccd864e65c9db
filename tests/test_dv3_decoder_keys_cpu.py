"""Decoders over a subset of the encoded keys (`cnn_keys.decoder` / `mlp_keys.decoder`) on the CPU: the oracle against the
executed-reference fixtures, the engine's kernel schedule on the torch test double against them (every gradient against
the oracle), state-dict layouts, the refusal of a decoder key that is not encoded, the player's `num_envs` resize and
the delegated `main` with `run_test: True`."""
import os

import pytest
import torch

from oracle import dv3_decoder_keys_oracle as ODK
from oracle import ref_harness
from oracle.make_golden_decoder_keys import FIXTURES as SPECS
from oracle.make_golden_decoder_keys import oracle_for
from oracle.ops_emul_decoupled import DecoupledEmulOps
from sheeprl_b200.configs import make_dv3_cfg
from sheeprl_b200.engine import DV3Engine
from tests.helpers import assert_params_close, image_channels, load_fixture
from tests.helpers import oracle_run as base_oracle_run

FIXTURES = list(SPECS)
LRS = {"wm": 1e-4, "actor": 8e-5, "critic": 8e-5}


def oracle_run(cfg, *a, **k):
    with oracle_for(cfg):
        return base_oracle_run(cfg, *a, **k)


def make_engine(cfg, adim, init, cont, ops):
    eng = DV3Engine(cfg, adim, in_channels=image_channels(cfg), device="cpu", ops=ops, is_continuous=cont)
    eng.wm.load(init["wm"]), eng.actor.load(init["actor"]), eng.critic.load(init["critic"]), eng.target.load(init["target"])
    return eng


def fixture_case(name):
    fx, cfg = load_fixture(name)
    fdata = [{k: v.float() for k, v in d.items()} for d in fx["data"]]
    return fx, cfg, fx["actions_dim"], len(fx["data"]), fx["is_continuous"], fdata


def check_grads(o_out, e_grads, cfg):
    """per tensor: |engine - oracle| <= 1e-4 (|oracle| + 1e-6 |all gradients|), after the oracle's clip"""
    for grp, max_norm in (("wm", cfg.algo.world_model.clip_gradients), ("actor", cfg.algo.actor.clip_gradients),
                          ("critic", cfg.algo.critic.clip_gradients)):
        og = o_out[f"grads/{grp}"]
        coef = min(1.0, max_norm / (float(o_out["Grads/" + {"wm": "world_model"}.get(grp, grp)]) + 1e-6))
        gnorm = float(torch.sqrt(sum((v.double() ** 2).sum() for v in og.values())))
        assert set(og) == set(e_grads[grp]), grp
        for k, v in og.items():
            diff = e_grads[grp][k] * coef - v
            rel = float(diff.double().norm()) / (float(v.double().norm()) + 1e-6 * gnorm + 1e-30)
            assert rel <= 1e-4, (grp, k, "per-tensor relative gradient error", rel)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_matches_the_executed_reference(name):
    fx, cfg, adim, steps, cont, fdata = fixture_case(name)
    a = cfg.algo
    assert list(a.cnn_keys.decoder) != list(a.cnn_keys.encoder) or list(a.mlp_keys.decoder) != list(a.mlp_keys.encoder)
    st, outs, ms, _ = oracle_run(cfg, adim, fx["init"], fdata, fx["noise"], steps, is_continuous=cont)
    for s in range(steps):
        for k, v in fx["metrics"][s].items():
            assert float(outs[s][k]) == pytest.approx(v, rel=3e-5, abs=1e-6), (s, k)
    for n in ("wm", "actor", "critic"):
        assert_params_close(st[n], fx["after"][n], LRS[n], steps, tol=2e-6, label=n)
    assert float(ms["high"]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


def test_decoder_keys_oracle_equals_the_coupled_oracle_when_the_keys_match():
    fx, cfg = load_fixture("dv3_tiny_v")
    fdata = [{k: v.float() for k, v in d.items()} for d in fx["data"]]
    a, _, _, _ = base_oracle_run(cfg, fx["actions_dim"], fx["init"], fdata, fx["noise"], 1)
    with ODK.decoder_keys():
        b, _, _, _ = base_oracle_run(cfg, fx["actions_dim"], fx["init"], fdata, fx["noise"], 1)
    for n in ("wm", "actor", "critic"):
        for k in a[n]:
            assert torch.allclose(a[n][k], b[n][k], rtol=0, atol=1e-6), (n, k)


@pytest.mark.skipif(not ref_harness.reference_available(), reason="the reference package is not installed")
def test_oracle_pinned_to_the_live_reference():
    from oracle.make_golden_decoder_keys import build_case

    cfg, adim, sd, data, noise, after, metrics, moments, (cp, ms) = build_case(dict(SPECS["dv3_dec_diambra"], steps=1), seed=3)
    for n, got in zip(("wm", "actor", "critic"), cp):
        assert_params_close(got, after[n], LRS[n], 1, tol=2e-6, label=n)
    assert float(ms["high"]) == pytest.approx(float(moments["high"]), rel=1e-4, abs=1e-7)


@pytest.mark.parametrize("name", FIXTURES)
def test_engine_schedule_matches_oracle_and_reference(name):
    fx, cfg, adim, steps, cont, fdata = fixture_case(name)
    _, o_outs, _, _ = oracle_run(cfg, adim, fx["init"], fdata, fx["noise"], steps, keep=True, is_continuous=cont)
    eng = make_engine(cfg, adim, fx["init"], cont, DecoupledEmulOps())
    e_outs = []
    for s in range(steps):
        eng.train_step({k: v.clone().float() for k, v in fx["data"][s].items()}, fx["noise"][s])
        e_outs.append({k: float(v) for k, v in eng.metrics_dict().items()})
        if s == 0:
            check_grads(o_outs[0], {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()}
                                    for g in ("wm", "actor", "critic")}, cfg)
    for s in range(steps):
        for k, v in fx["metrics"][s].items():
            assert e_outs[s][k] == pytest.approx(v, rel=3e-5, abs=1e-6), (s, k)
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        assert_params_close(g.views, fx["after"][n], LRS[n], steps, tol=2e-6, label=n)
    assert float(eng.moments_state[1]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


def test_only_the_decoders_that_exist_have_buffers():
    for name, cnn, vec in (("dv3_dec_crafter", True, False), ("dv3_dec_nocnn", False, True),
                           ("dv3_dec_diambra", True, True), ("dv3_dec_twoimg", True, True)):
        fx, cfg, adim, _, cont, _ = fixture_case(name)
        eng = make_engine(cfg, adim, fx["init"], cont, DecoupledEmulOps())
        assert (eng.has_cnn_dec, eng.has_vec_dec) == (cnn, vec), name
        assert ("recon" in eng._bufs) == cnn and ("dec_lin" in eng._bufs) == cnn, name
        assert ("vrecon" in eng._bufs) == vec and ("vdec.out" in eng._bufs or "vdec.act0" in eng._bufs) == vec, name
    # decoder == encoder: the targets are the encoder's inputs, no extra buffers
    fx, cfg = load_fixture("dv3_tiny_v")
    eng = make_engine(cfg, fx["actions_dim"], fx["init"], False, DecoupledEmulOps())
    assert eng.x_dec is eng.x0 and eng.vtgt is eng.vx and "x_dec" not in eng._bufs and "vtgt" not in eng._bufs


class Space:
    def __init__(self, *shape):
        self.shape = shape


def obs_space_of(cfg):
    cch = dict(cfg.env.get("cnn_channels", {}) or {})
    sp = {k: Space(cch.get(k, 3), 64, 64) for k in cfg.algo.cnn_keys.encoder}
    sp.update({k: Space(d) for k, d in cfg.env.mlp_dims.items()})
    return sp


class Fab:
    device = torch.device("cpu")


@pytest.mark.parametrize("name", FIXTURES)
def test_state_dict_keys_and_shapes_are_the_reference_ones(name):
    """fx["init"] is the reference build_agent's state dict: same keys and shapes, and it loads both ways"""
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent

    fx, cfg = load_fixture(name)
    wm, actor, critic, target, player = build_agent(Fab, fx["actions_dim"], fx["is_continuous"], cfg, obs_space_of(cfg),
                                                    ops=DecoupledEmulOps())
    for mod, n in ((wm, "wm"), (actor, "actor"), (critic, "critic"), (target, "target")):
        assert {k: tuple(v.shape) for k, v in mod.state_dict().items()} == \
            {k: tuple(v.shape) for k, v in fx["init"][n].items()}, n
        mod.load_state_dict(fx["init"][n])
        assert all(torch.equal(v, fx["init"][n][k]) for k, v in mod.state_dict().items()), n


@pytest.mark.parametrize("kind", ["cnn_keys", "mlp_keys"])
def test_decoder_key_that_is_not_encoded_is_refused(kind):
    over = {f"algo__{kind}__decoder": ["rgb", "depth"] if kind == "cnn_keys" else ["state", "missing"]}
    cfg = make_dv3_cfg(**dict(SPECS["dv3_dec_crafter"]["cfg"], mlp_keys={"state": 2}, **over))
    with pytest.raises(ValueError, match="depth" if kind == "cnn_keys" else "missing"):
        DV3Engine(cfg, (2,), device="cpu", ops=DecoupledEmulOps())


def test_both_decoders_empty_is_refused():
    cfg = make_dv3_cfg(**dict(SPECS["dv3_dec_crafter"]["cfg"], algo__cnn_keys__decoder=[]))
    with pytest.raises(ValueError, match="at least one decoder"):
        DV3Engine(cfg, (2,), device="cpu", ops=DecoupledEmulOps())


def test_minedojo_actor_is_refused():
    cfg = make_dv3_cfg(**dict(SPECS["dv3_dec_crafter"]["cfg"], algo__actor__cls="sheeprl.algos.dreamer_v3.agent.MinedojoActor"))
    with pytest.raises(NotImplementedError, match="MineDojo"):
        DV3Engine(cfg, (2,), device="cpu", ops=DecoupledEmulOps())


def test_player_resizes_to_num_envs_and_ignores_masks():
    """`player.num_envs = n` (the reference's test()) re-creates the acting rows over the same parameters; a mask dict is
    ignored by the plain actor, as `Actor.forward` ignores it"""
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent

    fx, cfg = load_fixture("dv3_dec_diambra")
    cfg.env.num_envs = 3
    *_, player = build_agent(Fab, fx["actions_dim"], False, cfg, obs_space_of(cfg), ops=DecoupledEmulOps())
    eng = player.eng
    assert player.num_envs == 3 and player.actions.shape[1] == 3
    player.num_envs = 3
    assert player.eng is eng                                           # unchanged size: nothing re-created
    player.num_envs = 1
    player.init_states()
    assert player.eng is not eng and player.eng.wm is eng.wm and player.eng.actor is eng.actor
    g = torch.Generator().manual_seed(0)
    obs = {"rgb": torch.rand(1, 1, 3, 64, 64, generator=g) - 0.5}
    obs.update({k: torch.randn(1, 1, d, generator=g) for k, d in cfg.env.mlp_dims.items()})
    noise = {"z": torch.ones(1, player.eng.Z), "a": torch.ones(1, player.eng.A)}
    acts = player.get_actions(obs, False, {}, noise=noise)
    assert [tuple(x.shape) for x in acts] == [(1, 1, ad) for ad in fx["actions_dim"]]
    player.init_states()
    again = player.get_actions(obs, False, {"mask_action_type": torch.zeros(1, 1, 3)}, noise=noise)
    assert all(torch.equal(x, y) for x, y in zip(acts, again))


@pytest.mark.skipif(not ref_harness.reference_available(), reason="the reference package is not installed")
def test_delegated_main_runs_the_crafter_shape_with_run_test(tmp_path):
    """the reference's own `main` on an image + 1-d vector environment with `mlp_keys.decoder: []`, 2 environments and
    `run_test: True`: the reference's test() resizes the player to one environment and passes an empty mask dict"""
    import sheeprl_b200.algos.dreamer_v3.agent as A
    import sheeprl_b200.algos.dreamer_v3.dreamer_v3 as B
    from sheeprl_b200.data import buffers as Bf
    from tests import fake_gym
    from tests.test_main_delegation_cpu import Fabric, _harness, _loop_cfg

    R = _harness(tmp_path)
    import sheeprl.algos.dreamer_v3.utils as RU

    env_fn = lambda cfg, seed, rank_off, log_dir, prefix, vector_env_idx=0: (  # noqa: E731
        lambda: fake_gym.DummyImageEnv(seed=seed, vector_dim=1))
    orig_make_env, R.make_env, RU.make_env = RU.make_env, env_fn, env_fn
    os.makedirs(tmp_path / "run" / "checkpoint", exist_ok=True)
    cfg, fab = _loop_cfg(tmp_path, run_test=True), Fabric(tmp_path)
    cfg.env.num_envs = 2
    cfg.algo.mlp_keys.encoder, cfg.algo.mlp_keys.decoder = ["state"], []
    engines, players, orig_train, orig_test = [], [], B.train, R.test

    def counting_train(*a, **k):
        engines.append(a[1]._b200_engine)
        return orig_train(*a, **k)

    def recording_test(player, *a, **k):
        players.append(player)
        return orig_test(player, *a, **k)

    A.DEFAULT_OPS, Bf.DEFAULTS["ops"] = DecoupledEmulOps(), DecoupledEmulOps()
    B.train, R.test = counting_train, recording_test
    try:
        B.main(fab, cfg)
    finally:
        B.train, R.test, RU.make_env = orig_train, orig_test, orig_make_env
        A.DEFAULT_OPS, Bf.DEFAULTS["ops"], Bf.DEFAULTS["device"] = None, None, "cuda"
    assert len(engines) >= 3 and not engines[0].has_vec_dec and engines[0].vec_keys == ["state"]
    assert len(players) == 1 and players[0].num_envs == 1
    (ck,) = fab.checkpoints
    wm = ck["state"]["world_model"]
    assert not any(k.startswith("observation_model.mlp_decoder") for k in wm)
    assert "encoder.mlp_encoder.model._model.0.weight" in wm
    assert all(torch.isfinite(v).all() for v in wm.values())
