"""The MineDojo actor (`algo.actor.cls: MinedojoActor`) in Dreamer-V3 and Plan2Explore on the CPU: the oracle and the
engine's kernel schedule on the torch test double against the executed-reference fixtures (tests/golden/dv3_minedojo.pt,
tests/golden/p2e_minedojo.pt, oracle/make_golden_minedojo.py), mode actions in imagination, state dicts, the
refusals, the player's masked sample against the reference MinedojoActor, the masked acting step's op trace, the
replay buffers' mask / equipment dtypes and the reference's own `main` on a MultiDiscrete environment with mask keys."""
import copy
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import ref_harness
from oracle.make_golden_minedojo import ACTIONS_DIM, DV3_ACTOR, MASKS, P2E_ACTOR
from oracle.ops_emul_minedojo import MASK_KEYS, MinedojoEmulOps, minedojo_sample_spec
from sheeprl_b200.configs import make_dv3_cfg, make_p2e_dv3_cfg
from sheeprl_b200.engine import DV3Engine
from tests.helpers import GOLDEN, assert_params_close, image_channels, load_fixture
from tests.test_dv3_decoder_keys_cpu import LRS, Fab, check_grads, obs_space_of, oracle_run
from tests.test_p2e_cpu import LR, check_metrics, check_moments

needs_reference = pytest.mark.skipif(not ref_harness.reference_available(), reason="the reference package is not installed")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dv3_case():
    fx, cfg = load_fixture("dv3_minedojo")
    return fx, cfg, [{k: v.float() for k, v in d.items()} for d in fx["data"]]


def dv3_engine(fx, cfg, ops=None):
    eng = DV3Engine(cfg, fx["actions_dim"], in_channels=image_channels(cfg), device="cpu", ops=ops or MinedojoEmulOps())
    for n in ("wm", "actor", "critic", "target"):
        getattr(eng, n).load(fx["init"][n])
    return eng


def p2e_case():
    fx = torch.load(os.path.join(GOLDEN, "p2e_minedojo.pt"), weights_only=False)
    return fx, make_p2e_dv3_cfg(**fx["cfg"])


def p2e_engine(fx, cfg, ops=None):
    from sheeprl_b200.algos.p2e_dv3.engine import P2EDV3Engine

    eng = P2EDV3Engine(cfg, fx["actions_dim"], in_channels=3, device="cpu", ops=ops or MinedojoEmulOps())
    for name, g in eng.groups().items():
        g.load(fx["init"][name])
    eng.load_ensembles(fx["init"]["ens"])
    return eng


def without_action_noise(noise):
    return {k: v for k, v in noise.items() if not k.startswith("img_action")}


# ------------------------------------------------------------------ training: fixtures from the executed reference
def test_fixtures_have_the_minedojo_layout():
    fx, cfg, _ = dv3_case()
    assert tuple(fx["actions_dim"]) == ACTIONS_DIM and str(cfg.algo.actor.cls) == DV3_ACTOR
    assert list(cfg.algo.mlp_keys.encoder) == list(cfg.algo.mlp_keys.decoder) == list(MASKS)
    fx, cfg = p2e_case()
    assert str(cfg.algo.actor.cls) == P2E_ACTOR and list(cfg.algo.mlp_keys.decoder) == list(MASKS)
    for name in ("dv3_minedojo", "p2e_minedojo"):
        assert os.path.getsize(os.path.join(GOLDEN, name + ".pt")) < 1 << 20


def test_dv3_oracle_matches_the_executed_reference():
    fx, cfg, fdata = dv3_case()
    st, outs, ms, _ = oracle_run(cfg, ACTIONS_DIM, fx["init"], fdata, fx["noise"], len(fdata))
    for s, m in enumerate(fx["metrics"]):
        for k, v in m.items():
            assert float(outs[s][k]) == pytest.approx(v, rel=3e-5, abs=1e-6), (s, k)
    for n in ("wm", "actor", "critic"):
        assert_params_close(st[n], fx["after"][n], LRS[n], len(fdata), tol=2e-6, label=n)
    assert float(ms["high"]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


def test_dv3_engine_imagines_mode_actions_and_matches_the_reference():
    fx, cfg, fdata = dv3_case()
    _, o_outs, _, _ = oracle_run(cfg, ACTIONS_DIM, fx["init"], fdata, fx["noise"], 1, keep=True)
    eng = dv3_engine(fx, cfg)
    assert eng.minedojo
    for s in range(len(fdata)):
        eng.train_step({k: v.clone() for k, v in fdata[s].items()}, without_action_noise(fx["noise"][s]))
        if s == 0:
            check_grads(o_outs[0], {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()}
                                    for g in ("wm", "actor", "critic")}, cfg)
            want = o_outs[0]["imagined_actions"]
            assert torch.equal(eng.actions, want), "imagined actions differ from the reference's mode actions"
            # the mode: the arg-max of each head's logits on the imagined state
            off = 0
            for ad in ACTIONS_DIM:
                raw = eng.actor_raw.view(*eng.actions.shape[:2], -1)[..., off:off + ad]
                assert torch.equal(eng.actions[..., off:off + ad].argmax(-1), raw.argmax(-1))
                off += ad
        for k, v in fx["metrics"][s].items():
            assert float(eng.metrics_dict()[k]) == pytest.approx(v, rel=3e-5, abs=1e-6), (s, k)
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        assert_params_close(g.views, fx["after"][n], LRS[n], len(fdata), tol=2e-6, label=n)
    assert float(eng.moments_state[1]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


def test_p2e_oracle_matches_the_executed_reference():
    from oracle.make_golden_minedojo import run_oracle_p2e

    fx, cfg = p2e_case()
    p, metrics, moments = run_oracle_p2e(cfg, copy.deepcopy(fx["init"]),
                                         [{k: v.float() for k, v in d.items()} for d in fx["data"]], fx["noise"])
    for s, m in enumerate(fx["metrics"]):
        check_metrics(metrics[s], m, f"step{s}")
    for name, want in fx["after"].items():
        assert_params_close(p[name], want, LR.get(name, 8e-5), len(fx["data"]), label=name)
    check_moments(moments, fx["moments"])


def test_p2e_engine_matches_the_executed_reference():
    fx, cfg = p2e_case()
    eng = p2e_engine(fx, cfg)
    assert eng.minedojo
    for s in range(len(fx["data"])):
        eng.train_step({k: v.clone().float() for k, v in fx["data"][s].items()}, without_action_noise(fx["noise"][s]))
        check_metrics({k: v for k, v in eng.metrics_dict().items()}, fx["metrics"][s], f"engine step{s}")
    got = {name: dict(g.state_dict()) for name, g in eng.groups().items()}
    got["ens"] = dict(eng.ensembles_state_dict())
    for name, want in fx["after"].items():
        assert_params_close(got[name], want, LR.get(name, 8e-5), len(fx["data"]), label=name)
    check_moments({"task": eng.moments_state, **{k: c["moments_state"] for k, c in eng.critics_expl.items()}},
                  fx["moments"])


def test_no_action_noise_is_drawn_for_imagination():
    """the Philox action streams are not filled: the rollouts take the mode of every head"""
    fx, cfg, fdata = dv3_case()
    eng = dv3_engine(fx, cfg)
    calls = []
    orig = eng.ops.fill_exponential
    eng.ops.fill_exponential = lambda out, seed, stream, t: (calls.append(stream), orig(out, seed, stream, t))
    eng.train_step({k: v.clone() for k, v in fdata[0].items()})
    assert calls == [0, 1]
    fx, cfg = p2e_case()
    eng = p2e_engine(fx, cfg)
    calls.clear()
    orig = eng.ops.fill_exponential
    eng.ops.fill_exponential = lambda out, seed, stream, t: (calls.append(stream), orig(out, seed, stream, t))
    eng.train_step({k: v.clone().float() for k, v in fx["data"][0].items()})
    assert calls == [0, 1, 3]


def test_state_dicts_load_both_ways():
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent

    fx, cfg, _ = dv3_case()
    wm, actor, critic, target, player = build_agent(Fab, ACTIONS_DIM, False, cfg, obs_space_of(cfg), ops=MinedojoEmulOps())
    for mod, n in ((wm, "wm"), (actor, "actor"), (critic, "critic"), (target, "target")):
        assert {k: tuple(v.shape) for k, v in mod.state_dict().items()} == \
            {k: tuple(v.shape) for k, v in fx["init"][n].items()}, n
        mod.load_state_dict(fx["init"][n])
        assert all(torch.equal(v, fx["init"][n][k]) for k, v in mod.state_dict().items()), n
    assert player.eng.minedojo


# ------------------------------------------------------------------ refusals
@pytest.mark.parametrize("actions_dim, cont", [((19, 40), False), ((18, 40, 72), False), ((19, 40, 72, 3), False),
                                               ((4,), False), ((3,), True)])
def test_other_action_layouts_are_refused(actions_dim, cont):
    cfg = make_dv3_cfg(**dict(size="S", per_rank_batch_size=2, per_rank_sequence_length=4, horizon=4, dense_units=32,
                              mlp_layers=2, recurrent_state_size=24, hidden_size=24, stochastic_size=6, discrete_size=5,
                              bins=31, algo__actor__cls=DV3_ACTOR))
    with pytest.raises(NotImplementedError, match="MineDojo"):
        DV3Engine(cfg, actions_dim, device="cpu", ops=MinedojoEmulOps(), is_continuous=cont)


def test_a_backend_without_the_masked_sample_is_refused():
    from oracle.ops_emul import EmulOps

    fx, cfg, _ = dv3_case()
    with pytest.raises(NotImplementedError, match="masked sample"):
        DV3Engine(cfg, ACTIONS_DIM, device="cpu", ops=EmulOps())


def test_p2e_alias_is_accepted():
    fx, cfg = p2e_case()
    assert str(cfg.algo.actor.cls).endswith("p2e_dv3.agent.MinedojoActor") and p2e_engine(fx, cfg).minedojo


# ------------------------------------------------------------------ acting: masks
def hand_masks(E, g):
    """masks whose rows exercise every branch: functional actions 15 / 16 / 17 / 18 forced by mask_action_type, and
    rows where another action is the only one allowed"""
    K0, K1, K2 = ACTIONS_DIM
    m = {"mask_action_type": torch.zeros(E, K0, dtype=torch.bool),
         "mask_craft_smelt": torch.rand(E, K1, generator=g) < 0.3, "mask_equip_place": torch.rand(E, K2, generator=g) < 0.2,
         "mask_destroy": torch.rand(E, K2, generator=g) < 0.2}
    forced = [15, 16, 17, 18, 3, 15, 18, 0]
    for e in range(E):
        m["mask_action_type"][e, forced[e % len(forced)]] = True
        m["mask_craft_smelt"][e, e % K1] = True
        m["mask_equip_place"][e, e % K2] = m["mask_destroy"][e, (3 * e) % K2] = True
    return m


def reference_actor(actor_sd, cfg):
    """the reference MinedojoActor with the fixture's actor weights"""
    ref_harness.install()
    from sheeprl.algos.dreamer_v3.agent import MinedojoActor

    a, w = cfg.algo, cfg.algo.world_model
    actor = MinedojoActor(w.stochastic_size * w.discrete_size + w.recurrent_model.recurrent_state_size, ACTIONS_DIM, False,
                          {"type": "auto"}, dense_units=a.dense_units, mlp_layers=a.mlp_layers, activation=torch.nn.SiLU,
                          layer_norm_kw={"eps": a.mlp_layer_norm.kw.eps}, unimix=a.unimix)
    actor.load_state_dict(actor_sd)
    return actor


@needs_reference
def test_spec_masked_probs_and_mode_equal_the_reference_minedojo_actor():
    fx, cfg, _ = dv3_case()
    actor = reference_actor(fx["init"]["actor"], cfg)
    g = torch.Generator().manual_seed(3)
    E = 16
    state = torch.randn(1, E, actor.model._model[0].in_features, generator=g) * 2
    masks = hand_masks(E, g)
    with torch.no_grad():
        acts, dists = actor(state, True, {k: v.unsqueeze(0).clone() for k, v in masks.items()})
        raw = torch.cat([h(actor.model(state)) for h in actor.mlp_heads], -1)[0]
    hot, probs = minedojo_sample_spec(raw, None, cfg.algo.unimix, ACTIONS_DIM,
                                      [masks[k].float() for k in MASK_KEYS])
    assert torch.equal(hot, torch.cat(acts, -1)[0])
    for p, d in zip(probs, dists):
        assert torch.allclose(p, d.probs[0], rtol=1e-6, atol=1e-7)
    a0 = torch.cat(acts, -1)[0, :, :19].argmax(-1)
    assert {15, 16, 17, 18} <= set(a0.tolist()) and len(set(a0.tolist()) - {15, 16, 17, 18}) > 0


def player_of(cfg, E, ops=None):
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent

    cfg = copy.deepcopy(cfg)
    cfg.env.num_envs = E
    *_, player = build_agent(Fab, ACTIONS_DIM, False, cfg, obs_space_of(cfg), ops=ops or MinedojoEmulOps())
    return player


def obs_of(cfg, E, g, masks):
    obs = {"rgb": torch.rand(1, E, 3, 64, 64, generator=g) - 0.5}
    obs.update({k: v.unsqueeze(0).float() for k, v in masks.items()})
    return obs


@needs_reference
def test_player_masked_mode_equals_the_reference():
    """PlayerDV3 with the fixture's weights against the reference MinedojoActor(greedy=True, mask) on the player's own
    latent state"""
    fx, cfg, _ = dv3_case()
    E = 8
    player = player_of(cfg, E)
    for n in ("wm", "actor", "critic", "target"):
        getattr(player.trainer, n).load(fx["init"][n])
    actor = reference_actor(fx["init"]["actor"], cfg)
    g = torch.Generator().manual_seed(4)
    player.init_states()
    for step in range(3):
        masks = hand_masks(E, g)
        obs = obs_of(cfg, E, g, masks)
        got = player.get_actions(obs, True, {k: v.unsqueeze(0) for k, v in masks.items()})
        with torch.no_grad():
            want, _ = actor(player.eng.latent.view(1, E, -1).clone(), True, {k: v.unsqueeze(0).clone() for k, v in masks.items()})
        for x, y in zip(got, want):
            assert torch.equal(x, y), step


def test_player_sample_respects_the_masks_and_the_chain():
    fx, cfg, _ = dv3_case()
    E = 64
    player = player_of(cfg, E)
    g = torch.Generator().manual_seed(5)
    player.init_states()
    masks = hand_masks(E, g)
    a0, a1, a2 = player.get_actions(obs_of(cfg, E, g, masks), False, {k: v.unsqueeze(0) for k, v in masks.items()})
    f = a0[0].argmax(-1)
    assert bool(masks["mask_action_type"][torch.arange(E), f].all())
    c, i = a1[0].argmax(-1), a2[0].argmax(-1)
    for e in range(E):
        if f[e] == 15:
            assert masks["mask_craft_smelt"][e, c[e]]
        if f[e] in (16, 17):
            assert masks["mask_equip_place"][e, i[e]]
        if f[e] == 18:
            assert masks["mask_destroy"][e, i[e]]


def test_player_mask_errors_and_deviations():
    fx, cfg, _ = dv3_case()
    E = 2
    player = player_of(cfg, E)
    g = torch.Generator().manual_seed(6)
    player.init_states()
    masks = hand_masks(E, g)
    obs = obs_of(cfg, E, g, masks)
    full = {k: v.unsqueeze(0) for k, v in masks.items()}
    with pytest.raises(KeyError):
        player.get_actions(obs, False, {k: v for k, v in full.items() if k != "mask_destroy"})
    with pytest.raises(ValueError, match="mask_craft_smelt"):
        player.get_actions(obs, False, dict(full, mask_craft_smelt=torch.ones(1, E, 41, dtype=torch.bool)))
    # an empty dict acts unmasked (the reference's MinedojoActor raises KeyError on it): the same as no mask
    noise = {"z": torch.ones(E, player.eng.Z), "a": torch.rand(E, player.eng.A, generator=g) + 0.5}
    player.init_states()
    a = player.get_actions(obs, False, {}, noise=noise)
    player.init_states()
    b = player.get_actions(obs, False, None, noise=noise)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    # all-true masks: the unmasked sample
    player.init_states()
    c = player.get_actions(obs, False, {k: torch.ones_like(v) for k, v in full.items()}, noise=noise)
    assert all(torch.equal(x, y) for x, y in zip(a, c))


def test_all_masked_group_falls_back_to_the_unmasked_head():
    """a mask row that allows nothing: the head's unmasked distribution (the reference's logits would all be -inf)"""
    g = torch.Generator().manual_seed(7)
    M = 6
    raw = torch.randn(M, sum(ACTIONS_DIM), generator=g)
    q = torch.empty_like(raw).exponential_(generator=g)
    none = [torch.zeros(M, k) for k in (19, 40, 72, 72)]
    none[0][:, 15] = 1.0                                        # craft: head 1 sees an all-false craft mask
    hot, _ = minedojo_sample_spec(raw, q, 0.01, ACTIONS_DIM, none)
    free, _ = minedojo_sample_spec(raw, q, 0.01, ACTIONS_DIM, [None] * 4)
    assert torch.equal(hot[:, 19:], free[:, 19:]) and bool((hot[:, :19].argmax(-1) == 15).all())


def _recorder():
    spec = importlib.util.spec_from_file_location("trace_dense_ops", os.path.join(ROOT, "tools", "trace_dense_ops.py"))
    T = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(T)
    return T


def test_masked_acting_step_adds_one_op_after_the_head_products():
    """op trace of one acting step (ops calls and the torch ops issued outside them): masked = unmasked up to the three
    head products, then one minedojo_sample in place of the three cat_sample calls; neither copies to the host"""
    from oracle import ops_emul, ops_emul_minedojo

    T = _recorder()
    classes = (ops_emul.EmulOps, ops_emul_minedojo.MinedojoEmulOps)
    saved = {c: dict(vars(c)) for c in classes}
    fx, cfg, _ = dv3_case()
    E = 2
    g = torch.Generator().manual_seed(8)
    masks = hand_masks(E, g)
    obs = obs_of(cfg, E, g, masks)
    traces = {}
    try:
        for c in classes:
            T.wrap_ops(c)
        player = player_of(cfg, E)
        for name, mk in (("plain", None), ("masked", {k: v.unsqueeze(0) for k, v in masks.items()})):
            player.init_states()
            T.LINES.clear()
            with T.AtenRecorder():
                player.get_actions(obs, False, mk)
            traces[name] = list(T.LINES)
    finally:
        for c, d in saved.items():
            for k in list(vars(c)):
                if k not in d:
                    delattr(c, k)
            for k, v in d.items():
                if k not in ("__dict__", "__weakref__") and vars(c).get(k) is not v:
                    setattr(c, k, v)
    ops_only = {n: [x.split("(", 1)[0] for x in t if x.startswith("ops.")] for n, t in traces.items()}
    plain, masked = ops_only["plain"], ops_only["masked"]
    last_gemm = max(i for i, n in enumerate(plain) if n == "ops.gemm")
    assert plain[last_gemm + 1:] == ["ops.cat_sample"] * 3
    assert masked[:last_gemm + 1] == plain[:last_gemm + 1]
    assert masked[last_gemm + 1:] == ["ops.minedojo_sample"]
    for t in traces.values():
        assert not any(x.startswith(("aten._local_scalar_dense", "aten.item")) for x in t)     # no .item() / sync
    # the one torch op the masks add: each bool mask to float rows on the engine's device (a cast, not a copy home)
    extra = [x for x in traces["masked"] if x.startswith("aten.") and x not in traces["plain"]]
    assert len([x for x in extra if x.startswith("aten._to_copy")]) == 4 \
        and all("bool" in x and "float32" in x for x in extra if x.startswith("aten._to_copy"))


# ------------------------------------------------------------------ data plane: mask and equipment dtypes
def test_replay_buffers_round_trip_bool_masks_and_int32_equipment():
    from oracle.ops_emul import EmulOps
    from sheeprl_b200.data import buffers as Bf

    n_envs, T = 2, 6
    g = np.random.default_rng(0)
    steps = [{"mask_action_type": g.random((1, n_envs, 19)) < 0.5, "mask_destroy": g.random((1, n_envs, 72)) < 0.5,
              "equipment": g.integers(0, 2, (1, n_envs, 72)).astype(np.int32),
              "rewards": g.random((1, n_envs, 1)).astype(np.float32)} for _ in range(T)]
    for cls_name in ("SequentialReplayBuffer", "EnvIndependentReplayBuffer"):
        cls = getattr(Bf, cls_name, None)
        if cls is None:
            continue
        kw = {"buffer_cls": Bf.SequentialReplayBuffer} if cls_name == "EnvIndependentReplayBuffer" else {}
        rb = cls(16, n_envs, device="cpu", ops=EmulOps(), **kw)
        for s in steps:
            rb.add({k: v.copy() for k, v in s.items()})
        batch = rb.sample_tensors(2, sequence_length=3, n_samples=1)
        for k in ("mask_action_type", "mask_destroy", "equipment"):
            want = {"mask_action_type": torch.bool, "mask_destroy": torch.bool, "equipment": torch.int32}[k]
            assert batch[k].dtype == want, (cls_name, k, batch[k].dtype)
            stored = np.concatenate([s[k] for s in steps], 0)               # [T, n_envs, K]
            got = batch[k].reshape(-1, 3, batch[k].shape[-1]) if batch[k].dim() == 4 else batch[k]
            rows = {tuple(r) for r in stored.reshape(-1, stored.shape[-1]).astype(np.int64).tolist()}
            assert all(tuple(r) in rows for r in got.reshape(-1, got.shape[-1]).long().tolist()), (cls_name, k)


# ------------------------------------------------------------------ the reference's own main
class MinedojoLikeEnv:
    """64x64x3 uint8 pixels, the four bool action masks and an int32 `equipment` vector, MultiDiscrete([19, 40, 72])
    actions: the observation and action layout of sheeprl/envs/minedojo.py at synthetic item counts"""

    def __init__(self, seed=0, length=10):
        from tests import fake_gym

        K0, K1, K2 = ACTIONS_DIM
        obs = {"rgb": fake_gym.Box(0, 255, (3, 64, 64), np.uint8), "equipment": fake_gym.Box(0, 1, (K2,), np.int32)}
        obs.update({k: fake_gym.Box(0, 1, (d,), bool) for k, d in MASKS.items()})
        self.observation_space = fake_gym.Dict(obs)
        self.action_space = fake_gym.MultiDiscrete(np.array(ACTIONS_DIM))
        self.rng, self.length, self.t = np.random.default_rng(seed), length, 0
        self.actions = []

    def _obs(self):
        o = {"rgb": self.rng.integers(0, 256, (3, 64, 64), dtype=np.uint8),
             "equipment": self.rng.integers(0, 2, ACTIONS_DIM[2]).astype(np.int32)}
        for k, d in MASKS.items():
            m = self.rng.random(d) < 0.3
            m[self.rng.integers(d)] = True
            o[k] = m
        o["mask_action_type"][15:19] = True
        self.last = o
        return o

    def reset(self, seed=None, options=None):
        self.t = 0
        return self._obs(), {}

    def step(self, action):
        a = np.asarray(action).reshape(-1)
        self.actions.append((a.copy(), {k: v.copy() for k, v in self.last.items() if k.startswith("mask")}))
        self.t += 1
        return self._obs(), float(self.rng.normal()), self.t >= self.length, False, {}

    def close(self):
        pass


@needs_reference
def test_reference_main_runs_with_the_minedojo_actor_and_run_test(tmp_path):
    """the reference's own `main` on a 2-environment MultiDiscrete environment with mask keys, the MineDojo actor and
    `run_test: True`: every action the player takes honours the masks of the observation it acted on"""
    import sheeprl_b200.algos.dreamer_v3.agent as A
    import sheeprl_b200.algos.dreamer_v3.dreamer_v3 as B
    from sheeprl_b200.data import buffers as Bf
    from tests.test_main_delegation_cpu import Fabric, _harness, _loop_cfg

    R = _harness(tmp_path)
    import sheeprl.algos.dreamer_v3.utils as RU

    envs = []

    def env_fn(cfg, seed, rank_off, log_dir, prefix, vector_env_idx=0):
        def make():
            envs.append(MinedojoLikeEnv(seed=seed))
            return envs[-1]
        return make

    orig_make_env, R.make_env, RU.make_env = RU.make_env, env_fn, env_fn
    os.makedirs(tmp_path / "run" / "checkpoint", exist_ok=True)
    cfg, fab = _loop_cfg(tmp_path, run_test=True), Fabric(tmp_path)
    cfg.env.num_envs = 2
    keys = list(MASKS) + ["equipment"]
    cfg.algo.mlp_keys.encoder, cfg.algo.mlp_keys.decoder = keys, keys
    cfg.algo.actor.cls = DV3_ACTOR
    # a MineDojo wrapper target: main() then acts through the player from the first step (dreamer_v3.py:560-564)
    cfg.env.wrapper._target_ = "tests.test_minedojo_cpu.MinedojoLikeEnv"
    engines, players, orig_train, orig_test = [], [], B.train, R.test

    def counting_train(*a, **k):
        engines.append(a[1]._b200_engine)
        return orig_train(*a, **k)

    def recording_test(player, *a, **k):
        players.append(player)
        return orig_test(player, *a, **k)

    A.DEFAULT_OPS, Bf.DEFAULTS["ops"] = MinedojoEmulOps(), MinedojoEmulOps()
    B.train, R.test = counting_train, recording_test
    try:
        B.main(fab, cfg)
    finally:
        B.train, R.test, RU.make_env = orig_train, orig_test, orig_make_env
        A.DEFAULT_OPS, Bf.DEFAULTS["ops"], Bf.DEFAULTS["device"] = None, None, "cuda"
    assert len(engines) >= 3 and engines[0].minedojo and engines[0].actions_dim == ACTIONS_DIM
    assert len(players) == 1 and players[0].num_envs == 1
    acted = [x for e in envs for x in e.actions]
    assert len(acted) > 40
    for a, m in acted:
        f, c, i = int(a[0]), int(a[1]), int(a[2])
        assert m["mask_action_type"][f]
        if f == 15:
            assert m["mask_craft_smelt"][c]
        if f in (16, 17):
            assert m["mask_equip_place"][i]
        if f == 18:
            assert m["mask_destroy"][i]
    (ck,) = fab.checkpoints
    assert all(torch.isfinite(v).all() for v in ck["state"]["world_model"].values())
