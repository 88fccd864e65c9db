"""Recurrent PPO on a GPU-less host: the oracle against the executed reference (tests/golden/ppo_rec_*.pt), and the
engine's kernel schedule (hand-derived backward through the LSTM) against the same fixtures with the torch test double
in place of the CUDA ops; the player, the public surface and its refusals."""
import os

import pytest
import torch

from oracle import ppo_recurrent_oracle as RO
from oracle.dv3_oracle import AdamState
from tests.test_ppo_cpu import assert_params_close

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ["ppo_rec_vector", "ppo_rec_branches", "ppo_rec_pixel"]
LOSS_KEYS = ("Loss/policy_loss", "Loss/value_loss", "Loss/entropy_loss")


def load(name):
    """a fixture with its initial parameters regenerated from the stored seed and the parameters after train()
    rebuilt from the stored fp16 update (oracle/make_golden_ppo_recurrent.py)"""
    fx = torch.load(os.path.join(GOLDEN, f"{name}.pt"), weights_only=False)
    fx["init"] = RO.init_params(fx["spec"], fx["init_seed"])
    fx["after"] = RO.unpack_after(fx["init"], fx["after_delta"])
    if "rgb" in fx["data"]:
        fx["data"]["rgb"] = fx["data"]["rgb"].float()
    return fx


class Fab:
    device, world_size, global_rank = torch.device("cpu"), 1, 0


def test_fixtures_have_padding_with_lengths_one_and_T():
    for name in NAMES:
        mask = load(name)["data"]["mask"]
        lengths = mask.sum(0)
        assert int(lengths.min()) == 1 and int(lengths.max()) == mask.shape[0], name


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    fx = load(name)
    p = {k: v.clone() for k, v in fx["init"].items()}
    assert {k: tuple(v.shape) for k, v in p.items()} == RO.param_shapes(fx["spec"])
    logs = RO.train(p, AdamState(p, 1e-3, 1e-4), fx["spec"], fx["data"], fx["index_batches"], fx["hp"])
    for got, want in zip(logs, fx["losses"]):
        for k, v in want.items():
            assert abs(got[k] - v) <= 1e-4 * max(1.0, abs(v)), (k, got[k], v)
    assert_params_close(p, fx["after"], name, steps=len(logs))


# ---------------------------------------------------------------------------------------------------------
# engine schedule with the torch test double
# ---------------------------------------------------------------------------------------------------------
def make_engine(fx, device="cpu", ops=None):
    from oracle.ops_emul_recurrent import RecurrentEmulOps as EmulOps
    from sheeprl_b200.algos.ppo_recurrent.engine import RecurrentPPOEngine

    eng = RecurrentPPOEngine(fx["spec"], fx["hp"], {"lr": 1e-3, "eps": 1e-4, "betas": (0.9, 0.999)}, device,
                             ops or EmulOps())
    assert dict(eng.reference_shapes()) == RO.param_shapes(fx["spec"])
    eng.load_reference_state(fx["init"])
    return eng


def check_engine(fx, eng, name, uint8_image=False):
    dev = eng.device
    data = {k: v.to(dev) for k, v in fx["data"].items()}
    if uint8_image and "rgb" in data:
        data["rgb"] = data["rgb"].to(torch.uint8)
    logs = []
    eng.train(data, fx["index_batches"], lambda l: logs.append(l.cpu()))
    assert len(logs) == len(fx["losses"])
    for got, want in zip(logs, fx["losses"]):
        for i, k in enumerate(LOSS_KEYS):
            assert abs(float(got[i]) - want[k]) <= 1e-4 * max(1.0, abs(want[k])), (name, k, float(got[i]), want[k])
    assert_params_close(eng.export_reference_state(), fx["after"], name, steps=len(logs))


@pytest.mark.parametrize("name", NAMES)
def test_engine_schedule_matches_reference(name):
    fx = load(name)
    check_engine(fx, make_engine(fx), name)


def test_engine_refuses_a_mask_that_is_not_a_prefix():
    fx = load("ppo_rec_vector")
    eng = make_engine(fx)
    data = {k: v.clone() for k, v in fx["data"].items()}
    data["mask"][0, 2] = False                 # a hole before valid steps
    with pytest.raises(ValueError, match="prefix"):
        eng.train(data, fx["index_batches"])


def test_ops_emul_masked_loss_single_row_skips_normalisation():
    from oracle.ops_emul_recurrent import RecurrentEmulOps as EmulOps

    em = EmulOps()
    B, dims = 6, [3]
    g = torch.Generator().manual_seed(0)
    head = torch.randn(B, 3, generator=g)
    acts = torch.nn.functional.one_hot(torch.randint(0, 3, (B,), generator=g), 3).float()
    cols = [torch.randn(B, generator=g) for _ in range(5)]
    mask = torch.zeros(B)
    mask[4] = 1
    dh, dv, losses = torch.zeros(B, 3), torch.zeros(B), torch.zeros(3)
    em.ppo_loss_masked(head, acts, *cols, mask, dh, dv, losses, dims, 0, True, True, 0.2, 0.5, 0.01)
    dh1, dv1, l1 = torch.zeros(1, 3), torch.zeros(1), torch.zeros(3)
    em.ppo_loss(head[4:5], acts[4:5], *(c[4:5] for c in cols), dh1, dv1, l1, dims, 0, True, False, 0.2, 0.5, 0.01)
    assert torch.equal(losses, l1) and torch.equal(dh[4:5], dh1) and float(dh[:4].abs().sum()) == 0.0


# ---------------------------------------------------------------------------------------------------------
# public surface
# ---------------------------------------------------------------------------------------------------------
def _cfg(fx, num_envs=1):
    from oracle.make_golden_ppo_recurrent import rec_cfg

    return rec_cfg(fx["spec"], fx["hp"], fx["batches"], fx["epochs"], num_envs=num_envs)


def _build(fx, cfg=None, fab=Fab, state="init", continuous=False):
    from oracle.make_golden_ppo import obs_space
    from oracle.ops_emul_recurrent import RecurrentEmulOps as EmulOps
    from sheeprl_b200.algos.ppo_recurrent.agent import build_agent

    return build_agent(fab, fx["spec"]["actions_dim"], continuous, cfg or _cfg(fx), obs_space(fx["spec"]),
                       agent_state=fx[state] if state else None, ops=EmulOps())


@pytest.mark.parametrize("name", NAMES)
def test_public_api_draws_the_reference_minibatches(name):
    """train() without explicit indices draws the reference's RandomSampler/BatchSampler stream: under the fixture's
    sampler seed it visits the recorded sequence batches and lands on the reference's parameters."""
    from sheeprl_b200.algos.ppo_recurrent.ppo_recurrent import make_optimizer, train

    fx = load(name)
    cfg = _cfg(fx)
    agent, _ = _build(fx, cfg)
    opt = make_optimizer(agent, cfg)

    class Agg:
        disabled, rows = False, []

        def update(self, k, v):
            self.rows.append((k, float(v)))

    agg = Agg()
    torch.manual_seed(fx["sampler_seed"])
    train(Fab, agent, opt, {k: v.clone() for k, v in fx["data"].items()}, agg, cfg)
    assert len(agg.rows) == 3 * len(fx["losses"])
    assert [k for k, _ in agg.rows[:3]] == list(LOSS_KEYS)
    assert abs(agg.rows[-1][1] - fx["losses"][-1]["Loss/entropy_loss"]) < 1e-4
    assert_params_close(agent.state_dict(), fx["after"], "public", steps=len(fx["losses"]))
    assert opt.state_dict()["state"][0]["step"] == len(fx["losses"])


def test_build_agent_keys_shapes_and_round_trip():
    fx = load("ppo_rec_branches")
    agent, player = _build(fx, state=None)
    sd = agent.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in fx["init"].items()}
    agent.load_state_dict(fx["init"])
    for k, v in agent.state_dict().items():
        assert torch.equal(v, fx["init"][k]), k
    assert agent.rnn_hidden_size == player.rnn_hidden_size == fx["spec"]["rnn"]["hidden"]
    hx, cx = agent.initial_states
    assert hx.shape == cx.shape == (1, 1, fx["spec"]["rnn"]["hidden"]) and not bool(hx.any())
    assert player.actor.is_continuous is False and player.eval() is player


def test_build_agent_refusals():
    fx = load("ppo_rec_vector")
    with pytest.raises(NotImplementedError, match="discrete"):
        _build(fx, continuous=True, state=None)

    class Fab2(Fab):
        world_size = 2

    with pytest.raises(NotImplementedError, match="Join"):
        _build(fx, fab=Fab2, state=None)
    cfg = _cfg(fx)
    cfg.algo.rnn.post_rnn_mlp.apply = True
    cfg.algo.rnn.post_rnn_mlp.dense_units = 32
    with pytest.raises(ValueError, match="hidden_size"):
        _build(fx, cfg=cfg, state=None)


@pytest.mark.parametrize("target,wd,ok", [("torch.optim.AdamW", 0, True), ("torch.optim.Adam", 0, True),
                                          ("torch.optim.AdamW", 0.01, False), ("torch.optim.Adam", 1e-4, False),
                                          ("torch.optim.AdamW", None, False), ("torch.optim.SGD", 0, False)])
def test_optimizer_factory(target, wd, ok):
    from sheeprl_b200.algos.ppo_recurrent.ppo_recurrent import _optimizer_factory

    fx = load("ppo_rec_vector")
    agent, _ = _build(fx)
    make = _optimizer_factory([agent])
    conf = {"_target_": target, "lr": 3e-4, "eps": 1e-5}
    if wd is not None:
        conf["weight_decay"] = wd
    if ok:
        opt = make(conf, list(agent.parameters()))
        assert opt.lr == pytest.approx(3e-4)
    else:
        with pytest.raises(NotImplementedError):
            make(conf, list(agent.parameters()))


# ---------------------------------------------------------------------------------------------------------
# RecurrentPPOPlayer against the executed reference player (tests/golden/ppo_rec_player.pt)
# ---------------------------------------------------------------------------------------------------------
def _close(got, want, rtol=1e-4, what=""):
    got = got.detach().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert float((got - want).abs().max()) <= rtol * max(1.0, float(want.abs().max())), (what, float((got - want).abs().max()))


def check_player(name, device="cpu", ops=None):
    from sheeprl_b200.algos.ppo_recurrent.agent import RecurrentPPOPlayer

    rec = torch.load(os.path.join(GOLDEN, "ppo_rec_player.pt"), weights_only=False)[name]
    fx = load(name)
    eng = make_engine(fx, device=device, ops=ops)
    E = rec["init_prev"].shape[1]
    player = RecurrentPPOPlayer(eng, num_envs=E)
    to = lambda x: x.to(device)  # noqa: E731
    states, prev = tuple(to(s) for s in rec["init_states"]), to(rec["init_prev"])
    for i, st in enumerate(rec["steps"]):
        obs = {k: to(v) for k, v in RO.player_obs(st["obs"]).items()}
        given, keep = states, tuple(s.clone() for s in states)
        actions, logp, values, states = player(obs, prev_actions=prev, prev_states=states, noise=to(st["noise"]))
        for got, want in zip(actions, st["actions"]):
            assert torch.equal(got.cpu(), want), (name, i)
        _close(logp, st["logp"], what="logp")
        _close(values, st["values"], what="values")
        for got, want in zip(states, st["states"]):
            _close(got, want, what="states")
        assert all(torch.equal(a, b) for a, b in zip(given, keep))          # the caller's states are left as they were
        prev = torch.cat(actions, -1)
    first = tuple(s.clone() for s in states)
    sub = rec["sub"]
    obs = {k: to(v) for k, v in RO.player_obs(rec["steps"][-1]["obs"]).items()}
    vals, st2 = player.get_values({k: v[:, sub] for k, v in obs.items()}, prev[:, sub], tuple(s[:, sub] for s in states))
    _close(vals, rec["sub_values"], what="get_values")
    for got, want in zip(st2, rec["sub_states"]):
        _close(got, want, what="sub states")
    greedy, st3 = player.get_actions(obs, prev, states, greedy=True)
    for got, want in zip(greedy, rec["greedy"]):
        assert torch.equal(got.cpu(), want)
    for got, want in zip(st3, rec["greedy_states"]):
        _close(got, want, what="greedy states")
    # the states a caller keeps are not overwritten by later calls
    for a, b in zip(states, first):
        assert torch.equal(a, b)


@pytest.mark.parametrize("name", NAMES)
def test_player_matches_reference(name):
    check_player(name)
