"""Recurrent PPO against the executing reference (where its checkout is available):

  * the registered `ppo_recurrent` entry point drives the UNMODIFIED reference interaction loop
    (ppo_recurrent.py:119-524) with this package's build_agent / train / optimizer handle substituted, on a fake vector
    env whose episodes end inside the rollout (so the sequences are padded), writes checkpoints in the reference's
    layout and resumes from one;
  * continuous actions: the reference's own train() and player fail (RecurrentPPOAgent._get_actions passes a tuple /
    None to Normal.log_prob), which is why build_agent refuses them.
Kernels are the torch test double."""
import os

import pytest
import torch

from oracle import ref_harness
from oracle.ops_emul_recurrent import RecurrentEmulOps as EmulOps
from sheeprl_b200.utils.utils import dotdict
from tests import fake_gym

pytestmark = pytest.mark.skipif(not ref_harness.reference_available(), reason="reference tree not present")


class Fabric(ref_harness.FakeFabric):
    def __init__(self):
        super().__init__("cpu")
        self.logged, self.checkpoints, self.loggers = {}, [], []

    def load(self, path):
        return torch.load(path, weights_only=False)

    def log_dict(self, d, step):
        self.logged.update(d)

    def log(self, k, v, step):
        self.logged[k] = v

    def call(self, hook, **kw):
        assert hook == "on_checkpoint_coupled"
        self.checkpoints.append(kw)
        os.makedirs(os.path.dirname(kw["ckpt_path"]), exist_ok=True)
        torch.save(kw["state"], kw["ckpt_path"])


def _cfg(tmp, total_steps=64, resume=None):
    from oracle.make_golden_ppo_recurrent import rec_cfg

    spec = dict(cnn_channels=0, screen=64, mlp_dim=3, dense=16, layers=1, layer_norm=True, cnn_features=8,
                mlp_features=8, actions_dim=(2,), is_continuous=False, act="relu",
                rnn=dict(hidden=16, pre=None, post=None))
    hp = dict(clip_coef=0.2, vf_coef=0.2, ent_coef=0.001, clip_vloss=False, normalize_advantages=True,
              max_grad_norm=0.5)
    cfg = rec_cfg(spec, hp, batches=2, epochs=2, num_envs=2)
    cfg.algo.update(dict(name="ppo_recurrent", total_steps=total_steps, rollout_steps=16, per_rank_sequence_length=8,
                         per_rank_batch_size=4, anneal_lr=False, anneal_clip_coef=False, anneal_ent_coef=True,
                         gamma=0.99, gae_lambda=0.95, reset_recurrent_state_on_done=True, run_test=False))
    cfg.update(dict(seed=3, dry_run=False, root_dir=str(tmp), run_name="run"))
    cfg.checkpoint = {"resume_from": resume, "every": 32, "save_last": True, "keep_last": 5}
    cfg.metric = {"log_level": 0, "log_every": 32, "sync_on_compute": False, "aggregator": {}}
    cfg.model_manager = {"disabled": True}
    cfg.buffer = {"size": 16, "memmap": False, "checkpoint": False, "validate_args": False, "from_numpy": False,
                  "share_data": False}
    cfg.env.update({"sync_env": True, "action_repeat": 1, "wrapper": {"_target_": "tests.fake_gym.DummyImageEnv"}})
    return dotdict(_plain(cfg))


def _plain(d):
    return {k: _plain(v) for k, v in d.items()} if isinstance(d, dict) else d


def _harness():
    ref_harness.install()
    import sheeprl.algos.ppo_recurrent.ppo_recurrent as R
    from sheeprl.utils.metric import MetricAggregator
    from sheeprl.utils.timer import timer

    R.gym = fake_gym.module()
    R.make_env = lambda cfg, seed, rank_off, log_dir, prefix, vector_env_idx=0: (
        lambda: fake_gym.DummyImageEnv(size=8, length=11, seed=seed, vector_dim=3))
    R.get_logger = lambda fabric, cfg: None
    R.get_log_dir = lambda fabric, root, run: os.path.join(root, run)
    R.save_configs = lambda cfg, log_dir: None
    MetricAggregator.disabled = True
    timer.disabled = True
    return R


def test_registered_main_runs_the_reference_loop_and_resumes(tmp_path, monkeypatch):
    R = _harness()
    import sheeprl_b200.algos.ppo_recurrent.agent as A
    import sheeprl_b200.algos.ppo_recurrent.ppo_recurrent as B
    from sheeprl_b200.utils.registry import find_algorithm

    found = find_algorithm("ppo_recurrent")
    assert found is not None and found[0] == "sheeprl_b200.algos.ppo_recurrent" and found[1]["entrypoint"] == "main"
    real_build = A.build_agent
    monkeypatch.setattr(A, "build_agent", lambda *a, **k: real_build(*a, ops=EmulOps(), **k))
    seen = {"train": 0, "padded": 0, "engines": []}
    orig_train = B.train

    def counting_train(fabric, agent, optimizer, data, aggregator, cfg, **k):
        seen["train"] += 1
        seen["padded"] += int((~data["mask"]).sum())
        seen["engines"].append(agent._b200_engine)
        return orig_train(fabric, agent, optimizer, data, aggregator, cfg, **k)

    monkeypatch.setattr(B, "train", counting_train)
    ref_train, ref_build = R.train, R.build_agent
    fab = Fabric()
    B.main(fab, _cfg(tmp_path))
    assert R.train is ref_train and R.build_agent is ref_build          # the reference module is left as it was
    assert seen["train"] == 2 and seen["padded"] > 0                     # two iterations, padded sequences
    eng = seen["engines"][0]
    n_mb = eng.group.step
    assert n_mb >= 2 * 2 * 2
    ck = fab.checkpoints[-1]["state"]
    assert set(ck) >= {"agent", "optimizer", "iter_num", "batch_size", "last_log", "last_checkpoint"}
    assert "rnn._lstm.weight_hh_l0" in ck["agent"] and "actor.actor_heads.0.weight" in ck["agent"]
    assert len(ck["optimizer"]["state"]) == len(eng.group.shapes) and int(ck["optimizer"]["state"][0]["step"]) == n_mb
    assert all(torch.isfinite(v).all() for v in ck["agent"].values())
    assert fab.logged["Info/ent_coef"] < 0.001                           # annealed between iterations
    # resume from the last checkpoint: parameters and Adam moments go back into the flat group, the step continues
    path = fab.checkpoints[-1]["ckpt_path"]
    fab2 = Fabric()
    B.main(fab2, _cfg(tmp_path, total_steps=96, resume=path))
    eng2 = seen["engines"][-1]
    assert eng2 is not eng and seen["train"] == 3
    st2 = fab2.checkpoints[-1]["state"]
    assert int(st2["optimizer"]["state"][0]["step"]) > n_mb and st2["iter_num"] > ck["iter_num"]


def _continuous_reference(tmp_path):
    ref_harness.install()
    import sheeprl.algos.ppo_recurrent.agent as A

    from oracle.make_golden_ppo import obs_space

    A.get_single_device_fabric = lambda f: f
    spec = dict(cnn_channels=0, screen=0, mlp_dim=3, dense=16, layers=1, layer_norm=False, cnn_features=8,
                mlp_features=8, actions_dim=(2,), is_continuous=True, act="tanh", rnn=dict(hidden=8, pre=None, post=None))
    from oracle.make_golden_ppo_recurrent import rec_cfg

    cfg = rec_cfg(spec, dict(clip_coef=0.2, vf_coef=0.5, ent_coef=0.0, clip_vloss=False, normalize_advantages=False,
                             max_grad_norm=0.0), batches=1, epochs=1, num_envs=2)
    agent, player = A.build_agent(ref_harness.FakeFabric(), (2,), True, cfg, obs_space(spec), None)
    return spec, cfg, agent, player


def test_reference_fails_with_continuous_actions(tmp_path):
    import sheeprl.algos.ppo_recurrent.ppo_recurrent as P

    spec, cfg, agent, player = _continuous_reference(tmp_path)
    T, S = 3, 2
    data = {"state": torch.randn(T, S, 3), "actions": torch.randn(T, S, 2), "prev_actions": torch.zeros(T, S, 2),
            "logprobs": torch.zeros(T, S, 1), "values": torch.zeros(T, S, 1), "returns": torch.zeros(T, S, 1),
            "advantages": torch.randn(T, S, 1), "prev_hx": torch.zeros(T, S, 8), "prev_cx": torch.zeros(T, S, 8),
            "mask": torch.ones(T, S, dtype=torch.bool)}
    opt = torch.optim.Adam(agent.parameters(), lr=1e-3)
    with pytest.raises((ValueError, TypeError, AttributeError, RuntimeError)):
        P.train(ref_harness.FakeFabric(), agent, opt, data, None, cfg)
    with pytest.raises((ValueError, TypeError, AttributeError, RuntimeError)), torch.no_grad():
        player({"state": torch.randn(1, S, 3)}, prev_actions=torch.zeros(1, S, 2),
               prev_states=(torch.zeros(1, S, 8), torch.zeros(1, S, 8)))
    # ... and the engine refuses them up front
    from oracle.make_golden_ppo import obs_space
    from sheeprl_b200.algos.ppo_recurrent.agent import build_agent

    class Fab:
        device, world_size, global_rank = torch.device("cpu"), 1, 0

    with pytest.raises(NotImplementedError):
        build_agent(Fab, (2,), True, cfg, obs_space(spec), ops=EmulOps())


def test_reference_train_raises_on_padding_with_validation_on():
    """the deviation DESIGN.md records: with torch's default distribution argument validation the reference's train()
    rejects the all-zero action rows of padded steps; the fixtures and this engine follow it with validation off"""
    ref_harness.install()
    import sheeprl.algos.ppo_recurrent.agent as A
    import sheeprl.algos.ppo_recurrent.ppo_recurrent as P

    from oracle import ppo_recurrent_oracle as RO
    from oracle.make_golden_ppo import obs_space
    from oracle.make_golden_ppo_recurrent import FIXTURES, rec_cfg

    A.get_single_device_fabric = lambda f: f
    fx = FIXTURES["ppo_rec_vector"]
    cfg = rec_cfg(fx["spec"], fx["hp"], fx["batches"], 1)
    agent, _ = A.build_agent(ref_harness.FakeFabric(), fx["spec"]["actions_dim"], False, cfg, obs_space(fx["spec"]), None)
    data = RO.make_rollout(fx["spec"], fx["T"], fx["lengths"], 0)
    prev = torch.distributions.Distribution._validate_args
    torch.distributions.Distribution.set_default_validate_args(True)
    try:
        with pytest.raises(ValueError):
            P.train(ref_harness.FakeFabric(), agent, torch.optim.Adam(agent.parameters()), data, None, cfg)
    finally:
        torch.distributions.Distribution.set_default_validate_args(prev)
