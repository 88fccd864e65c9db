"""A2C against the executing reference (where its checkout is available):

  * the registered `a2c` entry point drives the UNMODIFIED reference interaction loop (a2c.py:118-440) with this
    package's build_agent / train / RMSprop handle substituted, with `anneal_lr` (PolynomialLR on the handle), writes
    checkpoints in the reference's layout and resumes from one;
  * `sheeprl-eval`'s `evaluate_a2c` runs through the rebound build_agent.
Kernels are the torch test double."""
import os

import pytest
import torch

from oracle import ref_harness
from oracle.ops_emul_a2c import A2CEmulOps
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


def _cfg(tmp, total_steps=32, resume=None):
    from oracle.make_golden_a2c import HP, RMSPROP, a2c_cfg

    spec = dict(cnn_channels=0, screen=64, mlp_dim=3, dense=16, layers=2, cnn_features=8, mlp_features=8,
                actions_dim=(2,), is_continuous=False, act="tanh")
    cfg = a2c_cfg(spec, dict(HP, ent_coef=0.01), 5, dict(RMSPROP, momentum=0.5))
    cfg.algo.update(dict(total_steps=total_steps, rollout_steps=8, anneal_lr=True, gamma=0.99, gae_lambda=0.95,
                         run_test=False))
    cfg.update(dict(seed=3, dry_run=False, root_dir=str(tmp), run_name="run"))
    cfg.checkpoint = {"resume_from": resume, "every": 16, "save_last": True, "keep_last": 5}
    cfg.metric = {"log_level": 0, "log_every": 16, "sync_on_compute": False, "aggregator": {}}
    cfg.model_manager = {"disabled": True}
    cfg.buffer = {"size": 8, "memmap": False, "checkpoint": False, "validate_args": False, "from_numpy": False,
                  "share_data": False}
    cfg.env = {"num_envs": 2, "sync_env": True, "action_repeat": 1, "screen_size": 64,
               "wrapper": {"_target_": "tests.fake_gym.DummyImageEnv"}}
    return dotdict(_plain(cfg))


def _plain(d):
    return {k: _plain(v) for k, v in d.items()} if isinstance(d, dict) else d


def _env(cfg, seed, *a, **k):
    return lambda: fake_gym.DummyImageEnv(size=8, length=11, seed=seed or 0, vector_dim=3)


def _harness():
    ref_harness.install()
    import sheeprl.algos.a2c.a2c as R
    from sheeprl.utils.metric import MetricAggregator
    from sheeprl.utils.timer import timer

    R.gym = fake_gym.module()
    R.make_env = _env
    R.get_logger = lambda fabric, cfg: None
    R.get_log_dir = lambda fabric, root, run: os.path.join(root, run)
    R.save_configs = lambda cfg, log_dir: None
    MetricAggregator.disabled = True
    timer.disabled = True
    return R


def test_registered_main_runs_the_reference_loop_and_resumes(tmp_path, monkeypatch):
    R = _harness()
    import sheeprl_b200.algos.a2c.a2c as B
    import sheeprl_b200.algos.a2c.agent as A
    from sheeprl_b200.utils.registry import find_algorithm

    found = find_algorithm("a2c")
    assert found is not None and found[0] == "sheeprl_b200.algos.a2c" and found[1]["entrypoint"] == "main"
    real_build = A.build_agent
    monkeypatch.setattr(A, "build_agent", lambda *a, **k: real_build(*a, ops=A2CEmulOps(), **k))
    seen = {"train": 0, "rows": [], "lr": [], "engines": [], "opt": [], "state_in": []}
    orig_train = B.train

    def counting_train(fabric, agent, optimizer, data, aggregator, cfg, **k):
        seen["train"] += 1
        seen["rows"].append(int(data["actions"].shape[0]))
        seen["lr"].append(optimizer.param_groups[0]["lr"])
        seen["engines"].append(agent._b200_engine)
        seen["opt"].append(optimizer)
        seen["state_in"].append(optimizer.state_dict())
        return orig_train(fabric, agent, optimizer, data, aggregator, cfg, **k)

    monkeypatch.setattr(B, "train", counting_train)
    ref_train, ref_build = R.train, R.build_agent
    fab = Fabric()
    B.main(fab, _cfg(tmp_path))
    assert R.train is ref_train and R.build_agent is ref_build          # the reference module is left as it was
    assert seen["train"] == 2 and seen["rows"] == [16, 16]
    assert isinstance(seen["opt"][0], B.B200RMSprop)
    # PolynomialLR attaches to the handle; the reference's loop never steps it (a2c.py:258-264), so lr stays
    assert seen["lr"] == [1e-3, 1e-3]
    eng = seen["engines"][0]
    assert eng.group.step == 2                                           # one optimizer step per train() call
    ck = fab.checkpoints[-1]["state"]
    assert set(ck) >= {"agent", "optimizer", "scheduler", "iter_num", "batch_size", "last_log", "last_checkpoint"}
    assert ck["scheduler"]["base_lrs"] == [1e-3]
    sd = ck["optimizer"]
    assert len(sd["state"]) == len(ck["agent"]) and int(sd["state"][0]["step"]) == 2
    assert set(sd["state"][0]) == {"step", "square_avg", "momentum_buffer"}
    for i, (k, v) in enumerate(ck["agent"].items()):
        assert sd["state"][i]["square_avg"].shape == v.shape, k
    assert all(torch.isfinite(v).all() for v in ck["agent"].values())
    # resume from the last checkpoint: parameters, RMSprop state and the scheduler go back in, the step continues
    path = fab.checkpoints[-1]["ckpt_path"]
    fab2 = Fabric()
    B.main(fab2, _cfg(tmp_path, total_steps=48, resume=path))
    eng2 = seen["engines"][-1]
    assert eng2 is not eng and seen["train"] == 3
    st2 = fab2.checkpoints[-1]["state"]
    assert int(st2["optimizer"]["state"][0]["step"]) == 3 and st2["iter_num"] > ck["iter_num"]
    resumed = seen["state_in"][-1]                                       # what the resumed run started from
    for i in sd["state"]:
        for k in ("step", "square_avg", "momentum_buffer"):
            assert torch.equal(resumed["state"][i][k], sd["state"][i][k]), (i, k)


def test_evaluate_a2c_runs_through_the_rebound_build_agent(tmp_path, monkeypatch):
    ref_harness.install()
    import sheeprl.algos.a2c.evaluate as RE
    import sheeprl.algos.ppo.utils as PU

    import sheeprl_b200.algos.a2c.agent as A
    from sheeprl_b200.algos.a2c.evaluate import evaluate_a2c

    cfg = _cfg(tmp_path)
    cfg.dry_run = True
    monkeypatch.setattr(RE, "gym", fake_gym.module())
    monkeypatch.setattr(RE, "make_env", _env)
    monkeypatch.setattr(PU, "make_env", _env)
    monkeypatch.setattr(RE, "get_logger", lambda fabric, cfg: None)
    monkeypatch.setattr(RE, "get_log_dir", lambda fabric, root, run: os.path.join(root, run))
    built = []
    real_build = A.build_agent

    def build(*a, **k):
        out = real_build(*a, ops=A2CEmulOps(), **k)
        built.append(out)
        return out

    monkeypatch.setattr(A, "build_agent", build)
    from oracle import a2c_oracle as AO

    spec = dict(cnn_channels=0, screen=0, mlp_dim=3, dense=16, layers=2, cnn_features=8, mlp_features=8,
                actions_dim=(2,), is_continuous=False, act="tanh")
    state = {"agent": AO.init_params(spec, 5)}
    fab = Fabric()
    evaluate_a2c(fab, cfg, state)
    assert RE.build_agent is not build and len(built) == 1               # rebound only for the call
    agent, player = built[0]
    for k, v in agent.state_dict().items():
        assert torch.equal(v, state["agent"][k]), k
