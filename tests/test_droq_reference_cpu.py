"""DroQ against the executing reference (where its checkout is available):

  * the registered `droq` entry point drives the UNMODIFIED reference interaction loop (droq.py:167-463) with this
    package's build_agent / train / Adam handles / replay buffer substituted, writes checkpoints in the reference's
    layout and resumes from one;
  * `sheeprl-eval`'s DroQ `evaluate` runs through the rebound build_agent.
Kernels are the torch test double."""
import os

import pytest
import torch

from oracle import ref_harness
from oracle.ops_emul_droq import DroQEmulOps
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


def _plain(d):
    return {k: _plain(v) for k, v in d.items()} if isinstance(d, dict) else d


def _cfg(tmp, total_steps=24, resume=None):
    from oracle.make_golden_droq import droq_cfg

    spec = dict(hidden=16, n_critics=2, B=4, p=0.1, seed=3)
    cfg = _plain(droq_cfg(spec))
    cfg["algo"].update(dict(total_steps=total_steps, learning_starts=8, replay_ratio=1.0, per_rank_pretrain_steps=0,
                            run_test=False))
    cfg.update(dict(dry_run=False, root_dir=str(tmp), run_name="run"))
    cfg["checkpoint"] = {"resume_from": resume, "every": 8, "save_last": True, "keep_last": 5}
    cfg["metric"] = {"log_level": 0, "log_every": 8, "sync_on_compute": False, "aggregator": {}}
    cfg["model_manager"] = {"disabled": True}
    cfg["buffer"] = {"size": 64, "memmap": False, "checkpoint": False, "validate_args": False, "from_numpy": False,
                     "sample_next_obs": False}
    cfg["env"] = {"num_envs": 2, "sync_env": True, "action_repeat": 1, "id": "dummy",
                  "wrapper": {"_target_": "tests.fake_gym.DummyImageEnv"}}
    return dotdict(cfg)


def _env(cfg, seed, *a, **k):
    return lambda: fake_gym.DummyImageEnv(size=8, length=11, seed=seed or 0, continuous=True, vector_dim=3)


def _harness():
    ref_harness.install()
    import sheeprl.algos.droq.droq as R
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
    import sheeprl_b200.algos.droq.agent as A
    import sheeprl_b200.algos.droq.droq as B
    from sheeprl_b200.data import buffers as Bf
    from sheeprl_b200.utils.registry import find_algorithm

    found = find_algorithm("droq")
    assert found is not None and found[0] == "sheeprl_b200.algos.droq" and found[1]["entrypoint"] == "main"
    real_build = A.build_agent
    monkeypatch.setattr(A, "build_agent", lambda *a, **k: real_build(*a, ops=DroQEmulOps(), **k))
    monkeypatch.setitem(Bf.DEFAULTS, "ops", DroQEmulOps())
    seen = {"train": 0, "G": [], "engines": [], "opt": [], "rb": []}
    orig_train = B.train

    def counting_train(fabric, agent, actor_opt, qf_opt, alpha_opt, rb, aggregator, cfg, g, **k):
        seen["train"] += 1
        seen["G"].append(g)
        seen["engines"].append(agent._b200_engine)
        seen["opt"].append((actor_opt, qf_opt, alpha_opt))
        seen["rb"].append(rb)
        return orig_train(fabric, agent, actor_opt, qf_opt, alpha_opt, rb, aggregator, cfg, g, **k)

    monkeypatch.setattr(B, "train", counting_train)
    ref_train, ref_build, ref_rb = R.train, R.build_agent, R.ReplayBuffer
    fab = Fabric()
    B.main(fab, _cfg(tmp_path))
    assert R.train is ref_train and R.build_agent is ref_build and R.ReplayBuffer is ref_rb
    assert seen["train"] > 0 and all(g >= 1 for g in seen["G"])
    assert isinstance(seen["rb"][0], Bf.ReplayBuffer)
    assert all(isinstance(o, B.B200Adam) for o in seen["opt"][0])
    eng = seen["engines"][0]
    assert eng.qf.step == sum(seen["G"])                             # one Adam step per critic minibatch
    ck = fab.checkpoints[-1]["state"]
    assert set(ck) >= {"agent", "qf_optimizer", "actor_optimizer", "alpha_optimizer", "ratio", "iter_num",
                       "batch_size", "last_log", "last_checkpoint"}
    assert any(k.startswith("_qfs_unwrapped.") for k in ck["agent"])
    qsd = ck["qf_optimizer"]
    assert len(qsd["state"]) == 20 and int(qsd["state"][0]["step"]) == sum(seen["G"])
    assert all(torch.isfinite(v).all() for v in ck["agent"].values())
    # resume from the last checkpoint: parameters and Adam states go back in, the step count continues
    n_before = seen["train"]
    path = fab.checkpoints[-1]["ckpt_path"]
    fab2 = Fabric()
    B.main(fab2, _cfg(tmp_path, total_steps=40, resume=path))
    eng2 = seen["engines"][-1]
    assert eng2 is not eng and seen["train"] > n_before
    st2 = fab2.checkpoints[-1]["state"]
    assert int(st2["qf_optimizer"]["state"][0]["step"]) == sum(seen["G"]) and st2["iter_num"] > ck["iter_num"]


def test_evaluate_runs_through_the_rebound_build_agent(tmp_path, monkeypatch):
    ref_harness.install()
    import sheeprl.algos.droq.evaluate as RE
    import sheeprl.algos.sac.utils as SU

    import sheeprl_b200.algos.droq.agent as A
    from sheeprl_b200.algos.droq.evaluate import evaluate_droq

    cfg = _cfg(tmp_path)
    cfg.dry_run = True
    monkeypatch.setattr(RE, "gym", fake_gym.module())
    monkeypatch.setattr(RE, "make_env", _env)
    monkeypatch.setattr(SU, "make_env", _env)
    monkeypatch.setattr(RE, "get_logger", lambda fabric, cfg: None)
    monkeypatch.setattr(RE, "get_log_dir", lambda fabric, root, run: os.path.join(root, run))
    built = []
    real_build = A.build_agent

    def build(*a, **k):
        out = real_build(*a, ops=DroQEmulOps(), **k)
        built.append(out)
        return out

    monkeypatch.setattr(A, "build_agent", build)
    src, _ = build(Fabric(), cfg, {"state": fake_gym.Box(-1, 1, (3,))}, fake_gym.Box(-1.0, 1.0, (2,)))
    state = {"agent": src.state_dict()}
    evaluate_droq(Fabric(), cfg, state)
    assert RE.build_agent is not build and len(built) == 2               # rebound only for the call
    agent, player = built[1]
    for k, v in agent.state_dict().items():
        assert torch.equal(v, state["agent"][k]), k
    obs = torch.zeros(1, 3)
    assert player.get_actions(obs, greedy=True).shape == (1, 2)
