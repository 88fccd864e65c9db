"""Plan2Explore (Dreamer-V3) with continuous actions on the GPU through the C-ABI: the engine and the public
build_agent()/train() surface against the executed reference (tests/golden/p2e_tiny_c.pt), and on-device Philox noise."""
import pytest
import torch

from tests.test_p2e_continuous_cpu import check_engine, check_public_api, load, make_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


def test_engine_matches_reference(cu):
    fx, cfg = load()
    check_engine(fx, make_engine(fx, cfg, device="cuda", ops=cu))


def test_public_api_matches_reference(cu):
    check_public_api(device="cuda", ops=cu)


def test_production_noise_step_is_finite_and_explores(cu):
    """on-device Philox noise: two updates stay finite and move the exploration actor, the ensemble members disagree
    (intrinsic reward > 0), and the exploration and task rollouts draw different action noise (N(0,1): both signs)"""
    fx, cfg = load()
    eng = make_engine(fx, cfg, device="cuda", ops=cu)
    data = {k: v.clone().float().cuda() for k, v in fx["data"][0].items()}
    before = eng.actor_expl.flat.clone()
    for _ in range(2):
        eng.train_step(data, None)
    md = {k: float(v) for k, v in eng.metrics_dict().items()}
    assert all(v == v and abs(v) < 1e30 for v in md.values()), md
    assert md["Rewards/intrinsic_intrinsic"] > 0
    assert not torch.equal(eng.actor_expl.flat, before)
    assert not torch.equal(eng.noise_img_action_expl, eng.noise_img_action)
    assert not torch.equal(eng.noise_img_state_expl, eng.noise_img_state)
    assert float(eng.noise_img_action_expl.min()) < 0 < float(eng.noise_img_action_expl.max())
