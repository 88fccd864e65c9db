"""Decoders over a subset of the encoded keys on the H100: the engine through the C-ABI against the executed-reference
fixtures, the DIAMBRA shape (image + three vector keys, two of them decoded in another order) at the BASELINE S size
against the autograd oracle including every gradient, and eager `train()` against the replayed CUDA graph."""
import pytest
import torch

from oracle.make_golden_decoder_keys import FIXTURES as SPECS
from oracle.make_golden_decoder_keys import oracle_for
from tests.helpers import assert_params_close, load_fixture
from tests.helpers import oracle_run as base_oracle_run
from tests.test_gpu_engine import check_grads, make_engine, to_cuda

pytestmark = pytest.mark.gpu
LRS = {"wm": 1e-4, "actor": 8e-5, "critic": 8e-5}


def oracle_run(cfg, *a, **k):
    with oracle_for(cfg):
        return base_oracle_run(cfg, *a, **k)


@pytest.mark.parametrize("name", list(SPECS))
def test_engine_cuda_matches_decoder_keys_fixture(name):
    fx, cfg = load_fixture(name)
    adim, steps, cont = fx["actions_dim"], len(fx["data"]), fx["is_continuous"]
    fdata = [{k: v.float() for k, v in d.items()} for d in fx["data"]]
    _, o_outs, _, _ = oracle_run(cfg, adim, fx["init"], fdata, fx["noise"], steps, keep=True, is_continuous=cont)
    eng = make_engine(cfg, adim, fx["init"], cont)
    for s in range(steps):
        eng.train_step({k: v.clone().float().cuda() for k, v in fx["data"][s].items()}, to_cuda(fx["noise"][s]))
        if s == 0:
            grads = {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")}
            check_grads(grads, o_outs[0], cfg, 3e-5)
        got = {k: float(v) for k, v in eng.metrics_dict().items()}
        for k, v in fx["metrics"][s].items():
            assert got[k] == pytest.approx(v, rel=1e-4, abs=1e-6), (s, k)
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        assert_params_close({k: v.cpu() for k, v in g.views.items()}, fx["after"][n], LRS[n], steps, tol=3e-6, label=n)
    assert float(eng.moments_state[1]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


def diambra_case(**over):
    from oracle import dv3_oracle as O
    from sheeprl_b200.configs import make_dv3_cfg

    cfg = make_dv3_cfg("S", mlp_keys={"own": 12, "opp": 12, "reward": 1}, **{"algo__mlp_keys__decoder": ["opp", "own"], **over})
    adim = (9, 4)
    wm, actor, critic, target = O.init_params(cfg, adim, seed=0)
    g = torch.Generator().manual_seed(3)
    for d in (wm, actor, critic):
        for v in d.values():
            v.add_(torch.randn(v.shape, generator=g) * 0.02)
    init = {"wm": wm, "actor": actor, "critic": critic, "target": target}
    data = O.make_batch(cfg, adim, seed=4)
    data["is_first"][7, 3] = 1.0
    a, w = cfg.algo, cfg.algo.world_model
    noise = O.draw_noise(a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon, w.stochastic_size, w.discrete_size,
                         adim, seed=5)
    return cfg, adim, init, data, noise


def test_diambra_shape_at_baseline_size_vs_oracle():
    """BASELINE S (B16 T64 H15) with `reward` encoded only and the decoder's keys in another order: every gradient
    against the autograd oracle, the posterior samples and the updated parameters"""
    cfg, adim, init, data, noise = diambra_case()
    st, o_outs, _, _ = oracle_run(cfg, adim, init, [data], [noise], 1, condition_margin=1e-3, keep=True)
    eng = make_engine(cfg, adim, init)
    assert eng.has_vec_dec and not eng.vec_dec_same and eng.Dvd == 24 and eng.Dv == 25
    eng.train_step({k: v.clone().float().cuda() for k, v in data.items()}, to_cuda(noise))
    torch.cuda.synchronize()
    grads = {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")}
    check_grads(grads, o_outs[0], cfg, 1e-4)
    assert torch.equal(eng.latent[:, : eng.Z].cpu().reshape(o_outs[0]["latent"][..., : eng.Z].shape),
                       o_outs[0]["latent"][..., : eng.Z].round()), "posterior samples differ"
    got = {k: float(v) for k, v in eng.metrics_dict().items()}
    assert got["Loss/observation_loss"] == pytest.approx(float(o_outs[0]["Loss/observation_loss"]), rel=1e-4)
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        assert_params_close({k: v.cpu() for k, v in g.views.items()}, st[n], 1e-4, 1, tol=3e-6, frac=2e-3, label=n)


@pytest.mark.parametrize("decoder", [["opp", "own"], []])
def test_train_eager_and_graph_replay_agree(decoder):
    """the public build_agent() + train() on the DIAMBRA and the Crafter (`mlp_keys.decoder: []`) shapes: three calls
    eager and three with the graph (the third is captured and replayed) leave the same parameters"""
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent
    from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import make_optimizers, train
    from sheeprl_b200.algos.dreamer_v3.utils import Moments

    cfg0, adim, init, data, _ = diambra_case(algo__mlp_keys__decoder=decoder)
    if not decoder:
        init["wm"] = {k: v for k, v in init["wm"].items() if not k.startswith("observation_model.mlp_decoder")}

    class Fab:
        device = torch.device("cuda")

    class Space:
        def __init__(self, *shape):
            self.shape = shape

    class Agg:
        disabled = True

    space = {"rgb": Space(3, 64, 64), "own": Space(12), "opp": Space(12), "reward": Space(1)}
    after = []
    for graph in (False, True):
        cfg, *_ = diambra_case(algo__mlp_keys__decoder=decoder)
        cfg.algo.cuda_graph = graph
        wm, actor, critic, target, player = build_agent(Fab, adim, False, cfg, space, init["wm"], init["actor"],
                                                        init["critic"], init["target"])
        eng = wm._b200_engine
        eng.rng_seed = 1234
        opts = make_optimizers(eng, cfg)
        mo = cfg.algo.actor.moments
        moments = Moments(mo.decay, mo.max, mo.percentile.low, mo.percentile.high)
        for _ in range(3):
            train(Fab, wm, actor, critic, target, *opts, {k: v.clone().cuda() for k, v in data.items()}, Agg(), cfg, False,
                  adim, moments)
        torch.cuda.synchronize()
        after.append({k: v.clone().cpu() for k, v in eng.wm.views.items()})
    for k, v in after[0].items():
        moved = float((v - init["wm"][k]).double().norm())
        assert float((after[1][k] - v).double().norm()) <= 0.05 * moved + 1e-7, (k, moved)


def test_player_acts_after_resizing_to_one_env():
    """the reference's test(): `player.num_envs = 1`, `init_states()`, then `get_actions` with an empty mask dict"""
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent

    fx, cfg = load_fixture("dv3_dec_diambra")

    class Fab:
        device = torch.device("cuda")

    class Space:
        def __init__(self, *shape):
            self.shape = shape

    space = {"rgb": Space(3, 64, 64)}
    space.update({k: Space(d) for k, d in cfg.env.mlp_dims.items()})
    *_, player = build_agent(Fab, fx["actions_dim"], False, cfg, space, fx["init"]["wm"], fx["init"]["actor"],
                             fx["init"]["critic"], fx["init"]["target"])
    player.num_envs = 1
    player.init_states()
    obs = {"rgb": torch.randint(0, 256, (1, 1, 3, 64, 64), dtype=torch.uint8, device="cuda")}
    obs.update({k: torch.randn(1, 1, d, device="cuda") for k, d in cfg.env.mlp_dims.items()})
    for _ in range(3):
        acts = player.get_actions(obs, False, {})
    torch.cuda.synchronize()
    assert [tuple(x.shape) for x in acts] == [(1, 1, ad) for ad in fx["actions_dim"]]
    assert all(float(x.sum()) == 1.0 for x in acts)


@pytest.mark.parametrize("decoder", [["opp", "own"], []])
def test_replayed_graph_targets_and_latents_are_bit_equal_to_eager(decoder):
    """one eager step, then the same step (same parameters, same Philox position) captured and replayed: the inputs,
    the decoder targets and the latent states must be bit-identical — a target buffer baked stale into the graph would
    differ here.  The per-row losses agree to 1e-6: the narrow head products (the continue logit, the vector decoder's
    heads) take the SIMT GEMM's split-K route, whose partial sums are added with atomics in run-dependent order."""
    from sheeprl_b200.graph import StepGraph

    _, adim, init, data, _ = diambra_case(algo__mlp_keys__decoder=decoder)
    if not decoder:
        init["wm"] = {k: v for k, v in init["wm"].items() if not k.startswith("observation_model.mlp_decoder")}
    cfg, *_ = diambra_case(algo__mlp_keys__decoder=decoder)
    eng = make_engine(cfg, adim, init)
    eng.rng_seed = 77
    batch = {k: v.clone().float().cuda() for k, v in data.items()}
    wm0, rng0 = eng.wm.flat.clone(), eng.rng_t.clone()
    names = ["x0", "vx", "latent"] + (["vtgt"] if decoder else [])
    rows = ["obs_rows", "rew_rows", "cont_rows", "kl_rows"] + (["vec_rows"] if decoder else [])
    eng.train_step({k: v.clone() for k, v in batch.items()}, None)
    torch.cuda.synchronize()
    eager = {n: getattr(eng, n).clone() for n in names + rows}
    eng.wm.flat.copy_(wm0)
    eng.rng_t.copy_(rng0)
    StepGraph(eng.device, warmup=0).run(lambda d: eng.train_step(d, None), batch)
    torch.cuda.synchronize()
    for n in names:
        assert torch.equal(getattr(eng, n), eager[n]), n
    for n in rows:
        err = float((getattr(eng, n) - eager[n]).abs().max())
        assert err <= 1e-6 * max(1.0, float(eager[n].abs().max())), (n, err)
    assert eng.has_vec_dec == bool(decoder)
