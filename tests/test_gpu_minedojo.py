"""The MineDojo actor on the H100: `b200rl_minedojo_sample` against its float64 specification
(oracle/ops_emul_minedojo.py) and against `b200rl_cat_sample`, across head widths and strided / unaligned column blocks,
its sampling frequencies, its determinism, and the Dreamer-V3 / Plan2Explore engines with the MineDojo actor through
the C-ABI (executed-reference fixtures, a MineDojo-shaped step at the dreamer_v3_XS sizes against the oracle, a replayed
CUDA graph against an eager step)."""
import copy

import pytest
import torch

from oracle.make_golden_minedojo import ACTIONS_DIM
from oracle.ops_emul_minedojo import minedojo_sample_spec
from tests.helpers import assert_params_close, load_fixture
from tests.test_gpu_engine import check_grads, make_engine

pytestmark = pytest.mark.gpu
UNIMIX = 0.01
WIDTHS = [19, 33, 244, 640, 2048]


@pytest.fixture(scope="module")
def ops():
    from sheeprl_b200.lib import CudaOps

    return CudaOps("cuda")


def case(M, dims, seed, scale=3.0, col=0, pad=0):
    """raw logits, Exp(1) noise and one-hot output as [M, A] column blocks starting at column `col` of wider rows
    (row stride A + col + pad: strided and, for odd col, not 16-byte aligned); the output's guard columns are NaN"""
    g = torch.Generator().manual_seed(seed)
    A = sum(dims)
    ld = A + col + pad
    raw = (torch.randn(M, ld, generator=g) * scale).cuda()
    q = torch.empty(M, ld).exponential_(generator=g).cuda()
    out = torch.full((M, ld), float("nan"), device="cuda")
    return raw[:, col:col + A], q[:, col:col + A], out, out[:, col:col + A]


def rand_masks(M, dims, g, p=0.3, force=True):
    K0, K1, K2 = dims
    m = [torch.rand(M, K0, generator=g) < 0.5, torch.rand(M, K1, generator=g) < p, torch.rand(M, K2, generator=g) < p,
         torch.rand(M, K2, generator=g) < p]
    if force and K0 > 18:                      # every branch of the chain: rows forced to 15, 16, 17, 18, other
        for r in range(M):
            c = [15, 16, 17, 18, r % 15][r % 5]
            m[0][r] = False
            m[0][r, c] = True
    return [x.float().cuda() for x in m]


@pytest.mark.parametrize("greedy", [False, True])
@pytest.mark.parametrize("dims", [(19, 40, 72), (19, 244, 640), (19, 2048, 33)])
def test_kernel_matches_float64_spec(ops, dims, greedy):
    M = 512
    raw, q, _, hot = case(M, dims, seed=1, col=3, pad=5)
    masks = rand_masks(M, dims, torch.Generator().manual_seed(2))
    ops.minedojo_sample(raw, None if greedy else q, UNIMIX, dims, hot, *masks)
    want, _ = minedojo_sample_spec(raw.double().cpu(), None if greedy else q.double().cpu(), UNIMIX, dims,
                                   [m.double().cpu() for m in masks])
    assert torch.equal(hot.cpu().double(), want)


@pytest.mark.parametrize("K", WIDTHS)
@pytest.mark.parametrize("col", [0, 1])
def test_all_true_masks_are_bit_identical_to_cat_sample(ops, K, col):
    dims = (19, K, K if K != 2048 else 7)
    M = 300
    raw, q, guarded, hot = case(M, dims, seed=K + col, col=col, pad=3)
    ones = [torch.ones(M, k, device="cuda") for k in (dims[0], dims[1], dims[2], dims[2])]
    ref = torch.empty_like(hot)
    off = 0
    for k in dims:
        ops.cat_sample(raw[:, off:off + k], q[:, off:off + k], UNIMIX, 1, k, ref[:, off:off + k])
        off += k
    for masks in (ones, [None] * 4):
        guarded.fill_(float("nan"))
        ops.minedojo_sample(raw, q, UNIMIX, dims, hot, *masks)
        assert torch.equal(hot, ref)
        assert bool(guarded[:, :col].isnan().all()) and bool(guarded[:, col + sum(dims):].isnan().all())


@pytest.mark.parametrize("K", WIDTHS)
def test_widths_on_strided_unaligned_blocks_respect_the_masks(ops, K):
    dims = (19, K, K)
    M = 257
    raw, q, guarded, hot = case(M, dims, seed=K, col=5, pad=1)
    masks = rand_masks(M, dims, torch.Generator().manual_seed(K))
    ops.minedojo_sample(raw, q, UNIMIX, dims, hot, *masks)
    h = hot.cpu()
    assert bool((h.sum(-1) == 3).all()) and bool(((h == 0) | (h == 1)).all())
    a0, a1, a2 = h[:, :19].argmax(-1), h[:, 19:19 + K].argmax(-1), h[:, 19 + K:].argmax(-1)
    m = [x.cpu() for x in masks]
    r = torch.arange(M)
    assert bool(m[0][r, a0].all())
    craft, equip, destroy = a0 == 15, (a0 == 16) | (a0 == 17), a0 == 18
    for sel, mk, a in ((craft, m[1], a1), (equip, m[2], a2), (destroy, m[3], a2)):
        ok = mk[r, a].bool() | ~mk.bool().any(-1)
        assert bool(ok[sel].all())
    assert bool(guarded[:, :5].isnan().all()) and bool(guarded[:, 5 + sum(dims):].isnan().all())


def test_all_masked_group_falls_back_to_a_valid_one_hot(ops):
    dims = (19, 244, 640)
    M = 64
    raw, q, _, hot = case(M, dims, seed=9)
    m0 = torch.zeros(M, 19, device="cuda")
    m0[: M // 2, 15] = 1.0                          # half the rows: craft with an all-false craft mask
    none = [m0, torch.zeros(M, 244, device="cuda"), torch.zeros(M, 640, device="cuda"), torch.zeros(M, 640, device="cuda")]
    ops.minedojo_sample(raw, q, UNIMIX, dims, hot, *none)
    free = torch.empty_like(hot)
    ops.minedojo_sample(raw, q, UNIMIX, dims, free)
    assert bool((hot.sum(-1) == 3).all()) and bool(torch.isfinite(hot).all())
    assert bool((hot[: M // 2, :19].argmax(-1) == 15).all())
    assert torch.equal(hot[:, 19:], free[:, 19:])            # the all-false masks fall back to the unmasked heads
    assert torch.equal(hot[M // 2:, :19], free[M // 2:, :19])


def test_sample_frequencies_match_the_masked_probabilities(ops):
    """one masked row repeated 32768 times on seeded Exp(1) noise: the total-variation distance of each head's
    empirical distribution (per functional action for the chained heads) from the float64 masked probabilities stays
    under 0.03 (head 0, about 3x its expected sampling error) and 0.03 + 2 sqrt(K / n) for the n rows of a functional
    action (the chained heads)"""
    dims = (19, 40, 72)
    M = 32768
    g = torch.Generator().manual_seed(11)
    row = torch.randn(1, sum(dims), generator=g) * 1.5
    row[0, :19] = torch.linspace(-0.5, 0.5, 19)
    masks = [x[:1].expand(M, -1).contiguous() for x in rand_masks(8, dims, g, p=0.5, force=False)]
    masks[0].zero_()
    masks[0][:, [0, 15, 16, 18]] = 1.0                           # every branch of the chain, each ~1/4 of the rows
    raw = row.expand(M, -1).contiguous().cuda()
    q = torch.empty(M, sum(dims)).exponential_(generator=g).cuda()
    hot = torch.empty_like(raw)
    ops.minedojo_sample(raw, q, UNIMIX, dims, hot, *masks)
    h = hot.cpu()
    a0 = h[:, :19].argmax(-1)
    _, probs = minedojo_sample_spec(row.double(), None, UNIMIX, dims, [m[:1].double().cpu() for m in masks])
    tv0 = 0.5 * float((torch.bincount(a0, minlength=19).double() / M - probs[0][0]).abs().sum())
    assert tv0 < 0.03, tv0
    for f in (15, 16, 18, 0):
        sel = a0 == f
        n = int(sel.sum())
        assert n > 500, (f, n)
        # head-1/2 probabilities given the functional action f: recompute with head 0 forced to f
        m0 = torch.zeros(1, 19, dtype=torch.float64)
        m0[0, f] = 1.0
        _, pf = minedojo_sample_spec(row.double(), None, UNIMIX, dims, [m0] + [m[:1].double().cpu() for m in masks[1:]])
        for head, (lo, k) in ((1, (19, 40)), (2, (59, 72))):
            emp = torch.bincount(h[sel, lo:lo + k].argmax(-1), minlength=k).double() / n
            tv = 0.5 * float((emp - pf[head][0]).abs().sum())
            assert tv < 0.03 + 2.0 * (k / n) ** 0.5, (f, head, tv, n)


def test_reruns_are_bit_identical_in_deterministic_mode(ops):
    dims = (19, 244, 640)
    raw, q, _, hot = case(4096, dims, seed=13)
    masks = rand_masks(4096, dims, torch.Generator().manual_seed(14))
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (True, False):
            torch.use_deterministic_algorithms(det)
            ops.set_deterministic(det)
            outs = []
            for _ in range(3):
                ops.minedojo_sample(raw, q, UNIMIX, dims, hot, *masks)
                outs.append(hot.clone())
            assert all(torch.equal(outs[0], o) for o in outs[1:]), det
    finally:
        torch.use_deterministic_algorithms(prev)
        ops.set_deterministic(prev)


# ------------------------------------------------------------------ engines through the C-ABI
def test_dv3_engine_cuda_matches_the_minedojo_fixture():
    from tests.test_minedojo_cpu import oracle_run, without_action_noise

    fx, cfg = load_fixture("dv3_minedojo")
    fdata = [{k: v.float() for k, v in d.items()} for d in fx["data"]]
    _, o_outs, _, _ = oracle_run(cfg, ACTIONS_DIM, fx["init"], fdata, fx["noise"], 1, keep=True)
    eng = make_engine(cfg, ACTIONS_DIM, fx["init"])
    assert eng.minedojo
    for s in range(len(fdata)):
        noise = {k: v.cuda() for k, v in without_action_noise(fx["noise"][s]).items()}
        eng.train_step({k: v.clone().cuda() for k, v in fdata[s].items()}, noise)
        if s == 0:
            check_grads({g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")},
                        o_outs[0], cfg, 3e-5)
            assert torch.equal(eng.actions.cpu(), o_outs[0]["imagined_actions"])
        got = {k: float(v) for k, v in eng.metrics_dict().items()}
        for k, v in fx["metrics"][s].items():
            assert got[k] == pytest.approx(v, rel=1e-4, abs=1e-6), (s, k)
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        assert_params_close({k: v.cpu() for k, v in g.views.items()}, fx["after"][n], 1e-4 if n == "wm" else 8e-5,
                            len(fdata), tol=3e-6, label=n)


def test_p2e_engine_cuda_matches_the_minedojo_fixture():
    from sheeprl_b200.algos.p2e_dv3.engine import P2EDV3Engine
    from tests.test_minedojo_cpu import p2e_case, without_action_noise
    from tests.test_p2e_cpu import LR, check_metrics, check_moments

    fx, cfg = p2e_case()
    eng = P2EDV3Engine(cfg, fx["actions_dim"], in_channels=3, device="cuda")
    for name, g in eng.groups().items():
        g.load(fx["init"][name])
    eng.load_ensembles(fx["init"]["ens"])
    for s in range(len(fx["data"])):
        noise = {k: v.cuda() for k, v in without_action_noise(fx["noise"][s]).items()}
        eng.train_step({k: v.clone().float().cuda() for k, v in fx["data"][s].items()}, noise)
        check_metrics({k: v.cpu() for k, v in eng.metrics_dict().items()}, fx["metrics"][s], f"engine step{s}")
    got = {name: {k: v.cpu() for k, v in g.state_dict().items()} for name, g in eng.groups().items()}
    got["ens"] = {k: v.cpu() for k, v in eng.ensembles_state_dict().items()}
    for name, want in fx["after"].items():
        assert_params_close(got[name], want, LR.get(name, 8e-5), len(fx["data"]), tol=3e-6, label=name)
    check_moments({"task": eng.moments_state.cpu(), **{k: c["moments_state"].cpu() for k, c in eng.critics_expl.items()}},
                  fx["moments"])


XS_DIMS = (19, 244, 640)


def xs_case():
    from oracle import dv3_oracle as O
    from oracle.make_golden_minedojo import DV3_ACTOR
    from sheeprl_b200.configs import make_dv3_cfg

    masks = {"mask_action_type": 19, "mask_craft_smelt": 244, "mask_equip_place": 640, "mask_destroy": 640}
    cfg = make_dv3_cfg("XS", mlp_keys=masks, algo__actor__cls=DV3_ACTOR)
    wm, actor, critic, target = O.init_params(cfg, XS_DIMS, seed=0)
    g = torch.Generator().manual_seed(3)
    for d in (wm, actor, critic):
        for v in d.values():
            v.add_(torch.randn(v.shape, generator=g) * 0.02)
    init = {"wm": wm, "actor": actor, "critic": critic, "target": target}
    data = O.make_batch(cfg, XS_DIMS, seed=4)
    for k in masks:
        data[k] = (data[k] > 0).float()
    a, w = cfg.algo, cfg.algo.world_model
    noise = O.draw_noise(a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon, w.stochastic_size, w.discrete_size,
                         XS_DIMS, seed=5)
    noise["img_action"] = [[None] * (a.horizon + 1) for _ in XS_DIMS]
    return cfg, init, data, noise


def test_minedojo_step_at_xs_size_vs_oracle():
    """dreamer_v3_XS sizes with MineDojo-like head widths [19, 244, 640] and the four mask keys encoded and decoded:
    the world-model gradients against the autograd oracle, the imagined mode actions (a mode may flip on a near-tie
    between two logits, so at most 0.1% of the rows may differ) and the behaviour metrics"""
    from oracle.dv3_decoder_keys_oracle import decoder_keys
    from tests.helpers import oracle_run

    cfg, init, data, noise = xs_case()
    with decoder_keys():
        st, o_outs, _, _ = oracle_run(cfg, XS_DIMS, init, [data], [noise], 1, condition_margin=1e-3, keep=True)
    eng = make_engine(cfg, XS_DIMS, init)
    assert eng.minedojo and eng.A == sum(XS_DIMS)
    noise_c = {k: v.cuda() for k, v in noise.items() if k != "img_action"}
    eng.train_step({k: v.clone().float().cuda() for k, v in data.items()}, noise_c)
    torch.cuda.synchronize()
    grads = {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")}
    og = o_outs[0]["grads/wm"]
    gnorm = float(torch.sqrt(sum((v.double() ** 2).sum() for v in og.values())))
    coef = min(1.0, cfg.algo.world_model.clip_gradients / (float(o_outs[0]["Grads/world_model"]) + 1e-6))
    for k, v in og.items():
        rel = float((grads["wm"][k].cpu() * coef - v).double().norm()) / (float(v.double().norm()) + 1e-6 * gnorm + 1e-30)
        assert rel <= 1e-4, (k, rel)
    acts, want = eng.actions.cpu(), o_outs[0]["imagined_actions"]
    assert bool((acts.sum(-1) == 3).all())
    same = (acts == want).all(-1).double().mean()
    assert float(same) >= 0.999, float(same)
    got = {k: float(v) for k, v in eng.metrics_dict().items()}
    for k in ("Loss/world_model_loss", "Loss/observation_loss", "State/kl"):
        assert got[k] == pytest.approx(float(o_outs[0][k]), rel=1e-4), k
    for k in ("Loss/policy_loss", "Loss/value_loss"):
        assert got[k] == pytest.approx(float(o_outs[0][k]), rel=1e-2, abs=1e-4), k


def test_replayed_graph_is_bit_identical_to_an_eager_step():
    """one eager MineDojo step, then the same step (same parameters, same Philox position) captured and replayed: the
    imagined mode actions and the latent states are bit-identical"""
    from sheeprl_b200.graph import StepGraph

    fx, cfg = load_fixture("dv3_minedojo")
    eng = make_engine(cfg, ACTIONS_DIM, fx["init"])
    eng.rng_seed = 77
    batch = {k: v.clone().float().cuda() for k, v in fx["data"][0].items()}
    flats = [g.flat.clone() for g in (eng.wm, eng.actor, eng.critic)]
    rng0 = eng.rng_t.clone()
    eng.train_step({k: v.clone() for k, v in batch.items()}, None)
    torch.cuda.synchronize()
    eager = {n: getattr(eng, n).clone() for n in ("latent", "actions", "traj")}
    for g, f in zip((eng.wm, eng.actor, eng.critic), flats):
        g.flat.copy_(f)
    eng.rng_t.copy_(rng0)
    StepGraph(eng.device, warmup=0).run(lambda d: eng.train_step(d, None), batch)
    torch.cuda.synchronize()
    for n, v in eager.items():
        assert torch.equal(getattr(eng, n), v), n


def test_player_masked_step_on_the_gpu_matches_the_spec():
    """the acting step through the C-ABI: the masked mode of the player's own head logits equals the float64
    specification, and a sampled step honours the masks"""
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent
    from tests.test_minedojo_cpu import Fab as _Fab
    from tests.test_minedojo_cpu import hand_masks, obs_space_of

    class Fab(_Fab):
        device = torch.device("cuda")

    fx, cfg = load_fixture("dv3_minedojo")
    cfg = copy.deepcopy(cfg)
    E = 16
    cfg.env.num_envs = E
    *_, player = build_agent(Fab, ACTIONS_DIM, False, cfg, obs_space_of(cfg), fx["init"]["wm"], fx["init"]["actor"],
                             fx["init"]["critic"], fx["init"]["target"])
    g = torch.Generator().manual_seed(4)
    masks = hand_masks(E, g)
    obs = {"rgb": (torch.rand(1, E, 3, 64, 64, generator=g) - 0.5).cuda()}
    obs.update({k: v.unsqueeze(0).cuda() for k, v in masks.items()})
    player.init_states()
    got = player.get_actions(obs, True, {k: v.unsqueeze(0).cuda() for k, v in masks.items()})
    raw = player.eng.actor_raw[:E].double().cpu()
    want, _ = minedojo_sample_spec(raw, None, cfg.algo.unimix, ACTIONS_DIM,
                                   [masks[k].double() for k in ("mask_action_type", "mask_craft_smelt", "mask_equip_place",
                                                                "mask_destroy")])
    assert torch.equal(torch.cat(got, -1)[0].cpu().double(), want)
