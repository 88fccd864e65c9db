"""Decoupled RSSM on the GPU: the persistent GRU-only scan kernels (`b200rl_gru_scan_fwd` / `_bwd`, csrc/rssm_scan.cu)
against the float64 reference over their envelope, their refusals outside it, and the engine through the C-ABI against
the executed-reference fixtures, the oracle at the BASELINE S shape, its own per-step schedule and a replayed graph."""
import math

import pytest
import torch

from oracle import dv3_decoupled_oracle as OD
from oracle.gru_scan_ref import gru_scan_reference
from tests.helpers import assert_params_close, load_fixture
from tests.helpers import oracle_run as coupled_oracle_run
from tests.test_gpu_engine import check_grads, make_engine, to_cuda
from tests.test_gpu_rssm_scan import BWD_RTOL, EPS, FWD_RTOL, make_first

pytestmark = pytest.mark.gpu

NAN = float("nan")


def oracle_run(*a, **k):
    with OD.decoupled():
        return coupled_oracle_run(*a, **k)

FWD_OUT, BWD_OUT = ("g_pre", "g_ln", "h_in", "latent"), ("d_g_ln", "d_h0")


@pytest.fixture(scope="module")
def ops():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


def make_problem(T, B, R, seed, first="random", pad=3):
    """Operands of the GRU scan: W_g is the full [3R, R + Dx] weight (its x columns must not be read: NaN), latent has
    z columns in front of h and padding behind (NaN: must stay untouched)."""
    g = torch.Generator().manual_seed(seed)
    Dx, off = 6, 10
    ld_lat = off + R + pad
    dims = dict(T=T, B=B, R=R, ld_wg=R + Dx, ld_lat=ld_lat, lat_off=off)
    W = torch.full((3 * R, R + Dx), NAN)
    W[:, :R] = torch.randn(3 * R, R, generator=g) / math.sqrt(R)
    if first == "ones":
        f = torch.ones(T, B)
    elif first == "row0":
        f = torch.zeros(T, B)
        f[0] = 1.0
    else:
        f = make_first(T, B, g, False).reshape(T, B).float()
        f[0] = 1.0
    N = T * B
    x_share = torch.randn(N, 3 * R, generator=g)
    t = dict(W_g=W, lng_g=1 + 0.1 * torch.randn(3 * R, generator=g), lng_b=0.1 * torch.randn(3 * R, generator=g),
             h0=torch.tanh(torch.randn(R, generator=g)), first=f.reshape(N), g_pre=x_share.clone(),
             g_ln=torch.full((N, 3 * R), NAN), h_in=torch.full((N, R), NAN), latent=torch.full((N, ld_lat), NAN))
    gr = dict(d_latent=torch.randn(N, ld_lat, generator=g), q_g=torch.full((N, R), NAN),
              d_g_ln=torch.full((N, 3 * R), NAN), d_h0=torch.full((R,), NAN))
    return dims, {k: v.cuda() for k, v in t.items()}, {k: v.cuda() for k, v in gr.items()}, x_share


def run_fwd(ops, dims, t, x_share, ws):
    t["g_pre"].copy_(x_share)
    ops.gru_scan_fwd(dims, EPS, t, ws)
    assert ops.rssm_scan_error(ws) == 0, "a hand-off of the forward scan timed out"
    return {k: t[k].clone() for k in FWD_OUT}


def run_bwd(ops, dims, t, gr, ws):
    ops.gru_scan_bwd(dims, EPS, t, gr, ws)
    assert ops.rssm_scan_error(ws) == 0, "a hand-off of the backward scan timed out"
    return {k: gr[k].clone() for k in BWD_OUT}


CASES = [(T, B, R, first) for T, B, R, first in [
    (1, 1, 8, "ones"), (2, 3, 24, "random"), (64, 16, 40, "random"), (2, 16, 512, "row0"), (64, 16, 512, "random"),
    (64, 7, 520, "random"), (2, 5, 1024, "ones"), (64, 16, 1024, "row0"), (64, 2, 8, "row0"), (2, 11, 40, "ones")]]


@pytest.mark.parametrize("T,B,R,first", CASES)
def test_gru_scan_kernels_match_float64_reference(ops, T, B, R, first):
    dims, t, gr, x_share = make_problem(T, B, R, seed=200 + R + B, first=first)
    assert ops.gru_scan_supported(dims, backward=False) and ops.gru_scan_supported(dims, backward=True)
    ws = ops.gru_scan_workspace(T, B, R)
    fwd = run_fwd(ops, dims, t, x_share.cuda(), ws)
    ops.gemm(t["g_pre"], t["W_g"][:, :R], gr["q_g"], False, False)
    bwd = run_bwd(ops, dims, t, gr, ws)
    cpu = {k: v.cpu() for k, v in (t | gr).items()}
    off, lat = dims["lat_off"], cpu["latent"]
    # ---- the kernels write exactly what they own
    assert lat[:, :off].isnan().all() and lat[:, off + R:].isnan().all(), "latent columns outside h were written"
    for k in ("g_pre", "g_ln", "h_in", "d_g_ln", "d_h0"):
        assert torch.isfinite(cpu[k]).all(), (k, "not every owned element was written (or it is not finite)")
    h = lat[:, off:off + R]
    assert torch.isfinite(h).all()
    # ---- chain consistency, bit-exact
    f = cpu["first"].reshape(T, B, 1) != 0
    prev_h = torch.cat((torch.zeros(1, B, R), h.reshape(T, B, R)[:-1]), 0)
    assert torch.equal(cpu["h_in"].reshape(T, B, R), torch.where(f, cpu["h0"].expand(T, B, R), prev_h)), "h_in"
    # ---- forward, one step at a time from the kernel's own h_in
    one = gru_scan_reference(dims, EPS, cpu, x_share, one_step=True)
    margins = {}
    for k, got in (("g_pre", cpu["g_pre"]), ("g_ln", cpu["g_ln"]), ("h", h)):
        err = float((got.double() - one[k]).abs().max())
        margins[k] = err / (FWD_RTOL * math.sqrt(R) * max(1e-3, float(one[k].abs().max())))
    # ---- backward against float64 autograd of the carried chain
    ref = gru_scan_reference(dims, EPS, cpu, x_share, d_latent=cpu["d_latent"])
    for k in BWD_OUT:
        err = float((cpu[k].double() - ref[k]).abs().max())
        margins[k] = err / (BWD_RTOL * max(1e-3, float(ref[k].abs().max())))
    assert max(margins.values()) <= 1.0, {k: round(v, 3) for k, v in margins.items()}
    # ---- bit-reproducible (fixed-order K-slice sums); the backward reruns on the same q_g
    fwd2 = run_fwd(ops, dims, t, x_share.cuda(), ws)
    for k in FWD_OUT:
        v1, v2 = ((x[:, off:off + R] if k == "latent" else x) for x in (fwd[k], fwd2[k]))
        assert torch.equal(v1, v2), (k, "second forward differs")
    bwd2 = run_bwd(ops, dims, t, gr, ws)
    for k in BWD_OUT:
        assert torch.equal(bwd[k], bwd2[k]), (k, "second backward differs")


REFUSALS = {"B17": (4, 17, 64), "R_odd": (4, 4, 63), "R1028": (4, 4, 1028), "short_workspace": (4, 4, 64)}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_gru_scan_check_and_launches_refuse_outside_envelope(ops, name):
    """The envelope query refuses in both directions, the launches refuse the same shapes (and a short workspace)
    before anything is launched: all outputs stay untouched."""
    from sheeprl_b200.lib import B200RLError

    T, B, R = REFUSALS[name]
    dims, t, gr, x_share = make_problem(T, B, R, seed=7)
    ws = ops.gru_scan_workspace(T, B, R)
    in_envelope = name == "short_workspace"
    assert ops.gru_scan_supported(dims, backward=False) == in_envelope
    assert ops.gru_scan_supported(dims, backward=True) == in_envelope
    if name == "short_workspace":
        ws, match = ws[:-1], "workspace"
    else:
        match = "supports|shared memory"
    for call in (lambda: ops.gru_scan_fwd(dims, EPS, t, ws), lambda: ops.gru_scan_bwd(dims, EPS, t, gr, ws)):
        with pytest.raises(B200RLError, match=match):
            call()
    torch.cuda.synchronize()
    assert torch.equal(t["g_pre"].cpu(), x_share), "g_pre written by a refused call"
    for k in ("g_ln", "h_in", "latent"):
        assert t[k].isnan().all(), (k, "written by a refused call")
    for k in BWD_OUT:
        assert gr[k].isnan().all(), (k, "written by a refused call")


@pytest.mark.parametrize("name", ["dv3_tiny_d", "dv3_tiny_dv"])
def test_engine_cuda_matches_decoupled_reference_fixture(name):
    fx, cfg = load_fixture(name)
    adim, steps, cont = fx["actions_dim"], len(fx["data"]), fx["is_continuous"]
    fdata = [{k: v.float() for k, v in d.items()} for d in fx["data"]]
    st, o_outs, ms, _ = oracle_run(cfg, adim, fx["init"], fdata, fx["noise"], steps, keep=True, is_continuous=cont)
    eng = make_engine(cfg, adim, fx["init"], cont)
    assert eng.decoupled and eng.fused_scan and eng.fused_scan_bwd
    for s in range(steps):
        eng.train_step({k: v.clone().float().cuda() for k, v in fx["data"][s].items()}, to_cuda(fx["noise"][s]))
        if s == 0:
            grads = {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")}
            check_grads(grads, o_outs[0], cfg, 3e-5)
        got = {k: float(v) for k, v in eng.metrics_dict().items()}
        for k, v in fx["metrics"][s].items():
            assert got[k] == pytest.approx(v, rel=1e-4, abs=1e-6), (s, k)
    assert eng.ops.rssm_scan_error(eng._scan_ws) == 0
    lrs = {"wm": 1e-4, "actor": 8e-5, "critic": 8e-5}
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        assert_params_close({k: v.cpu() for k, v in g.views.items()}, fx["after"][n], lrs[n], steps, tol=3e-6, label=n)
    assert float(eng.moments_state[0]) == pytest.approx(float(fx["moments"]["low"]), rel=1e-4, abs=1e-7)
    assert float(eng.moments_state[1]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


def baseline_case():
    from oracle import dv3_oracle as O
    from sheeprl_b200.configs import make_dv3_cfg

    cfg, adim = make_dv3_cfg("S", algo__world_model__decoupled_rssm=True), (2,)
    wm, actor, critic, target = OD.init_params(cfg, adim, seed=0)
    g = torch.Generator().manual_seed(3)
    for d in (wm, actor, critic):
        for v in d.values():
            v.add_(torch.randn(v.shape, generator=g) * 0.02)
    init = {"wm": wm, "actor": actor, "critic": critic, "target": target}
    data = O.make_batch(cfg, adim, seed=4)
    data["is_first"][7, 3] = 1.0
    data["is_first"][31, 0] = 1.0
    a, w = cfg.algo, cfg.algo.world_model
    noise = O.draw_noise(a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon, w.stochastic_size, w.discrete_size,
                         adim, seed=5)
    return cfg, adim, init, data, noise


def test_decoupled_engine_at_baseline_shape_vs_oracle_and_per_step():
    """BASELINE S shape (B16 T64 H15): every gradient against the autograd oracle, and the persistent GRU scan against
    the per-step schedule of the same engine."""
    cfg, adim, init, data, noise = baseline_case()
    st, o_outs, ms, _ = oracle_run(cfg, adim, init, [data], [noise], 1, condition_margin=1e-3, keep=True)
    outs = []
    for fused in (False, True):
        eng = make_engine(cfg, adim, init)
        assert eng.fused_scan and eng.fused_scan_bwd, "the S model is inside the GRU scan's envelope"
        eng.fused_scan = fused
        eng.train_step({k: v.clone().float().cuda() for k, v in data.items()}, to_cuda(noise))
        torch.cuda.synchronize()
        if fused:
            assert eng.ops.rssm_scan_error(eng._scan_ws) == 0, "a hand-off of the persistent scan timed out"
            grads = {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")}
            check_grads(grads, o_outs[0], cfg, 1e-4)
            assert torch.equal(eng.latent[:, : eng.Z].cpu().reshape(o_outs[0]["latent"][..., : eng.Z].shape),
                               o_outs[0]["latent"][..., : eng.Z].round()), "posterior samples differ"
            for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
                assert_params_close({k: v.cpu() for k, v in g.views.items()}, st[n], 1e-4, 1, tol=3e-6, frac=2e-3, label=n)
        outs.append({k: getattr(eng, k).clone() for k in (
            "latent", "z_in", "h_in", "a_in", "x_pre", "x_act", "g_pre", "g_ln", "rp_pre", "rp_act", "post_raw", "post_mix",
            "prior_mix", "d_post_raw", "d_rp_pre", "d_g_pre", "d_x_pre", "d_g_ln", "d_h0")}
            | {"wm_grad": eng.wm.grad.clone(), "metrics": eng.metrics.clone()})
    ref, got = outs
    for k in ref:
        err = float((ref[k] - got[k]).abs().max())
        assert err <= 5e-5 * max(1e-3, float(ref[k].abs().max())), (k, err, float(ref[k].abs().max()))


def test_decoupled_train_eager_and_graph_replay_agree():
    """the public build_agent() + train(): three calls with the graph disabled and three with it (the third is captured
    and replayed) leave the same parameters"""
    from sheeprl_b200.algos.dreamer_v3.agent import build_agent
    from sheeprl_b200.algos.dreamer_v3.dreamer_v3 import make_optimizers, train
    from sheeprl_b200.algos.dreamer_v3.utils import Moments

    cfg0, adim, init, data, noise = baseline_case()

    class Fab:
        device = torch.device("cuda")

    class Space:
        shape = (3, 64, 64)

    class Agg:
        disabled = True

    after = []
    for graph in (False, True):
        from sheeprl_b200.configs import make_dv3_cfg

        cfg = make_dv3_cfg("S", algo__world_model__decoupled_rssm=True)
        cfg.algo.cuda_graph = graph
        wm, actor, critic, target, player = build_agent(Fab, adim, False, cfg, {"rgb": Space}, init["wm"], init["actor"],
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
        assert eng.ops.rssm_scan_error(eng._scan_ws) == 0
        after.append({k: v.clone().cpu() for k, v in eng.wm.views.items()})
    # same Philox stream in both runs; reductions with atomics differ in the last bits between runs, which can flip a
    # near-tie draw or the sign of a numerically zero gradient: the runs must agree to a small share of the update itself
    for k, v in after[0].items():
        moved = float((v - init["wm"][k]).double().norm())
        assert float((after[1][k] - v).double().norm()) <= 0.05 * moved + 1e-7, (k, moved)


def test_player_cuda_matches_decoupled_reference():
    from sheeprl_b200.lib import CudaOps
    from tests.test_player_cpu import check, run_player

    fx, got, cont = run_player("dv3_player_decoupled", device="cuda", ops=CudaOps())
    check(fx, got, cont)
