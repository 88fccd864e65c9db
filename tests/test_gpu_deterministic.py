"""Deterministic mode on the GPU (torch.use_deterministic_algorithms(True) -> b200rl_set_deterministic(1)).

Kernels: every reduction that adds float partials with atomics in the default mode, at engine shapes and at warp, CTA,
split and tail edges: within the float64 bound, bit-identical across reruns and while a busy kernel runs on a second
stream, and writing nothing outside its output.  Engines: two fresh engines from the same parameters and seed, three
train() calls each (the Dreamer-V3 third one a CUDA-graph replay), and the Dreamer-V3 and PPO players over ten steps:
every parameter, gradient, optimizer moment, metric, buffer and sampled state and action bit-identical; and the existing
fixture comparisons of every engine and player still pass under the switch."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    from sheeprl_b200.lib import CudaOps

    return CudaOps()


@pytest.fixture
def det(cu):
    """torch's switch on for one test (and the library with it); both restored after"""
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    cu.set_deterministic(True)
    try:
        yield cu
    finally:
        torch.use_deterministic_algorithms(was)
        cu.set_deterministic(was)


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def bits(t):
    t = t.detach()
    if t.dtype == torch.float32:
        return t.contiguous().view(torch.int32)
    if t.dtype == torch.float64:
        return t.contiguous().view(torch.int64)
    return t


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


_BUSY = {}


def busy_side_stream():
    """a long matmul chain on a second stream, launched just before the kernel under test, to shift CTA scheduling"""
    if "s" not in _BUSY:
        _BUSY["s"] = torch.cuda.Stream()
        _BUSY["x"] = torch.randn(4096, 4096, device="cuda")
    s, x = _BUSY["s"], _BUSY["x"]
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(4):
            x = x @ x * 1e-2
    return s


def fill_pool_with_nan(cu):
    rc = cu.lib.b200rl_deterministic_pool_fill(0xFF, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, cu.lib.b200rl_last_error().decode()


def check_site(cu, run, ref, rel=1e-5, bounds=None):
    """run(): launches the site on fresh (guarded) outputs, checks the guards and returns the outputs; ref: the float64
    results; bounds (optional): per-element float64 error bounds, in place of rel * (max |ref| + 1)"""
    first = run()
    for i, (g, r) in enumerate(zip(first, ref)):
        err = (g.double().cpu() - r).abs()
        if bounds is not None:
            assert bool((err <= bounds[i]).all()), (i, float((err / bounds[i]).max()))
        else:
            scale = r.abs().max().item() + 1.0
            assert err.max().item() <= rel * scale, (err.max().item(), scale)
    again = run()
    assert all(same(a, b) for a, b in zip(first, again))
    fill_pool_with_nan(cu)                     # a rerun on a NaN-filled pool: no slot is read before it is written
    again = run()
    assert all(same(a, b) for a, b in zip(first, again))
    s = busy_side_stream()
    again = run()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert all(same(a, b) for a, b in zip(first, again))


GUARD = 64


def guarded(n, dtype=torch.float32):
    """a buffer of n elements with GUARD sentinel elements before and after it"""
    buf = torch.full((n + 2 * GUARD,), 12345.0, dtype=dtype, device="cuda")
    return buf[GUARD:GUARD + n], buf


def guard_intact(buf, n):
    return bool((buf[:GUARD] == 12345.0).all()) and bool((buf[GUARD + n:] == 12345.0).all())


# ---------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("n", [1, 3, 1000, 4097, 1 << 20, 3_000_001])
def test_sumsq(det, n):
    x = rnd(n, seed=n)
    xg = x.float().cuda()
    want = (x.float().double() ** 2).sum().reshape(1)

    def run():
        out, buf = guarded(1, torch.float64)
        det.sumsq(xg, out)
        torch.cuda.synchronize()
        assert guard_intact(buf, 1)
        return [out.clone()]

    check_site(det, run, [want], rel=1e-12)


@pytest.mark.parametrize("M,C", [(1, 5), (7, 3), (100_000, 3), (70_000, 33), (4097, 64), (64 * 64 * 64, 3), (333, 1000)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_col_sum(det, M, C, accumulate):
    X = rnd(M, C, seed=M + C)
    Xg = X.float().cuda()
    base = rnd(C, seed=1)
    want = X.float().double().sum(0) + (base.float().double() if accumulate else 0)

    def run():
        out, buf = guarded(C)
        out.copy_(base.float())
        det.col_sum(Xg, out, accumulate)
        torch.cuda.synchronize()
        assert guard_intact(buf, C)
        return [out.clone()]

    check_site(det, run, [want])


@pytest.mark.parametrize("M,C", [(4096, 32), (4097, 48), (1024, 128), (333, 512), (2048, 1536), (64, 2048), (300, 100),
                                 (77, 600), (8, 1024)])
@pytest.mark.parametrize("act", [0, 1])
def test_ln_act_bwd_param_grads(det, M, C, act):
    from oracle import ln_ref

    X, dY = rnd(M, C, seed=1), rnd(M, C, seed=2)
    g, b = 1 + 0.1 * rnd(C, seed=3), 0.1 * rnd(C, seed=4)
    Xg, dYg, gg, bg = (t.float().cuda() for t in (X, dY, g, b))
    dx, dgam64, dbet64, mag = ln_ref.ln_act_bwd64(X.float(), g.float(), b.float(), 1e-3, act, dY.float())
    dx_b, pg, pb = ln_ref.ln_act_bwd_bound(X.float(), g.float(), b.float(), 1e-3, act, dY.float())
    bounds = [ln_ref.param_bound(M, mag["dgamma"], pg), ln_ref.param_bound(M, mag["dbeta"], pb), dx_b]

    def run():
        dX = torch.empty(M, C, device="cuda")
        dgam, bufg = guarded(C)
        dbet, bufb = guarded(C)
        det.ln_act_bwd(Xg, gg, bg, 1e-3, act, dYg, dX, dgam, dbet)
        torch.cuda.synchronize()
        assert guard_intact(bufg, C) and guard_intact(bufb, C)
        return [dgam.clone(), dbet.clone(), dX.clone()]

    want = [dgam64, dbet64, dx.reshape(M, C)]
    check_site(det, run, want, bounds=bounds)


@pytest.mark.parametrize("nets,M,N,K", [(1, 64, 64, 4096), (2, 256, 17, 2048), (2, 33, 7, 1000), (4, 64, 1, 8192)])
def test_bgemm_split_k(det, nets, M, N, K):
    # weight-gradient layout: C[n] = A[n]^T-view @ B[n] with long K; A rows summed into rsum
    A, B = rnd(nets, M, K, seed=1), rnd(nets, K, N, seed=2)
    Ag, Bg = A.float().cuda(), B.float().cuda()
    want = [(A.float().double() @ B.float().double()).reshape(-1), A.float().double().sum(2).reshape(-1)]

    def run():
        C, bufc = guarded(nets * M * N)
        r, bufr = guarded(nets * M)
        det.bgemm(Ag, Bg, C.view(nets, M, N), rsum=r.view(nets, M))
        torch.cuda.synchronize()
        assert guard_intact(bufc, nets * M * N) and guard_intact(bufr, nets * M)
        return [C.clone(), r.clone()]

    check_site(det, run, want, rel=1e-5)


@pytest.mark.parametrize("M,N,K,transA", [(33, 47, 5000, True), (17, 129, 3001, False), (130, 31, 2048, True)])
def test_gemm_simt_split_k(det, M, N, K, transA):
    A = rnd(K, M, seed=1) if transA else rnd(M, K, seed=1)
    B = rnd(K, N, seed=2)
    Ag, Bg = A.float().cuda(), B.float().cuda()
    want = [((A.float().double().T if transA else A.float().double()) @ B.float().double()).reshape(-1)]

    def run():
        C, buf = guarded(M * N)
        det.gemm(Ag, Bg, C.view(M, N), transA, False)
        torch.cuda.synchronize()
        assert guard_intact(buf, M * N)
        return [C.clone()]

    check_site(det, run, want, rel=1e-5)


def conv_wgrad_ref(small, big):
    """dW[cs, cb, ky, kx] of the 4x4 stride-2 pad-1 convolution big -> small, float64"""
    b = big.permute(0, 3, 1, 2)
    s = small.permute(0, 3, 1, 2)
    return torch.nn.grad.conv2d_weight(b, (s.shape[1], b.shape[1], 4, 4), s, stride=2, padding=1)


@pytest.mark.parametrize("NB,h,w,Cs,Cb", [(16, 32, 32, 32, 3), (4, 32, 32, 96, 3), (8, 16, 16, 64, 3), (3, 5, 7, 32, 1),
                                          (4, 8, 8, 24, 3), (2, 6, 6, 20, 4), (4, 8, 8, 64, 96), (2, 3, 5, 70, 33)])
def test_conv_wgrad(det, NB, h, w, Cs, Cb):
    small, big = rnd(NB, h, w, Cs, seed=1), rnd(NB, 2 * h, 2 * w, Cb, seed=2)
    sg, bg = small.float().cuda().contiguous(), big.float().cuda().contiguous()
    want = [conv_wgrad_ref(small.float().double(), big.float().double()).reshape(-1)]
    n = Cs * Cb * 16

    def run():
        dW, buf = guarded(n)
        st = torch.cuda.current_stream().cuda_stream
        # the CUDA-core route (the tensor-core route's split-K is fixed-order in both modes)
        rc = det.lib.b200rl_conv_wgrad(sg.data_ptr(), bg.data_ptr(), dW.data_ptr(), NB, h, w, Cs, Cb, 0, st)
        assert rc == 0, det.lib.b200rl_last_error().decode()
        torch.cuda.synchronize()
        assert guard_intact(buf, n)
        return [dW.clone()]

    check_site(det, run, want, rel=1e-5)


def test_mode_round_trip(cu):
    was = cu.deterministic()
    try:
        cu.set_deterministic(True)
        assert cu.deterministic()
        cu.set_deterministic(False)
        assert not cu.deterministic()
        assert cu.lib.b200rl_set_deterministic(2) != 0
    finally:
        cu.set_deterministic(was)


# ---------------------------------------------------------------------------------------------------------- engines
def snapshot(eng):
    """every tensor the engine holds, directly, in a FlatGroup (parameters, gradients, moments) or in a dict"""
    from sheeprl_b200.params import FlatGroup

    out = {}
    for k, v in sorted(vars(eng).items()):
        if isinstance(v, torch.Tensor) and v.is_cuda:
            out[k] = v.detach().clone()
        elif isinstance(v, FlatGroup):
            for f in ("flat", "grad", "exp_avg", "exp_avg_sq", "grad_avg"):
                t = getattr(v, f, None)
                if isinstance(t, torch.Tensor):
                    out[f"{k}.{f}"] = t.detach().clone()
        elif isinstance(v, dict):
            for kk, t in sorted(v.items(), key=lambda kv: str(kv[0])):
                if isinstance(t, torch.Tensor) and t.is_cuda:
                    out[f"{k}[{kk}]"] = t.detach().clone()
    return out


def assert_same_state(a, b):
    assert a.keys() == b.keys()
    # the persistent scan's workspace also holds its per-phase cycle counters (rssm_scan_profile): timings, not results
    a, b = ({k: v for k, v in d.items() if k != "_scan_ws"} for d in (a, b))
    bad = [k for k in a if not same(a[k], b[k])]
    assert not bad, bad[:10]


def outputs(o, tag):
    """the tensors a step or player call returned"""
    if isinstance(o, torch.Tensor):
        return {tag: o.detach().clone()}
    if isinstance(o, dict):
        return {k: v for kk, x in sorted(o.items(), key=lambda kv: str(kv[0])) for k, v in outputs(x, f"{tag}.{kk}").items()}
    if isinstance(o, (list, tuple)):
        return {k: v for i, x in enumerate(o) for k, v in outputs(x, f"{tag}.{i}").items()}
    return {}


def assert_reproducible(build, calls=3):
    """two fresh runs of build() -> (engine, step): `calls` steps each; every tensor the engine holds and every tensor
    a step returned bit-identical"""
    states = []
    for _ in range(2):
        eng, step = build()
        outs = {}
        for i in range(calls):
            outs.update(outputs(step(), f"call{i}"))
        torch.cuda.synchronize()
        states.append({**snapshot(eng), **outs})
        del eng, step
    assert_same_state(*states)


def dv3_graph_step(eng, data):
    def step():
        batch = {k: v.clone().float().cuda() for k, v in data.items()}
        eng.step_graph().run(lambda d: eng.train_step(d, None), batch, key=eng.graph_key())
        return eng.metrics_dict()
    return step


def test_dv3_baseline_s_three_calls_bit_identical_with_graph_replay(det):
    """BASELINE S config (the bench's): the third call is the captured graph's first replay"""
    from oracle import dv3_oracle as O
    from sheeprl_b200.configs import make_dv3_cfg
    from sheeprl_b200.engine import DV3Engine

    cfg = make_dv3_cfg("S")
    adim = (2,)
    wm, actor, critic, target = O.init_params(cfg, adim, seed=0)
    data = O.make_batch(cfg, adim, seed=2)
    engines = []

    def build():
        eng = DV3Engine(cfg, adim, in_channels=3, device="cuda:0", ops=det)
        eng.wm.load(wm), eng.actor.load(actor), eng.critic.load(critic), eng.target.load(target)
        engines.append(eng)
        return eng, dv3_graph_step(eng, data)

    assert_reproducible(build)
    for eng in engines:
        assert eng._graph is not None and len(eng._graph._entries) == 1
        assert next(iter(eng._graph._entries.values())).graph is not None
        eng.step_graph().reset()


@pytest.mark.parametrize("name", ["dv3_tiny_d", "dv3_tiny_dv"])
def test_dv3_decoupled_three_calls_bit_identical_with_graph_replay(det, name):
    from sheeprl_b200.engine import DV3Engine
    from tests.helpers import load_fixture

    fx, cfg = load_fixture(name)
    adim, cont, init = fx["actions_dim"], fx.get("is_continuous", False), fx["init"]

    def build():
        eng = DV3Engine(cfg, adim, in_channels=3, device="cuda:0", ops=det, is_continuous=cont)
        eng.wm.load(init["wm"]), eng.actor.load(init["actor"]), eng.critic.load(init["critic"])
        eng.target.load(init["target"])
        return eng, dv3_graph_step(eng, fx["data"][0])

    assert_reproducible(build)


def test_p2e_exploration_three_calls_bit_identical(det):
    from tests.test_p2e_cpu import load, make_engine

    fx, cfg = load()
    data = {k: v.clone().float().cuda() for k, v in fx["data"][0].items()}

    def build():
        eng = make_engine(fx, cfg, device="cuda", ops=det)
        return eng, lambda: (eng.train_step({k: v.clone() for k, v in data.items()}, None), eng.metrics_dict())[1]

    assert_reproducible(build)


@pytest.mark.parametrize("name", ["ppo_vector", "ppo_pixel", "ppo_tanh_ln"])
def test_ppo_three_calls_bit_identical(det, name):
    from tests.test_ppo_cpu import load, make_engine

    fx = load(name)
    data = {k: v.cuda() for k, v in fx["data"].items()}

    def build():
        eng = make_engine(fx, device="cuda", ops=det)
        return eng, lambda: eng.train(data, fx["index_batches"]) or eng.losses

    assert_reproducible(build)


def test_recurrent_ppo_three_calls_bit_identical(det):
    from tests.test_ppo_recurrent_cpu import NAMES, load, make_engine

    for name in NAMES:
        fx = load(name)
        data = {k: v.cuda() for k, v in fx["data"].items()}

        def build():
            eng = make_engine(fx, device="cuda", ops=det)
            return eng, lambda: eng.train(data, fx["index_batches"]) or eng.losses

        assert_reproducible(build)


@pytest.mark.parametrize("name", ["a2c_vector", "a2c_pixel"])
def test_a2c_three_calls_bit_identical(det, name):
    from tests.test_a2c_cpu import build as build_a2c, load

    r = load(name)[0]
    c = r["calls"][0]
    data = {k: v.cuda() for k, v in c["data"].items()}

    def build():
        agent, _, _ = build_a2c(r, "cuda", det)
        eng = agent._b200_engine
        return eng, lambda: eng.train(data, c["index_batches"]) or eng.losses

    assert_reproducible(build)


def test_sac_three_calls_bit_identical(det):
    from oracle import sac_oracle as SO
    from sheeprl_b200.algos.sac.engine import SACEngine

    O, A, H, B = 17, 6, 256, 256
    opt = {"lr": 3e-4, "eps": 1e-4, "betas": (0.9, 0.999)}
    P = SO.init_params(O, A, H, 2, seed=0)
    data = {k: v.cuda() for k, v in SO.make_batch(B, O, A, seed=1).items()}

    def build():
        eng = SACEngine(O, A, H, H, 2, B, 0.99, 0.005, 1.0, -1.0, 1.0, opt, opt, opt, "cuda", det)
        eng.load_reference_state(P["actor"], P["qf"], P["qf_target"], P["log_alpha"]["log_alpha"])
        return eng, lambda: eng.train_step(data, True) or eng.metrics_dict()

    assert_reproducible(build)


@pytest.mark.parametrize("name", ["droq_tiny", "droq_exp"])
def test_droq_three_calls_bit_identical(det, name):
    from tests.test_droq_cpu import call_inputs, load, make_engine

    fx = load(name)
    critic, actor_obs = call_inputs(fx, 0)[:2]
    critic = {k: v.cuda() for k, v in critic.items()}
    actor_obs = actor_obs.cuda()

    def build():
        eng = make_engine(fx, device="cuda", ops=det)
        return eng, lambda: eng.train_call(critic, actor_obs) or eng.metrics_dict()      # device-drawn noise and masks

    assert_reproducible(build)


def test_dv3_player_ten_steps_bit_identical(det):
    from sheeprl_b200.algos.dreamer_v3.player import PlayerDV3
    from sheeprl_b200.engine import DV3Engine
    from tests.helpers import load_fixture

    tf, cfg = load_fixture("dv3_tiny_a")
    g = torch.Generator().manual_seed(3)
    obs = [torch.randint(0, 256, (1, 4, 3, 64, 64), dtype=torch.uint8, generator=g).cuda() for _ in range(10)]

    def build():
        eng = DV3Engine(cfg, tf["actions_dim"], in_channels=3, device="cuda", ops=det)
        eng.wm.load(tf["init"]["wm"]), eng.actor.load(tf["init"]["actor"])
        player = PlayerDV3(eng, 4)
        player.init_states()
        it = iter(obs)
        return player, lambda: (player.get_actions({"rgb": next(it)}), player.recurrent_state, player.stochastic_state)

    assert_reproducible(build, calls=10)


@pytest.mark.parametrize("name", ["ppo_pixel", "ppo_continuous"])
def test_ppo_player_ten_steps_bit_identical(det, name):
    import os

    from oracle.make_golden_ppo import split_obs
    from sheeprl_b200.algos.ppo.agent import PPOPlayer
    from tests.test_ppo_cpu import GOLDEN, load, make_engine

    fx = load(name)
    pf = torch.load(os.path.join(GOLDEN, "ppo_player.pt"), weights_only=False)[name]
    obs = split_obs(fx["spec"], {k: v.cuda() for k, v in pf["obs"].items()})

    def build():
        player = PPOPlayer(make_engine(fx, device="cuda", ops=det))
        return player, lambda: (player(obs), player.get_actions(obs))                   # device-drawn noise

    assert_reproducible(build, calls=10)


# the existing fixture comparisons, re-run with torch's switch on
@pytest.mark.parametrize("name", ["dv3_tiny_a", "dv3_tiny_b", "dv3_tiny_c", "dv3_tiny_v", "dv3_tiny_vo", "dv3_tiny_mk", "dv3_tiny_h0"])
def test_dv3_fixture_under_switch(det, name):
    from tests.test_gpu_engine import test_engine_cuda_matches_reference_fixture

    test_engine_cuda_matches_reference_fixture(name)


@pytest.mark.parametrize("name", ["dv3_tiny_d", "dv3_tiny_dv"])
def test_dv3_decoupled_fixture_under_switch(det, name):
    from tests.test_gpu_dv3_decoupled import test_engine_cuda_matches_decoupled_reference_fixture

    test_engine_cuda_matches_decoupled_reference_fixture(name)


def test_p2e_fixture_under_switch(det):
    from tests import test_gpu_p2e as T

    T.test_engine_matches_reference(det)
    T.test_public_api_matches_reference(det)


@pytest.mark.parametrize("name", ["ppo_vector", "ppo_branches", "ppo_continuous", "ppo_pixel", "ppo_tanh_ln", "ppo_multikey"])
def test_ppo_fixture_under_switch(det, name):
    from tests.test_ppo_cpu import check_engine, load, make_engine

    fx = load(name)
    check_engine(fx, make_engine(fx, device="cuda", ops=det), name, uint8_image=True)


def test_recurrent_ppo_fixture_under_switch(det):
    from tests import test_gpu_ppo_recurrent as T
    from tests.test_ppo_recurrent_cpu import NAMES

    for name in NAMES:
        T.test_engine_matches_reference(det, name)
        T.test_player_matches_reference(det, name)


@pytest.mark.parametrize("name", ["sac_tiny", "sac_c4"])
def test_sac_fixture_under_switch(det, name):
    from tests.test_sac_cpu import check_engine, load, make_engine

    fx = load(name)
    check_engine(fx, make_engine(fx, device="cuda", ops=det), name)


@pytest.mark.parametrize("name", ["droq_tiny", "droq_tiny_p0", "droq_exp"])
def test_droq_fixture_under_switch(det, name):
    from tests.test_gpu_droq import test_engine_matches_reference

    test_engine_matches_reference(det, name)


@pytest.mark.parametrize("name", ["a2c_vector", "a2c_branches", "a2c_continuous", "a2c_pixel"])
def test_a2c_fixture_under_switch(det, name):
    from tests.test_a2c_cpu import check_engine

    check_engine(name, device="cuda", ops=det, uint8_image=True)


def test_players_fixture_under_switch(det):
    from tests import test_gpu_player as DP
    from tests import test_gpu_ppo as PP

    for name in ("dv3_player_discrete", "dv3_player_continuous", "dv3_player_vector", "dv3_player_vector_only"):
        DP.test_player_matches_reference(det, name, True)
    for name in ("ppo_branches", "ppo_continuous", "ppo_pixel", "ppo_tanh_ln", "ppo_multikey"):
        PP.test_player_matches_reference(det, name, True)


def test_default_mode_untouched_by_the_switch_off(cu):
    """with torch's switch off, an engine call puts the library back in the default mode"""
    from sheeprl_b200.lib import sync_deterministic

    assert not torch.are_deterministic_algorithms_enabled()
    cu.set_deterministic(True)
    assert sync_deterministic(cu) is False
    assert not cu.deterministic()
