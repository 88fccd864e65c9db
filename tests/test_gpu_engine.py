"""End-to-end parity of the CUDA engine (every op through the C-ABI) on an H100:
  * against the committed reference fixtures (tests/golden, produced by the unmodified reference train());
  * against the oracle on the BASELINE config (S, B=16, T=64, H=15), incl. gradients;
  * size-independent properties at full size (finite, deterministic replay, sample one-hotness)."""

import pytest
import torch

from tests.helpers import assert_params_close, load_fixture, oracle_run

pytestmark = pytest.mark.gpu


def to_cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else [x.cuda() for x in v]) for k, v in d.items()}


def make_engine(cfg, adim, init, is_continuous=False):
    from sheeprl_b200.engine import DV3Engine

    from tests.helpers import image_channels

    eng = DV3Engine(cfg, adim, in_channels=image_channels(cfg), device="cuda", is_continuous=is_continuous)
    eng.wm.load(init["wm"]), eng.actor.load(init["actor"]), eng.critic.load(init["critic"])
    eng.target.load(init["target"])
    return eng


PER_TENSOR_RTOL = 1e-4      # north_star: 1e-4 fp32 tolerance, applied to every gradient tensor separately (l2 norms)


def check_grads(eng_grads, o_out, cfg, rtol):
    for grp, max_norm, nm in (("wm", cfg.algo.world_model.clip_gradients, "world_model"),
                              ("actor", cfg.algo.actor.clip_gradients, "actor"),
                              ("critic", cfg.algo.critic.clip_gradients, "critic")):
        og = o_out[f"grads/{grp}"]
        coef = min(1.0, max_norm / (float(o_out["Grads/" + nm]) + 1e-6))
        gmax = max(float(v.abs().max()) for v in og.values())
        gnorm = float(torch.sqrt(sum((v.double() ** 2).sum() for v in og.values())))
        worst = []
        for k, v in og.items():
            diff = eng_grads[grp][k].cpu() * coef - v
            d = float(diff.abs().max())
            assert d <= rtol * max(gmax, 1e-12) + 1e-9, (grp, k, d, gmax)
            # per-tensor: a small-magnitude tensor (LayerNorm bias, initial_recurrent_state) must be right on its OWN scale,
            # not only against the largest gradient of its group.  Floor: 1e-6 of the group's norm (below that a gradient
            # is rounding noise of the products that feed it).
            rel = float(diff.double().norm()) / (float(v.double().norm()) + 1e-6 * gnorm + 1e-30)
            worst.append((rel, k))
        worst.sort(reverse=True)
        assert worst[0][0] <= PER_TENSOR_RTOL, (grp, "per-tensor relative gradient error", worst[:5])


@pytest.mark.parametrize("name", ["dv3_tiny_a", "dv3_tiny_b", "dv3_tiny_c", "dv3_tiny_v", "dv3_tiny_vo", "dv3_tiny_mk", "dv3_tiny_h0"])
def test_engine_cuda_matches_reference_fixture(name):
    """dv3_tiny_c: continuous actions, policy gradient through the imagined rollout; dv3_tiny_v / _vo: vector observations
    (MLP encoder / decoder) next to / instead of the image"""
    fx, cfg = load_fixture(name)
    adim = fx["actions_dim"]
    steps = len(fx["data"])
    cont = fx.get("is_continuous", False)
    fdata = [{k: v.float() for k, v in d.items()} for d in fx["data"]]
    st, o_outs, ms, _ = oracle_run(cfg, adim, fx["init"], fdata, fx["noise"], steps, keep=True, is_continuous=cont)
    eng = make_engine(cfg, adim, fx["init"], cont)
    for s in range(steps):
        batch = {k: v.clone().float().cuda() for k, v in fx["data"][s].items()}
        eng.train_step(batch, to_cuda(fx["noise"][s]))
        if s == 0:
            grads = {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")}
            check_grads(grads, o_outs[0], cfg, 3e-5)
        got = {k: float(v) for k, v in eng.metrics_dict().items()}
        for k, v in fx["metrics"][s].items():
            assert got[k] == pytest.approx(v, rel=1e-4, abs=1e-6), (s, k)
    lrs = {"wm": 1e-4, "actor": 8e-5, "critic": 8e-5}
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        assert_params_close({k: v.cpu() for k, v in g.views.items()}, fx["after"][n], lrs[n], steps, tol=3e-6, label=n)
    assert float(eng.moments_state[0]) == pytest.approx(float(fx["moments"]["low"]), rel=1e-4, abs=1e-7)
    assert float(eng.moments_state[1]) == pytest.approx(float(fx["moments"]["high"]), rel=1e-4, abs=1e-7)


def test_engine_cuda_baseline_config_vs_oracle_and_reference_digest():
    """BASELINE.json configs[1]: Dreamer-V3 S, 64x64x3, bs16 seq64 horizon15.  Tolerance 1e-4 (north_star)."""
    from oracle import dv3_oracle as O
    from oracle.make_golden import perturbed_oracle_init, subsample

    fx, cfg = load_fixture("dv3_S_digest")
    adim = fx["actions_dim"]
    a, w = cfg.algo, cfg.algo.world_model
    init = perturbed_oracle_init(cfg, adim, fx["init_seed"], fx["perturb"])
    data = [O.make_batch(cfg, adim, seed=fx["data_seed"])]
    noise = [O.draw_noise(a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon, w.stochastic_size,
                          w.discrete_size, adim, seed=fx["noise_seed"])]
    st, o_outs, ms, _ = oracle_run(cfg, adim, init, data, noise, 1, condition_margin=1e-3, keep=True)
    eng = make_engine(cfg, adim, init)
    batch = {k: v.clone().cuda() for k, v in data[0].items()}
    batch["rgb"] = batch["rgb"].to(torch.uint8)          # uint8 fast path (values are integral)
    eng.train_step(batch, to_cuda(noise[0]))
    torch.cuda.synchronize()
    # intermediates named in SURVEY.md §8a
    N = eng.N
    assert torch.equal(eng.latent[:, : eng.Z].cpu().reshape(o_outs[0]["latent"][..., : eng.Z].shape),
                       o_outs[0]["latent"][..., : eng.Z].round()), "posterior samples differ"
    for nm, got, want in (("h", eng.latent[:, eng.Z:], o_outs[0]["latent"][..., eng.Z:].reshape(N, -1)),
                          ("post_logits", eng.post_mix, o_outs[0]["post_logits"].reshape(N, -1)),
                          ("prior_logits", eng.prior_mix, o_outs[0]["prior_logits"].reshape(N, -1)),
                          ("emb", eng.emb, o_outs[0]["emb"].reshape(N, -1)),
                          ("lambda", eng.lam, o_outs[0]["lambda_values"].squeeze(-1)),
                          ("values", eng.values, o_outs[0]["values"].squeeze(-1)),
                          ("discount", eng.discount, o_outs[0]["discount"].squeeze(-1))):
        err = float((got.cpu() - want).abs().max())
        assert err <= 1e-4 * max(1.0, float(want.abs().max())), (nm, err)
    assert torch.equal(eng.actions.cpu(), o_outs[0]["imagined_actions"].round()), "imagined actions differ"
    assert torch.equal(eng.traj[:, :, : eng.Z].cpu(), o_outs[0]["traj"][:, :, : eng.Z].round()), "imagined states differ"
    grads = {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")}
    check_grads(grads, o_outs[0], cfg, 1e-4)
    got = {k: float(v) for k, v in eng.metrics_dict().items()}
    for k, v in fx["metrics"][0].items():                 # numbers produced by the REAL reference
        assert got[k] == pytest.approx(v, rel=1e-4, abs=1e-6), k
    for n, g in (("wm", eng.wm), ("actor", eng.actor), ("critic", eng.critic)):
        sub = {k: subsample(v.cpu()) for k, v in g.views.items()}
        assert_params_close(sub, fx["after_sub"][n], 1e-4, 1, tol=3e-6, frac=5e-3, label=n)
        assert_params_close({k: v.cpu() for k, v in g.views.items()}, st[n], 1e-4, 1, tol=3e-6, frac=2e-3, label=n)


def test_engine_cuda_full_size_properties():
    """Size-independent properties at the BASELINE config with on-device Philox noise."""
    from oracle import dv3_oracle as O
    from sheeprl_b200.configs import make_dv3_cfg

    cfg = make_dv3_cfg("S")
    adim = (2,)
    wm, actor, critic, target = O.init_params(cfg, adim, seed=0)
    init = {"wm": wm, "actor": actor, "critic": critic, "target": target}
    data = O.make_batch(cfg, adim, seed=3, as_uint8=True)
    runs = []
    for rep in range(2):
        eng = make_engine(cfg, adim, init)
        eng.rng_seed = 99
        first_traj = None
        for s in range(2):
            eng.train_step({k: v.clone().cuda() for k, v in data.items()}, None)
            if s == 0:
                first_traj = eng.traj[:, :, : eng.Z].clone().cpu()
        torch.cuda.synchronize()
        runs.append((eng.metrics.clone().cpu(), first_traj))
        z = eng.traj[:, :, : eng.Z].reshape(-1, eng.S, eng.D)
        assert torch.all(z.sum(-1) == 1) and torch.all((z == 0) | (z == 1)), "states are not one-hot per group"
        assert torch.isfinite(eng.metrics).all() and torch.isfinite(eng.wm.flat).all()
        assert torch.isfinite(eng.actor.flat).all() and torch.isfinite(eng.critic.flat).all()
        d = eng.discount
        assert torch.all(d[1:] <= d[:-1] + 1e-6), "discount must be non-increasing along the horizon"
    # same Philox seed -> same samples up to exact near-ties (fp32 atomics make sums order-dependent at 1e-7)
    a0 = runs[0][1].reshape(-1, 32, 32).argmax(-1)
    a1 = runs[1][1].reshape(-1, 32, 32).argmax(-1)
    assert float((a0 != a1).float().mean()) < 2e-3
    assert float((runs[0][0] - runs[1][0]).abs().max()) <= 2e-3 * float(runs[0][0].abs().max())


SCAN_MODELS = {
    "S": dict(size="S"),
    "XS": dict(size="XS"),
    # two 4-column groups per CTA in the GRU and x layers, forward and backward fused
    "wide_mh2": dict(size="S", per_rank_sequence_length=6, horizon=3, dense_units=520, recurrent_state_size=520,
                     hidden_size=64, stochastic_size=8, discrete_size=8, mlp_layers=1, cnn_channels_multiplier=4),
    # the forward fits in shared memory, the backward does not: fused forward, per-step BPTT over its saves
    "mixed_bwd": dict(size="S", per_rank_batch_size=8, per_rank_sequence_length=6, horizon=3, dense_units=128,
                      recurrent_state_size=768, hidden_size=128, stochastic_size=16, discrete_size=16, mlp_layers=1,
                      cnn_channels_multiplier=4),
}


@pytest.mark.parametrize("name", ["dv3_tiny_a", "dv3_tiny_b", "S", "XS", "wide_mh2", "mixed_bwd"])
def test_fused_scan_equals_per_step_scan(name):
    """Persistent cooperative RSSM kernels (csrc/rssm_scan.cu, forward + BPTT) vs the per-step kernels:
    same saved activations, same world-model gradients."""
    from oracle import dv3_oracle as O
    from sheeprl_b200.configs import make_dv3_cfg

    if name in SCAN_MODELS:
        cfg, adim = make_dv3_cfg(**SCAN_MODELS[name]), (2,)
        wm, actor, critic, target = O.init_params(cfg, adim, seed=0)
        g = torch.Generator().manual_seed(3)
        for v in wm.values():
            v.add_(torch.randn(v.shape, generator=g) * 0.02)
        init = {"wm": wm, "actor": actor, "critic": critic, "target": target}
        data = O.make_batch(cfg, adim, seed=4)
        a, w = cfg.algo, cfg.algo.world_model
        noise = O.draw_noise(a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon, w.stochastic_size,
                             w.discrete_size, adim, seed=5)
        oracle_run(cfg, adim, init, [data], [noise], 1, condition_margin=1e-3)   # removes near-tie draws in place
    else:
        fx, cfg = load_fixture(name)
        adim, init, data, noise = fx["actions_dim"], fx["init"], fx["data"][0], fx["noise"][0]
    outs = []
    for fused in (False, True):
        eng = make_engine(cfg, adim, init)
        eng.fused_scan = fused
        eng.train_step({k: v.clone().float().cuda() for k, v in data.items()}, to_cuda(noise))
        torch.cuda.synchronize()
        if fused:
            assert eng.fused_scan, "fused scan was disabled"
            if name == "mixed_bwd":
                assert not eng.fused_scan_bwd, "the backward kernel should not fit this model"
            else:
                assert eng.fused_scan_bwd, "fused backward scan was disabled"
            assert eng.ops.rssm_scan_error(eng._scan_ws) == 0, "a hand-off of the persistent scan timed out"
        outs.append({k: getattr(eng, k).clone() for k in (
            "latent", "z_in", "h_in", "a_in", "x_pre", "x_act", "g_pre", "g_ln", "tr_pre", "tr_act", "rp_pre", "rp_act",
            "post_raw", "prior_raw", "post_mix", "prior_mix", "d_post_raw", "d_prior_raw", "d_rp_pre", "d_tr_pre",
            "d_g_pre", "d_x_pre", "d_rp_act", "d_tr_act", "d_g_ln", "d_x_act", "d_h0")}
            | {"wm_grad": eng.wm.grad.clone(), "metrics": eng.metrics.clone()})
    ref, got = outs
    Z = ref["z_in"].shape[1]
    assert torch.equal(ref["latent"][:, :Z], got["latent"][:, :Z]), "sampled posteriors differ"
    for k in ref:
        err = float((ref[k] - got[k]).abs().max())
        assert err <= 5e-5 * max(1e-3, float(ref[k].abs().max())), (k, err, float(ref[k].abs().max()))


def test_engine_cuda_xl_widths_vs_oracle():
    """BASELINE.json configs[4] model (Dreamer-V3 XL: 5 MLP layers, dense 1024, R=4096, conv 96/192/384/768) on a
    short batch (B=2, T=4, H=3): the per-step scan path (weights exceed the persistent kernel's shared memory), the
    tensor-core GEMM / conv paths at XL widths and every gradient against the oracle, 1e-4."""
    from oracle import dv3_oracle as O
    from oracle.make_golden import perturbed_oracle_init
    from sheeprl_b200.configs import make_dv3_cfg

    cfg = make_dv3_cfg("XL", per_rank_batch_size=2, per_rank_sequence_length=4, horizon=3)
    adim = (3,)
    a, w = cfg.algo, cfg.algo.world_model
    init = perturbed_oracle_init(cfg, adim, 21, 0.02)
    data = [O.make_batch(cfg, adim, seed=22)]
    noise = [O.draw_noise(a.per_rank_sequence_length, a.per_rank_batch_size, a.horizon, w.stochastic_size,
                          w.discrete_size, adim, seed=23)]
    st, o_outs, ms, _ = oracle_run(cfg, adim, init, data, noise, 1, condition_margin=1e-3, keep=True)
    eng = make_engine(cfg, adim, init)
    batch = {k: v.clone().cuda() for k, v in data[0].items()}
    eng.train_step(batch, to_cuda(noise[0]))
    torch.cuda.synchronize()
    assert not eng.fused_scan                               # XL falls back to the per-step kernels
    N = eng.N
    assert torch.equal(eng.latent[:, : eng.Z].cpu().reshape(o_outs[0]["latent"][..., : eng.Z].shape),
                       o_outs[0]["latent"][..., : eng.Z].round()), "posterior samples differ"
    for nm, got, want in (("h", eng.latent[:, eng.Z:], o_outs[0]["latent"][..., eng.Z:].reshape(N, -1)),
                          ("lambda", eng.lam, o_outs[0]["lambda_values"].squeeze(-1))):
        err = float((got.cpu() - want).abs().max())
        assert err <= 1e-4 * max(1.0, float(want.abs().max())), (nm, err)
    grads = {g: {k: v.clone() for k, v in getattr(eng, g).gviews.items()} for g in ("wm", "actor", "critic")}
    check_grads(grads, o_outs[0], cfg, 1e-4)
    got = {k: float(v) for k, v in eng.metrics_dict().items()}
    for k in got:
        # Grads/*: torch's fp32 CPU norm over 1e8-element tensors is itself only good to ~6e-4 here (the double-
        # precision norm of the ORACLE's own gradients equals the kernel's 7844.57, torch reports 7839.71), so the
        # logged norms are compared at 1e-3; every gradient tensor was compared at 1e-4 above.
        tol = 1e-3 if k.startswith("Grads/") else 1e-4
        assert got[k] == pytest.approx(float(o_outs[0][k]), rel=tol, abs=1e-6), k
