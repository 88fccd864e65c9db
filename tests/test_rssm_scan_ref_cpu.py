"""CPU validation of the float64 scan reference (oracle/rssm_scan_ref.py) that the persistent RSSM scan kernels are
tested against: driven by the samples of the engine's per-step scan on the executable op specification
(oracle/ops_emul.py), it must reproduce that scan's saved activations and its five BPTT gradients to fp32 accuracy."""
import pytest
import torch

from oracle import dv3_oracle as O
from oracle.ops_emul import EmulOps
from oracle.rssm_scan_ref import ACT_KEYS, GRAD_KEYS, scan_reference
from sheeprl_b200.configs import make_dv3_cfg
from sheeprl_b200.engine import DV3Engine
from tests.helpers import load_fixture

RTOL = 2e-5     # fp32 per-step ops against float64, relative to each tensor's largest magnitude


def scan_first(T, B, g):
    """is_first patterns the scan must honour: rows that do not start a sequence at t = 0 (they start from zeros), ~10 %
    resets mid-sequence, one step at which every row resets and one row that resets at every step"""
    first = (torch.rand(T, B, generator=g) < 0.1).float()
    first[0, : B // 2] = 1.0
    first[T // 2] = 1.0
    first[:, B - 1] = 1.0
    return first.reshape(-1)


def run_per_step_scan(cfg, adim, seed):
    """DV3Engine's per-step scan and BPTT (EmulOps has no fused scan op) on seeded inputs; the prior's KL gradient is
    zero so that the recurrence's only gradient inputs are d_latent and d_post_mix"""
    g = torch.Generator().manual_seed(seed)
    wm, actor, critic, target = O.init_params(cfg, adim, seed=seed)
    for v in wm.values():
        v.add_(torch.randn(v.shape, generator=g) * 0.05)
    eng = DV3Engine(cfg, adim, in_channels=3, device="cpu", ops=EmulOps())
    eng.wm.load(wm)
    T, B, Z = eng.T, eng.B, eng.Z
    first = scan_first(T, B, g)
    eng.pe.copy_(torch.randn(eng.pe.shape, generator=g))
    eng.shift_actions.copy_(torch.randn(eng.shift_actions.shape, generator=g))
    eng.noise_post.copy_(torch.empty(eng.noise_post.shape).exponential_(generator=g))
    eng._scan_forward(first)
    eng.d_latent.copy_(torch.randn(eng.d_latent.shape, generator=g) * 0.1)
    eng.d_post_mix.copy_(torch.randn(eng.d_post_mix.shape, generator=g) * 0.1)
    eng.d_prior_mix.zero_()
    d_latent, d_post_mix = eng.d_latent.clone(), eng.d_post_mix.clone()
    eng._scan_backward(first)
    return eng, first, d_latent, d_post_mix


def tiny_b():
    cfg = make_dv3_cfg("S", per_rank_batch_size=5, per_rank_sequence_length=7, horizon=2, dense_units=40,
                       mlp_layers=1, cnn_channels_multiplier=2, recurrent_state_size=36, hidden_size=28,
                       stochastic_size=3, discrete_size=7, bins=15)
    return cfg, (4,)


@pytest.mark.parametrize("name", ["dv3_tiny_a", "tiny_b"])
def test_scan_reference_reproduces_per_step_scan(name):
    if name == "tiny_b":
        cfg, adim = tiny_b()
    else:
        fx, cfg = load_fixture(name)
        adim = fx["actions_dim"]
    eng, first, d_latent, d_post_mix = run_per_step_scan(cfg, adim, seed=7)
    dims, tensors = eng._scan_dims(), eng._scan_tensors(first)
    ref = scan_reference(dims, eng.eps, eng.unimix, tensors, d_latent=d_latent, d_post_mix=d_post_mix)
    got = {k: getattr(eng, k) for k in ACT_KEYS if k != "h"} | {"h": eng.latent[:, eng.Z:]}
    got |= {k: getattr(eng, k) for k in GRAD_KEYS}
    for k in ACT_KEYS + GRAD_KEYS:
        want = ref[k]
        err = float((got[k].double() - want).abs().max())
        assert err <= RTOL * float(want.abs().max()), (k, err, float(want.abs().max()))
    # the engine sampled with the same rule: its pick is the reference's argmax of p / q wherever that is not a near-tie
    s = ref["scores"]
    picked = eng.latent[:, : eng.Z].reshape(s.shape).argmax(-1)
    top = s.topk(2, -1).values
    clear = top[..., 0] > top[..., 1] * (1 + 1e-4)
    assert torch.equal(picked[clear], s.argmax(-1)[clear])
    # one-step mode from the engine's own chain inputs gives the same activations
    one = scan_reference(dims, eng.eps, eng.unimix, tensors, one_step=True)
    for k in ACT_KEYS:
        assert float((one[k] - ref[k]).abs().max()) <= RTOL * float(ref[k].abs().max()), k
