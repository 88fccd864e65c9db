"""TEST INFRASTRUCTURE (oracle) — NOT part of the product path.

Float64 reference of the persistent RSSM scan (`b200rl_rssm_scan_fwd` / `b200rl_rssm_scan_bwd`, include/b200rl.h):
the posterior recurrence of RSSM.dynamic over T steps and its BPTT, written with the oracle's pinned building blocks
(`recurrent_step`, `layer_norm`, `unimix_logits`, `st_sample`, all checked against the executed reference by
tests/test_oracle_golden.py) instead of new formulas.

It takes the same `dims` / `tensors` dictionaries as `CudaOps.rssm_scan_fwd` (any device; copies are promoted to float64
on the CPU).  It is TEACHER-FORCED: the one-hot sample of every step is read from the kernel's own `latent[:, :Z]`, so
an fp32-versus-float64 near-tie cannot fork the trajectory.  The reference's own sampling scores `p / noise` are
returned so that a test can check that the kernel's pick is an argmax.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import dv3_oracle as O

Tensor = torch.Tensor
ACT_KEYS = ("x_pre", "x_act", "g_pre", "g_ln", "h", "rp_pre", "rp_act", "post_raw", "post_mix")
GRAD_KEYS = ("d_post_raw", "d_rp_act", "d_g_ln", "d_x_act", "d_h0")


def scan_reference(dims: Dict[str, int], eps: float, unimix: float, tensors: Dict[str, Tensor], one_step: bool = False,
                   d_latent: Optional[Tensor] = None, d_post_mix: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """Returns the saved activations (`ACT_KEYS`, [T*B, width] float64), `scores` ([T*B, S, D]: normalised unimix
    probabilities over the Exp(1) noise, the sampling rule argmax(p / q)) and, when `d_latent` [T*B, >= Z+R] and
    `d_post_mix` [T*B, Z] are given, the gradients `GRAD_KEYS` of  L = <d_latent, latent> + <d_post_mix, post_mix>
    (float64 autograd, straight-through sample one-hot + p - p.detach(); z0 gets no gradient).

    one_step: every step starts from the kernel's own `z_in`, `h_in` and `a_in` instead of the reference's carried
    state, so fp32 error does not build up over T (forward only)."""
    T, B, S, D, R, A, Dr = (int(dims[k]) for k in ("T", "B", "S", "D", "R", "A", "Dr"))
    Z = S * D
    want_grad = d_latent is not None
    assert not (want_grad and one_step), "gradients are defined on the carried chain"

    def f64(name, *shape):
        return tensors[name].detach().to("cpu", torch.float64).reshape(*shape)

    p, pr = "rssm.recurrent_model.", "rssm.representation_model._model."
    wm = {p + "mlp._model.0.weight": f64("W_in", -1, Z + A), p + "mlp._model.1.weight": f64("lnx_g", -1),
          p + "mlp._model.1.bias": f64("lnx_b", -1), p + "rnn.linear.weight": f64("W_g", 3 * R, -1),
          p + "rnn.layer_norm.weight": f64("lng_g", -1), p + "rnn.layer_norm.bias": f64("lng_b", -1)}
    # every activation of every step is a graph node (also at t = 0, where the chain inputs are constants)
    wm[p + "mlp._model.0.weight"].requires_grad_(want_grad)
    Wr1 = f64("W_r1", Dr, -1)[:, :R]
    lnr_g, lnr_b, W_r2, b_r2 = f64("lnr_g", -1), f64("lnr_b", -1), f64("W_r2", Z, Dr), f64("b_r2", -1)
    first = f64("first", T, B, 1)
    actions = f64("actions", T, B, A)
    pe = f64("pe", T, B, Dr)
    noise = f64("noise", T, B, S, D)
    z_kernel = f64("latent", T, B, -1)[..., :Z]
    h0 = f64("h0", R).requires_grad_(want_grad)
    z0 = f64("z0", Z)
    if one_step:
        z_in_k, h_in_k, a_in_k = f64("z_in", T, B, Z), f64("h_in", T, B, R), f64("a_in", T, B, A)

    out = {k: [] for k in ACT_KEYS + ("scores", "z")}
    h = torch.zeros(B, R, dtype=torch.float64)
    z = torch.zeros(B, Z, dtype=torch.float64)
    for t in range(T):
        f = first[t]
        if one_step:
            z_in, h_in, a_in = z_in_k[t], h_in_k[t], a_in_k[t]
        else:
            a_in = (1 - f) * actions[t]
            h_in = (1 - f) * h + f * h0
            z_in = (1 - f) * z + f * z0
        sv = {}
        h = O.recurrent_step(wm, z_in, a_in, h_in, eps, saves=sv)
        rp_pre = pe[t] + h @ Wr1.t()
        rp_act = F.silu(O.layer_norm(rp_pre, lnr_g, lnr_b, eps))
        post_raw = F.linear(rp_act, W_r2, b_r2)
        post_mix = O.unimix_logits(post_raw, S, D, unimix)
        st = O.st_sample(post_mix, S, D, noise[t])
        z = z_kernel[t] + (st - st.detach())             # the kernel's one-hot, the reference's straight-through term
        _, probs = O.categorical_normalise(post_mix.detach().reshape(B, S, D))
        for k, v in (("h", h), ("rp_pre", rp_pre), ("rp_act", rp_act), ("post_raw", post_raw), ("post_mix", post_mix),
                     ("scores", probs / noise[t]), ("z", z)) + tuple(sv.items()):
            if want_grad and k in ("x_act", "g_ln", "rp_act", "post_raw"):
                v.retain_grad()
            out[k].append(v)

    res = {k: torch.cat([v.detach() for v in out[k]], 0) for k in ACT_KEYS + ("scores",)}
    if want_grad:
        dl = d_latent.detach().to("cpu", torch.float64).reshape(T, B, -1)
        dm = d_post_mix.detach().to("cpu", torch.float64).reshape(T, B, Z)
        loss = sum((dl[t, :, :Z] * out["z"][t]).sum() + (dl[t, :, Z:Z + R] * out["h"][t]).sum()
                   + (dm[t] * out["post_mix"][t]).sum() for t in range(T))
        loss.backward()
        for k in ("post_raw", "rp_act", "g_ln", "x_act"):
            res["d_" + k] = torch.cat([v.grad for v in out[k]], 0)
        res["d_h0"] = h0.grad
    return res
