"""TEST INFRASTRUCTURE (oracle) — NOT part of the product path.

Float64 reference of the GRU-only scan of the decoupled RSSM (`b200rl_gru_scan_fwd` / `b200rl_gru_scan_bwd`,
include/b200rl.h), written with the oracle's pinned `layer_norm` and the gate of `recurrent_step`.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle import dv3_oracle as O

Tensor = torch.Tensor


def gru_scan_reference(dims: Dict[str, int], eps: float, tensors: Dict[str, Tensor], x_share: Tensor, one_step: bool = False,
                       d_latent: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """Per step h_in = (1-f) h_{t-1} + f h0, g_pre = x_share + h_in W_g[:, :R]^T, g_ln = LN(g_pre), the gate of
    LayerNormGRUCell (models.py:396-403).  Same `dims` / `tensors` as `CudaOps.gru_scan_fwd`; `x_share` [T*B, 3R] is
    what `g_pre` held on entry.  Returns g_pre, g_ln, h_in, h ([T*B, width]) and, with `d_latent` [T*B, ld_lat], the
    gradients d_g_ln and d_h0 of L = <d_latent[:, h columns], h> (float64 autograd).
    one_step: every step starts from the kernel's own `h_in`, so fp32 error does not build up over T (forward only)."""
    T, B, R = (int(dims[k]) for k in ("T", "B", "R"))
    off = int(dims["lat_off"])
    want_grad = d_latent is not None
    assert not (want_grad and one_step), "gradients are defined on the carried chain"

    def f64(t, *shape):
        return t.detach().to("cpu", torch.float64).reshape(*shape)

    Wh = f64(tensors["W_g"], 3 * R, -1)[:, :R]
    gam, bet = f64(tensors["lng_g"], -1), f64(tensors["lng_b"], -1)
    h0 = f64(tensors["h0"], R).requires_grad_(want_grad)
    first = f64(tensors["first"], T, B, 1)
    xs = f64(x_share, T, B, 3 * R)
    h_in_k = f64(tensors["h_in"], T, B, R)
    h = torch.zeros(B, R, dtype=torch.float64)
    out = {k: [] for k in ("g_pre", "g_ln", "h_in", "h")}
    for t in range(T):
        h_in = h_in_k[t] if one_step else (1 - first[t]) * h + first[t] * h0
        g_pre = xs[t] + h_in @ Wh.t()
        g_ln = O.layer_norm(g_pre, gam, bet, eps)
        if want_grad:
            g_ln.retain_grad()
        r, c, u = torch.chunk(g_ln, 3, -1)
        c = torch.tanh(torch.sigmoid(r) * c)
        u = torch.sigmoid(u - 1)
        h = u * c + (1 - u) * h_in
        for k, v in (("g_pre", g_pre), ("g_ln", g_ln), ("h_in", h_in), ("h", h)):
            out[k].append(v)
    res = {k: torch.cat(v, 0).detach() for k, v in out.items()}
    if want_grad:
        dl = f64(d_latent, T * B, -1)[:, off:off + R]
        (torch.cat(out["h"], 0) * dl).sum().backward()
        res["d_g_ln"] = torch.cat([g.grad for g in out["g_ln"]], 0)
        res["d_h0"] = h0.grad if h0.grad is not None else torch.zeros(R, dtype=torch.float64)
    return res
