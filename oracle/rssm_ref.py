"""Float64 reference of the RSSM element-wise and sampling kernels of csrc/rssm.cu that oracle/loss_ref.py (the KL)
and oracle/ln_ref.py (onehot_linear_ln) do not cover: cat_sample (both launch shapes), cat_sample_bwd, head_sample,
gru_gate_fwd / _bwd, mask_mix / mask_rows / mask_bwd and the plain gather form of onehot_linear, with first-order
bounds on the error of an honest fp32 implementation of each output.

Conventions are loss_ref's: functions take fp32 tensors on any device and compute in float64 on that device; every
gradient is float64 autograd of a forward written from the reference's own definitions (RSSM._uniform_mix / Actor.
_uniform_mix, OneHotCategoricalStraightThrough, LayerNormGRUCell's gate, RSSM.dynamic's is_first masking, the Linear
on [z, a]); scalars are the fp32 values a kernel receives (`f32`); bounds are SAFETY times the first-order worst case
plus TINY.

The sample.  A group's sample is argmax_k p(k) / E(k) for the noise E (the exponential race of torch.multinomial), or
argmax_k p(k) for the mode, with p = softmax(mix).  An fp32 kernel sees p with relative error delta_k (the softmax and
logsumexp errors of loss_ref plus the unimix error), so a kernel pick c is correct when
    r(c) >= max_k r(k) (1 - delta),   r(k) = p64(k) / E(k),   delta = SAFETY (delta_c + delta_argmax),
and a pick that differs from the float64 argmax is accepted only inside that margin (`judge_sample`).  Exact ties
(bit-equal fp32 inputs) go to the lowest index, as torch.argmax does.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor
from torch.distributions import OneHotCategoricalStraightThrough

from oracle.loss_ref import (FP32_EPS, SAFETY, TINY, _d, _safe, _softmax_rel, acc_bound, f32, lse_err, unimix_bwd_err,
                             unimix_fwd_err, uniform_mix64)
from oracle.simt_ref import U, tau1

SIG_REL = 4 * U          # expf-based sigmoid / tanhf: within 4u relative


# ------------------------------------------------------------------------------------------------ categorical
def _groups(t: Tensor, groups: int, K: int) -> Tensor:
    return _d(t).reshape(t.shape[0], groups, K)


def _p_rel(l: Tensor, E_l: Tensor) -> Tensor:
    """relative error of p = softmax(l) formed as exp(l - lse - max) / sum from l with absolute error E_l"""
    lg = l - torch.logsumexp(l, -1, keepdim=True)
    p = lg.exp()
    E_lg = E_l + lse_err(l) + (p * E_l).sum(-1, keepdim=True) + U * lg.abs()
    return E_lg + tau1(l.shape[-1]) + 5 * U


def cat_sample(raw: Tensor, noise: Optional[Tensor], unimix: float, groups: int, K: int):
    """mix = _uniform_mix(raw) per group (the stored `mix_out`), p = softmax(mix), and the sample's yardstick.
    Returns ({"mix": [M, G K], "p": [M, G, K], "r": p / E (p for the mode), "delta": [M, G]}, {"mix": bound})."""
    unimix = f32(unimix)
    x = _groups(raw, groups, K)
    _, _, _, _, l, E_l = unimix_fwd_err(x, unimix)
    p = torch.softmax(l, -1)
    e_p = _p_rel(l, E_l) + U                                    # + the division by the noise
    r = p if noise is None else p / _groups(noise, groups, K)
    top = r.argmax(-1, keepdim=True)
    delta = SAFETY * (e_p.amax(-1) + e_p.gather(-1, top).squeeze(-1))
    return {"mix": l.reshape(x.shape[0], -1), "p": p, "r": r, "delta": delta}, _safe({"mix": E_l.reshape(x.shape[0],
                                                                                                            -1)})


def judge_sample(onehot: Tensor, ref: dict, noise: Optional[Tensor] = None):
    """(format_ok, worst, non_argmax): format_ok = every group an exact one-hot of 1.0f / 0.0f; worst = the largest
    (max r - r(c)) / (max r delta) over the groups (<= 1 passes; a fp32 underflow of p costs TINY / min E more);
    non_argmax = the number of picks that are not the float64 argmax."""
    r, delta = ref["r"], ref["delta"]
    M, G, K = r.shape
    z = onehot.detach().reshape(M, G, K).to(r.device)
    fmt = bool(((z == 0) | (z == 1)).all()) and bool((z.sum(-1) == 1).all())
    if not fmt:
        return False, float("inf"), -1
    pick = z.argmax(-1, keepdim=True)
    rmax, top = r.max(-1, keepdim=True)
    rc = r.gather(-1, pick)
    emin = 1.0 if noise is None else _groups(noise, G, K).amin(-1, keepdim=True)
    slack = rmax * delta.unsqueeze(-1) + TINY / emin
    worst = float(((rmax - rc) / slack).max())
    return True, max(worst, 0.0), int((pick != top).sum())


def cat_sample_bwd(raw: Tensor, dz: Optional[Tensor], dmix: Optional[Tensor], unimix: float, groups: int, K: int):
    """draw = d(sum dz z + sum dmix mix) / d raw, z = OneHotCategoricalStraightThrough(logits=mix).rsample(),
    mix = _uniform_mix(raw).  Returns (draw [M, G K], bound)."""
    unimix = f32(unimix)
    M = raw.shape[0]
    x = _groups(raw, groups, K).requires_grad_(True)
    mix = uniform_mix64(x, unimix)
    dist = OneHotCategoricalStraightThrough(logits=mix)
    loss = torch.zeros((), dtype=torch.float64, device=x.device)
    if dz is not None:
        z = dist.mode + dist.probs - dist.probs.detach()           # rsample's straight-through form; the value is
        loss = loss + (z * _groups(dz, groups, K)).sum()            # the sample's, the gradient the probabilities'
    if dmix is not None:
        loss = loss + (mix * _groups(dmix, groups, K)).sum()
    if dz is None and dmix is None:
        return torch.zeros(M, groups * K, dtype=torch.float64, device=x.device), torch.zeros(M, groups * K)
    loss.backward()
    g = x.grad
    # bounds: gg = dmix + p (dz - sum p dz), then the unimix chain rule
    xd = x.detach()
    s, E_s, pm, E_pm, l, E_l = unimix_fwd_err(xd, unimix)
    gg = torch.zeros_like(xd) if dmix is None else _groups(dmix, groups, K).clone()
    E_gg = torch.zeros_like(xd)
    if dz is not None:
        p = torch.softmax(l, -1)
        e_p = _p_rel(l, E_l)
        d = _groups(dz, groups, K)
        pdz = (p * d).sum(-1, keepdim=True)
        E_pdz = (p * e_p * d.abs()).sum(-1, keepdim=True) + tau1(K) * (p * d).abs().sum(-1, keepdim=True)
        t = p * (d - pdz)
        gg = gg + t
        E_gg = p * e_p * (d - pdz).abs() + p * (E_pdz + U * (d - pdz).abs()) + U * t.abs() + TINY * (d - pdz).abs()
    E_gg = E_gg + U * gg.abs()
    if unimix > 0:
        _, b = unimix_bwd_err(s, E_s, pm, E_pm, gg, E_gg, unimix)
    else:
        b = E_gg
    return g.reshape(M, -1), _safe({"draw": b.reshape(M, -1)})["draw"]


def head_raw(X: Tensor, W: Tensor, bias: Optional[Tensor]):
    """raw = X W^T + bias (Actor.mlp_heads[i]) and its bound: one fp32 reduction of Kin products plus the bias"""
    x, w = _d(X), _d(W)
    raw, mag = x @ w.t(), x.abs() @ w.abs().t()
    if bias is not None:
        raw, mag = raw + _d(bias), mag + _d(bias).abs()
    return raw, SAFETY * tau1(X.shape[1]) * mag + TINY


# ------------------------------------------------------------------------------------------------ GRU gate
def gru_gate(G: Tensor, Hin: Tensor, dH: Optional[Tensor] = None):
    """LayerNormGRUCell's gate on the post-LayerNorm G = [reset | cand | update]:
    h = update cand + (1 - update) h_prev with reset = sigmoid(reset), cand = tanh(reset cand), update =
    sigmoid(update - 1).  With dH also dG and dHin (autograd).  Returns (outputs, bounds)."""
    g = _d(G).requires_grad_(dH is not None)
    hp = _d(Hin).requires_grad_(dH is not None)
    gr, gc, gu = torch.chunk(g, 3, -1)
    reset = torch.sigmoid(gr)
    cand = torch.tanh(reset * gc)
    update = torch.sigmoid(gu - 1)
    h = update * cand + (1 - update) * hp
    out = {"h": h.detach()}
    # forward bounds: sigmoid / tanh 4u relative, every product and sum u
    gr, gc, gu, hv = gr.detach(), gc.detach(), gu.detach(), hp.detach()
    r, c, u = reset.detach(), cand.detach(), update.detach()
    E_r = SIG_REL * r + TINY
    rc = r * gc
    E_rc = E_r * gc.abs() + U * rc.abs()
    E_c = (1 - c * c) * E_rc + SIG_REL * c.abs() + TINY
    E_u = u * (1 - u) * U * (gu - 1).abs() + SIG_REL * u + TINY
    E_1mu = E_u + U * (1 - u)
    E_h = E_u * c.abs() + u * E_c + U * (u * c).abs() + E_1mu * hv.abs() + U * ((1 - u) * hv).abs() \
        + U * (u * c).abs() + U * h.detach().abs()
    bound = {"h": E_h}
    if dH is not None:
        dh = _d(dH)
        (h * dh).sum().backward()
        R = hv.shape[-1]
        out["dG"], out["dHin"] = g.grad, hp.grad
        du = dh * (c - hv)
        E_du = dh.abs() * (E_c + U * (c - hv).abs()) + U * du.abs()
        omc2 = 1 - c * c
        E_omc2 = 2 * c.abs() * E_c + U * c * c + U * omc2
        drc = dh * u * omc2
        E_drc = dh.abs() * (E_u * omc2 + u * E_omc2) + 2 * U * drc.abs()
        E_rr = E_r * (1 - r) + r * (E_r + U * (1 - r)) + U * r * (1 - r)
        E_uu = E_u * (1 - u) + u * (E_u + U * (1 - u)) + U * u * (1 - u)
        b_r = E_drc * (gc * r * (1 - r)).abs() + (drc * gc).abs() * E_rr + 3 * U * (drc * gc * r * (1 - r)).abs()
        b_c = E_drc * r + drc.abs() * E_r + U * (drc * r).abs()
        b_u = E_du * u * (1 - u) + du.abs() * E_uu + 2 * U * (du * u * (1 - u)).abs()
        bound["dG"] = torch.cat((b_r, b_c, b_u), -1)
        bound["dHin"] = dh.abs() * E_1mu + U * (dh * (1 - u)).abs()
        assert out["dG"].shape[-1] == 3 * R
    return out, _safe(bound)


# ------------------------------------------------------------------------------------------------ is_first masking
def mask_mix(prev: Tensor, init: Optional[Tensor], first: Tensor) -> Tensor:
    """RSSM.dynamic's masking (1 - first) prev + first init (init None: (1 - first) prev): exact for first in {0, 1}"""
    f = _d(first).reshape(-1, 1)
    out = (1 - f) * _d(prev)
    return out if init is None else out + f * _d(init).reshape(1, -1)


def mask_bwd(dIn: Tensor, first: Tensor, dInit0: Optional[Tensor]):
    """(dPrev, dInit, dInit bound): dPrev = (1 - first) dIn exactly, dInit = dInit0 + sum_m first dIn with one fp32
    reduction of M terms and one rounding of the accumulate (dInit0 None: no dInit)"""
    f, d = _d(first).reshape(-1, 1), _d(dIn)
    dprev = (1 - f) * d
    if dInit0 is None:
        return dprev, None, None
    t = f * d
    s = t.sum(0)
    b = tau1(d.shape[0]) * t.abs().sum(0)
    out = _d(dInit0) + s
    return dprev, out, SAFETY * acc_bound(b, dInit0, s) + TINY


# ------------------------------------------------------------------------------------------------ onehot_linear
def onehot_linear(z: Tensor, act: Optional[Tensor], WT: Tensor, S: int, K: int):
    """Linear([z, a]) with the transposed weight WT [S K + A, N]: out = z WT[:S K] + a WT[S K:], z an exact one-hot
    per group; one fp32 sum of S + A terms per output"""
    zd, w = _d(z), _d(WT)
    out, mag = zd @ w[:S * K], zd.abs() @ w[:S * K].abs()
    A = 0 if act is None else act.shape[1]
    if A:
        out, mag = out + _d(act) @ w[S * K:], mag + _d(act).abs() @ w[S * K:].abs()
    return out, SAFETY * tau1(S + A) * mag + TINY
