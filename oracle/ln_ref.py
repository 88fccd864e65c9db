"""Float64 reference of the stand-alone LayerNorm family (csrc/norm.cu: LayerNorm + activation forward and backward with
the parameter gradients, column sums; csrc/rssm.cu: the gather + LayerNorm + SiLU of `onehot_linear_ln`) and first-order
bounds on the error of an fp32 implementation.

Like tc_ref / simt_ref, every function takes fp32 (or fp64) tensors on any device and computes in float64 on that
device.  act: 0 identity, 1 SiLU, 2 tanh, 3 ReLU.  Rows are the leading dimension, the C channels the last.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import Tensor

from oracle.simt_ref import U, tau1

# |act'| <= SLOPE (SiLU' peaks at 1.0998), |act''| <= CURV (|tanh''| <= 4 / 3^1.5 = 0.770, |SiLU''| <= 0.5)
SLOPE = {0: 1.0, 1: 1.1, 2: 1.0, 3: 1.0}
CURV = {0: 0.0, 1: 0.5, 2: 0.77, 3: 0.0}


def _d(t: Optional[Tensor]) -> Optional[Tensor]:
    return None if t is None else t.detach().double()


def act64(z: Tensor, act: int) -> Tensor:
    if act == 1:
        return z * torch.sigmoid(z)
    if act == 2:
        return torch.tanh(z)
    if act == 3:
        return z.clamp_min(0.0)
    assert act == 0, act
    return z


def dact64(z: Tensor, act: int) -> Tensor:
    """act'(z)"""
    if act == 1:
        s = torch.sigmoid(z)
        return s * (1 + z * (1 - s))
    if act == 2:
        return 1 - torch.tanh(z) ** 2
    if act == 3:
        return (z > 0).double()
    assert act == 0, act
    return torch.ones_like(z)


def _stats(x: Tensor, eps: float):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    return mu, rstd, (x - mu) * rstd


def ln_act_fwd64(X: Tensor, gamma: Tensor, beta: Tensor, eps: float, act: int):
    """y = act(LN(X)), LN(x) = (x - mu) rstd gamma + beta with the biased variance.  Returns (y, mu, rstd, xhat); mu and
    rstd are [M, 1]."""
    mu, rstd, xh = _stats(_d(X), eps)
    return act64(xh * _d(gamma) + _d(beta), act), mu, rstd, xh


def ln_act_bwd64(X: Tensor, gamma: Tensor, beta: Tensor, eps: float, act: int, dY: Tensor):
    """Backward of ln_act_fwd64 for the output gradient dY, with g = act'(LN(x)) dY:
        dX = rstd (g gamma - mean(g gamma) - xhat mean(g gamma xhat)),  dgamma = sum_rows g xhat,  dbeta = sum_rows g.
    Returns (dX, dgamma, dbeta, mag): mag = {"dgamma": sum_rows |g xhat|, "dbeta": sum_rows |g|}, the scales of the
    parameter gradients' reduction error."""
    _, rstd, xh = _stats(_d(X), eps)
    g = dact64(xh * _d(gamma) + _d(beta), act) * _d(dY)
    gg = g * _d(gamma)
    dx = rstd * (gg - gg.mean(-1, keepdim=True) - xh * (gg * xh).mean(-1, keepdim=True))
    return dx, (g * xh).sum(0), g.sum(0), {"dgamma": (g * xh).abs().sum(0), "dbeta": g.abs().sum(0)}


def col_sum64(X: Tensor):
    """(sum_rows X, sum_rows |X|)"""
    x = _d(X)
    return x.sum(0), x.abs().sum(0)


def ln_bound(pre64: Tensor, mag, gamma: Tensor, beta: Tensor, tau: float, eps: float) -> Tensor:
    """Per-element bound on |LN(pre) - LN64(pre64)| with LN(x) = (x - mu) rstd gamma + beta.

    The sum over j of |d LN_i / d x_j| is at most rstd |gamma_i| (2 + |xhat_i|), so an input error of at most D per row
    moves LN_i by at most rstd |gamma_i| (2 + |xhat_i|) D.  D is the product bound tau * sum|a||b| plus the fp32
    LayerNorm arithmetic seen as an input perturbation: mean and variance summed over N in fp32, (log2 N + 4) u max|x|.
    Storing the result adds 4 u (|LN_i| + |beta_i|).  A stand-alone LayerNorm has no product: tau = 0, mag = 0."""
    N = pre64.shape[-1]
    _, rstd, xhat = _stats(pre64, eps)
    D = (tau * mag + (math.log2(N) + 4) * U * pre64.abs()).amax(-1, keepdim=True)
    g, b = _d(gamma).abs(), _d(beta).abs()
    return rstd * g * (2 + xhat.abs()) * D + 4 * U * ((xhat * g).abs() + b)


def ln_act_fwd_bound(X: Tensor, gamma: Tensor, beta: Tensor, eps: float, act: int, y64: Tensor) -> Tensor:
    """Per-element bound on the fp32 forward: the activation's slope times ln_bound (no product term), plus 4 u |y| for
    expf / tanhf and the division of SiLU."""
    return SLOPE[act] * ln_bound(_d(X), 0.0, gamma, beta, 0.0, eps) + 4 * U * y64.abs()


def ln_act_bwd_bound(X: Tensor, gamma: Tensor, beta: Tensor, eps: float, act: int, dY: Tensor):
    """First-order bounds on an fp32 backward that recomputes the row statistics like the forward.  Returns
    (dX bound [M, C], dgamma propagated term [C], dbeta propagated term [C]); the parameter-gradient bounds are
    param_bound(M, mag, propagated).

    The forward, seen as ln_bound sees it (every x_j moved by at most D = (log2 C + 4) u max|x| per row), leaves
        xhat_fp = (xhat + c)(1 + e_r) + rho_i,  |c| <= rstd D (the mean),  |e_r| <= rstd D + 4u (rstd),
        |rho_i| <= rstd D + 3u |xhat_i| (the element and its two roundings),
    so |xhat_fp - xhat| <= E_i = rstd D (2 + |xhat_i|) + 4u |xhat_i|, and ln = xhat gamma + beta is off by
    |gamma| E_i + 2u (|xhat gamma| + |beta|).  g = act'(ln) dY is then off by
        e_g = |dY| (CURV |ln error| + a_i) + u |g|,
    a_i the evaluation error of act': SiLU 10u s (1 + |ln|) (sigmoid from expf, then three operations), tanh 10u
    (tanhf within 2 ulp, squared and subtracted), exact for identity and ReLU.  The row means s1 = mean(g gamma) and
    s2 = mean(g gamma xhat) are fp32 reductions of length C (tau1(C) of their sum |terms|), and inherit
        e_s1 = mean(|gamma| e_g + u |g gamma|) + tau1(C) mean|g gamma| + 2u |s1|,
        e_s2 = mean(|gamma xhat| e_g + |g gamma| |rho| + 2u |g gamma xhat|) + |c||s1| + e_r |s2|
               + tau1(C) mean|g gamma xhat| + 2u |s2|
    (a common shift c of xhat moves s2 by c s1).  dX_i = rstd (g_i gamma_i - s1 - xhat_i s2) is off by
        e_r |dX_i| + rstd (|gamma_i| e_g,i + u |g gamma|_i + e_s1 + |xhat_i| e_s2 + |s2| E_i)
        + 3u rstd (|g gamma|_i + |s1| + |xhat_i s2|) + u |dX_i|.
    The parameter gradients sum g xhat and g over the rows: each term carries |xhat| e_g + |g| E_i (dgamma) and
    e_g (dbeta), summed over the rows here."""
    x, gam, bet, dy = _d(X), _d(gamma), _d(beta), _d(dY)
    C = x.shape[-1]
    _, rstd, xh = _stats(x, eps)
    D = (math.log2(C) + 4) * U * x.abs().amax(-1, keepdim=True)
    c_max, e_r = rstd * D, rstd * D + 4 * U
    rho = rstd * D + 3 * U * xh.abs()
    E = c_max + e_r * xh.abs() + rho
    ln = xh * gam + bet
    e_ln = gam.abs() * E + 2 * U * ((xh * gam).abs() + bet.abs())
    if act == 1:
        s = torch.sigmoid(ln)
        a = 10 * U * s * (1 + ln.abs())
    elif act == 2:
        a = torch.full_like(ln, 10 * U)
    else:
        a = torch.zeros_like(ln)
    g = dact64(ln, act) * dy
    e_g = dy.abs() * (CURV[act] * e_ln + a) + U * g.abs()
    gg = g * gam
    s1, s2 = gg.mean(-1, keepdim=True), (gg * xh).mean(-1, keepdim=True)
    t = tau1(C)
    e_s1 = (gam.abs() * e_g + U * gg.abs()).mean(-1, keepdim=True) + t * gg.abs().mean(-1, keepdim=True) + 2 * U * s1.abs()
    e_s2 = ((gam * xh).abs() * e_g + gg.abs() * rho + 2 * U * (gg * xh).abs()).mean(-1, keepdim=True) \
        + c_max * s1.abs() + e_r * s2.abs() + t * (gg * xh).abs().mean(-1, keepdim=True) + 2 * U * s2.abs()
    dx = rstd * (gg - s1 - xh * s2)
    b_dx = e_r * dx.abs() + rstd * (gam.abs() * e_g + U * gg.abs() + e_s1 + xh.abs() * e_s2 + s2.abs() * E) \
        + 3 * U * rstd * (gg.abs() + s1.abs() + (xh * s2).abs()) + U * dx.abs()
    return b_dx, (xh.abs() * e_g + g.abs() * E).sum(0), e_g.sum(0)


def param_bound(M: int, mag: Tensor, prop=None, prior: Optional[Tensor] = None) -> Tensor:
    """Bound on a column sum over M rows in fp32 (dgamma, dbeta, col_sum): tau1(M) times the column's sum of |terms|
    (+ |prior| when the result is added to a prior value), plus the propagated error of the terms, summed over the rows."""
    m = mag if prior is None else mag + _d(prior).abs()
    return tau1(M) * m + (0.0 if prop is None else prop)


def gather64(z: Tensor, act: Tensor, WT: Tensor, S: int, K: int):
    """Linear([one-hot z, act]) as `onehot_linear` forms it: pre[m] = sum_g WT[g K + hot(m, g)] + sum_a act[m, a]
    WT[S K + a].  Returns (pre, magnitude = the same sum of |terms|)."""
    hot = _d(z).view(z.shape[0], S, K).argmax(-1) + torch.arange(S, device=z.device) * K     # [M, S] rows of WT
    w, a = _d(WT), _d(act)
    rows = w[hot]                                                                           # [M, S, N]
    wa = w[S * K:]
    pre, mag = rows.sum(1) + a @ wa, rows.abs().sum(1) + a.abs() @ wa.abs()
    return pre, mag
