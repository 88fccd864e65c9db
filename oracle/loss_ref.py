"""Float64 reference of the Dreamer-V3 objective kernels (csrc/losses.cu, csrc/dv3_cont.cu and the KL of csrc/rssm.cu)
and first-order bounds on the error of an honest fp32 implementation of each output.

Like tc_ref / simt_ref / ln_ref, every function takes fp32 tensors on any device and computes in float64 on that
device.  Each forward is written from the reference's own definitions (TwoHotEncodingDistribution, MSEDistribution,
Bernoulli, the categorical KL with free nats, compute_lambda_values with BernoulliSafeMode.mode continues, Moments,
the discrete objective with unimix, the `scaled_normal` actor with its detached clip factor), and every gradient is
float64 autograd of that forward, so a derivation error shared by a kernel and the fp32 emulator shows up.  Autograd
keeps torch's conventions: torch.maximum splits a tie evenly, clamp passes the gradient at its bounds.

Discrete decisions are taken as fp32 torch takes them on the same inputs: the continue flag sigmoid(l) > 0.5, the
two-hot `below` index, the free-nats switch, the quantile rank q (n - 1) and the argmax of a stored action.  Only the
continuous arithmetic is float64, so a logit of +1e-9 that fp32 rounds to "not continuing" is not a kernel error.
Scalar parameters (scales, gamma, lambda, ...) are the fp32 values a kernel receives (`f32`).

Bounds (u = 2^-24, tau1(n) = u (16 + 2 sqrt n) for an fp32 reduction of length n):
  - logsumexp of K logits with max shift: E_lse = tau1(K) + 3u + u sum_c p_c |l_c - max| + 2u (|max| + log K),
    the conditioning term |max| + log K; a softmax entry is then off by p_c (E_lse + u |l_c - lse| + 2u).
  - the two-hot target: symlog off by E_xs = 2u (1 + |xs|), a bin by E_b = 2u max(|low|, |high|) (the reference's
    bins are torch's fp32 linspace even for float64 logits; a kernel recomputing them may contract one rounding);
    the weights are continuous in xs with slope 1 / step, so they are off by E_w = 2 (E_xs + E_b) / step + 4u, which
    also covers a `below` index that fp32 puts on the other side of a bin edge.
  - twohot_mean: m = sum_c p_c b_c off by E_m = sum_c p_c (e_c |b_c| + E_b) + tau1(K) sum_c p_c |b_c| with the
    softmax's relative error e_c = tau1(K) + 5u + u |l_c - max|; symexp amplifies by exp(|m|).  Its backward
    exp(|m|) dV p_c (b_c - m) carries the same E_m.
  - lambda_returns: the recursion L_t = r + c ((1 - lambda) v + lambda L_{t+1}) carries its bound alongside the value,
    E_t = |c lambda| E_{t+1} + 3u |c (1 - lambda) v| + u |interm| + 2u |c lambda L_{t+1}| + u |L_t|, as
    simt_ref.lstm_bwd64 does for the LSTM; its backward carries G_t = dL_t + c lambda G_{t-1} the same way.  The
    discount cumprod of t + 1 factors is off by (t + 2) u |D_t|.
  - the KL: per group, E_lse of both sides and the relative error of each probability, a reduction of G K terms
    (tau1(G K)) for the row totals and of K terms for each group's KL inside d_post.
  - the actor objective: the softmax, the unimix mix (1 - unimix) s + unimix / K and its log, the logsumexp of the mix,
    then every product and the chain rule through the mix, term by term (actor_loss).
  - the continuous actor: sigmoid / tanh within 4u, every other operation u, the clip factor's error carried as that
    of |a| (the clipped action is continuous in a).
  - moments_update: no bound: the order statistics must equal fp32 torch.quantile's exactly, and the lerp must be within
    2 ulp of it (an FMA contraction can differ from the CPU by one rounding).  The EMA adds 3u of its terms.
  - sum_rows / weighted_mean: tau1(n) of the sum of |terms|, plus u of the result for the scale.
Each term above is the worst case of one rounding of an fp32 operation in the order the kernels apply them; the bounds
returned are twice their sum (SAFETY), so an implementation that orders or contracts the operations differently (an
FMA, another reduction tree) is held to the same bound, and a probability that underflows fp32 costs at most TINY.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch
import torch.nn.functional as F
from torch import Tensor
from torch.distributions import Bernoulli, Independent, Normal, OneHotCategorical
from torch.distributions.kl import kl_divergence

from oracle.simt_ref import U, tau1

FP32_EPS = 2.0 ** -23          # probs_to_logits clamps at the eps of the dtype the reference runs in (fp32)
HALF_LOG_2PI_E = 0.5 + 0.5 * math.log(2 * math.pi)
TINY = 2.0 ** -126             # smallest normal fp32: a probability below it may flush to 0 (absolute error floor)
SAFETY = 2.0                   # every bound is twice its first-order worst case (see the module docstring)


def _safe(bounds: dict) -> dict:
    """SAFETY times the first-order bound, floored at TINY: below it fp32 results are subnormal or flushed"""
    return {k: SAFETY * v + TINY for k, v in bounds.items()}


def f32(v: float) -> float:
    """the fp32 value a kernel receives for the Python float v"""
    return float(torch.tensor(v, dtype=torch.float32))


def _d(t: Optional[Tensor]) -> Optional[Tensor]:
    return None if t is None else t.detach().double()


def symlog64(x: Tensor) -> Tensor:
    return torch.sign(x) * torch.log(1 + torch.abs(x))


def symexp64(x: Tensor) -> Tensor:
    return torch.sign(x) * (torch.exp(torch.abs(x)) - 1)


def bins64(nb: int, low: float, high: float, device) -> Tensor:
    """TwoHotEncodingDistribution's bins: torch.linspace in the default dtype (fp32) whatever the logits' dtype"""
    return torch.linspace(low, high, nb, device=device).double()


def lse_err(l64: Tensor) -> Tensor:
    """E_lse over the last dimension, keepdim"""
    K = l64.shape[-1]
    mx = l64.amax(-1, keepdim=True)
    p = torch.softmax(l64, -1)
    return tau1(K) + 3 * U + U * (p * (l64 - mx).abs()).sum(-1, keepdim=True) + 2 * U * (mx.abs() + math.log(K))


def _bin_err(low: float, high: float) -> float:
    """a kernel's fp32 linspace against torch's: one rounding of the bin and one of step * i (an FMA contraction)"""
    return 2 * U * max(abs(low), abs(high))


def acc_bound(bound: Tensor, prior: Optional[Tensor], value: Tensor) -> Tensor:
    """the bound of `prior + value` stored in fp32 (accumulate): one more rounding of the sum"""
    if prior is None:
        return bound
    return bound + U * (_d(prior).abs() + (_d(prior) + value).abs())


# ------------------------------------------------------------------------------------------------ world-model losses
def mse(pred: Tensor, target: Tensor, scale: float):
    """-MSEDistribution(pred, agg="sum").log_prob(target) per row and d(scale * sum rows) / d pred"""
    p = _d(pred).requires_grad_(True)
    t = _d(target)
    loss = ((p - t) ** 2).sum(-1)
    (f32(scale) * loss).sum().backward()
    d = (p - t).detach()
    g = p.grad
    return {"loss": loss.detach(), "grad": g}, _safe({"loss": (tau1(d.shape[-1]) + 3 * U) * (d * d).sum(-1),
                                                      "grad": 3 * U * g.abs()})


def twohot_target(x: Tensor, nb: int, low: float, high: float):
    """The target of TwoHotEncodingDistribution.log_prob: (target [M, nb] float64, below, above, xs [M, 1]).  `below`
    is counted as fp32 torch counts it (fp32 linspace <= fp32 symlog), the weights are float64 distances."""
    x = x.reshape(-1)
    b32 = torch.linspace(low, high, nb, device=x.device)
    xs32 = torch.sign(x) * torch.log(1 + torch.abs(x))
    below = (b32 <= xs32.unsqueeze(-1)).to(torch.int64).sum(-1, keepdim=True) - 1
    above = torch.clamp(below + 1, max=nb - 1)
    below = torch.clamp(below, min=0)
    b = bins64(nb, low, high, x.device)
    xs = symlog64(_d(x)).unsqueeze(-1)
    equal = below == above
    one = torch.ones_like(xs)
    d_lo = torch.where(equal, one, (b[below] - xs).abs())
    d_hi = torch.where(equal, one, (b[above] - xs).abs())
    tot = d_lo + d_hi
    t = torch.zeros(x.shape[0], nb, dtype=torch.float64, device=x.device)
    t.scatter_add_(1, below, d_hi / tot).scatter_add_(1, above, d_lo / tot)
    return t, below, above, xs


def twohot_loss(logits: Tensor, x: Tensor, weight: Optional[Tensor], scale: float, low: float, high: float):
    """loss[m] = -TwoHotEncodingDistribution(logits).log_prob(x[m]) and d(scale * sum_m weight[m] loss[m]) / d logits"""
    M, nb = logits.shape
    t, below, above, xs = twohot_target(x, nb, low, high)
    l = _d(logits).requires_grad_(True)
    logp = l - torch.logsumexp(l, -1, keepdim=True)
    loss = -(t * logp).sum(-1)
    w = torch.ones(M, dtype=torch.float64, device=l.device) if weight is None else _d(weight).reshape(-1)
    wr = f32(scale) * w
    (wr * loss).sum().backward()
    g, lp = l.grad, logp.detach()
    p = lp.exp()
    E_lse = lse_err(l.detach())
    E_w = 2 * (2 * U * (1 + xs.abs()) + _bin_err(low, high)) / ((high - low) / (nb - 1)) + 4 * U
    lp_lo, lp_hi = lp.gather(1, below), lp.gather(1, above)
    w_lo, w_hi = t.gather(1, below), t.gather(1, above)
    b_loss = E_w * (lp_lo.abs() + lp_hi.abs()) + (w_lo + w_hi) * E_lse \
        + 4 * U * (w_lo * lp_lo.abs() + w_hi * lp_hi.abs())
    hit = torch.zeros_like(t).scatter_(1, below, 1.0).scatter_(1, above, 1.0)
    b_g = wr.abs().unsqueeze(-1) * (p * (E_lse + U * lp.abs() + 2 * U) + E_w * hit + 2 * U * (p - t).abs()) \
        + 2 * U * g.abs() + TINY * wr.abs().unsqueeze(-1)
    return {"loss": loss.detach(), "grad": g}, _safe({"loss": b_loss.squeeze(-1), "grad": b_g})


def bce(logit: Tensor, target: Tensor, loss_scale: float, scale: float):
    """loss = -loss_scale * Bernoulli(logits).log_prob(target) and d(scale * sum loss) / d logit"""
    ls, s = f32(loss_scale), f32(scale)
    l = _d(logit).reshape(-1).requires_grad_(True)
    y = _d(target).reshape(-1)
    loss = -ls * Bernoulli(logits=l).log_prob(y)
    (s * loss).sum().backward()
    g = l.grad
    lv, sg = l.detach(), torch.sigmoid(l.detach())
    b_loss = abs(ls) * 4 * U * (((1 - y) * lv).abs() + lv.abs() + torch.log1p(torch.exp(-lv.abs()))) \
        + U * loss.detach().abs()
    b_g = abs(ls * s) * (4 * U * sg + 3 * U * (sg - y).abs())
    return {"loss": loss.detach(), "grad": g}, _safe({"loss": b_loss, "grad": b_g})


def _softmax_rel(l64: Tensor) -> Tensor:
    """relative error of an fp32 softmax entry expf(l - max) / sum"""
    return tau1(l64.shape[-1]) + 5 * U + U * (l64 - l64.amax(-1, keepdim=True)).abs()


def twohot_mean(logits: Tensor, low: float, high: float, d_mean: Optional[Tensor] = None):
    """V = TwoHotEncodingDistribution(logits).mean per row; with d_mean also dlogits = d(sum d_mean V) / d logits"""
    M, nb = logits.shape
    l = _d(logits).requires_grad_(d_mean is not None)
    b = bins64(nb, low, high, l.device)
    p = torch.softmax(l, -1)
    m = (p * b).sum(-1)
    V = symexp64(m)
    pd, md = p.detach(), m.detach().unsqueeze(-1)
    e = _softmax_rel(l.detach())
    E_b = _bin_err(low, high)
    E_m = (pd * (e * b.abs() + E_b)).sum(-1, keepdim=True) + tau1(nb) * (pd * b.abs()).sum(-1, keepdim=True)
    amp = torch.exp(md.abs())
    out, bound = {"mean": V.detach()}, {"mean": (amp * (E_m + 3 * U)).squeeze(-1)}
    if d_mean is not None:
        (V * _d(d_mean).reshape(-1)).sum().backward()
        g = _d(d_mean).reshape(-1, 1).abs() * amp
        out["grad"] = l.grad
        bound["grad"] = g * (pd * (b - md).abs() * (E_m + e + 5 * U) + pd * (E_b + E_m) + TINY * ((b - md).abs() + 1))
    return out, _safe(bound)


# ------------------------------------------------------------------------------------------------ returns and moments
def continues(cont_logit: Tensor) -> Tensor:
    """BernoulliSafeMode(logits).mode as fp32 torch decides it, in float64"""
    return (torch.sigmoid(cont_logit.float()) > 0.5).double()


def lambda_values64(rewards: Tensor, values: Tensor, conts: Tensor, lmbda: float) -> Tensor:
    """compute_lambda_values (dreamer_v3/utils.py): rewards / values / conts are the H rows of steps 1..H"""
    vals = [values[-1:]]
    interm = rewards + conts * values * (1 - lmbda)
    for t in reversed(range(len(conts))):
        vals.append(interm[t] + conts[t] * lmbda * vals[-1])
    return torch.cat(list(reversed(vals))[:-1])


def lambda_returns(rew: Tensor, val: Tensor, cont_logit: Tensor, true_cont: Tensor, gamma: float, lmbda: float):
    """lam [H, N] = compute_lambda_values(r[1:], v[1:], continues[1:] gamma, lambda), discount [H+1, N] =
    cumprod(continues gamma) / gamma with continues[0] = true_cont"""
    gamma, lmbda = f32(gamma), f32(lmbda)
    r, v = _d(rew), _d(val)
    c = continues(cont_logit)
    c[0] = _d(true_cont).reshape(-1)
    H = r.shape[0] - 1
    lam = lambda_values64(r[1:], v[1:], c[1:] * gamma, lmbda)
    disc = torch.cumprod(c * gamma, 0) / gamma
    E = torch.zeros_like(lam)
    e_next, L_next = torch.zeros_like(v[0]), v[H]
    for t in reversed(range(H)):
        cg = c[t + 1] * gamma
        interm = r[t + 1] + cg * v[t + 1] * (1 - lmbda)
        e_next = (cg * lmbda).abs() * e_next + 3 * U * (cg * (1 - lmbda) * v[t + 1]).abs() + U * interm.abs() \
            + 2 * U * (cg * lmbda * L_next).abs() + U * lam[t].abs()
        E[t], L_next = e_next, lam[t]
    steps = torch.arange(H + 1, dtype=torch.float64, device=v.device).unsqueeze(-1)
    return {"lam": lam, "discount": disc}, _safe({"lam": E, "discount": (steps + 2) * U * disc.abs()})


def quantiles32(x: Tensor, p_low: float, p_high: float):
    """Moments' torch.quantile of the fp32 values, on x's device"""
    x = x.reshape(-1).float()
    return torch.quantile(x, p_low), torch.quantile(x, p_high)


def moments(x: Tensor, state: Tensor, decay: float, max_: float, p_low: float, p_high: float):
    """Moments.forward: state (low, high) EMA of the fp32 quantiles, out = (low, max(1 / max_, high - low)).
    Returns ((state, out), (q_low, q_high) in fp32, (state bound, out bound))."""
    lo, hi = quantiles32(x, p_low, p_high)
    dec, s = f32(decay), _d(state)
    st = torch.stack((dec * s[0] + (1 - dec) * lo.double(), dec * s[1] + (1 - dec) * hi.double()))
    inv_max = f32(1.0 / f32(max_))
    out = torch.stack((st[0], torch.maximum(torch.tensor(inv_max, dtype=torch.float64, device=st.device),
                                            st[1] - st[0])))
    b_st = SAFETY * 3 * U * ((dec * s).abs() + (1 - dec) * torch.stack((lo, hi)).double().abs())
    b_out = torch.stack((b_st[0], b_st[0] + b_st[1] + U * (st[1] - st[0]).abs()))
    return (st, out), (lo, hi), (b_st, b_out)


# ------------------------------------------------------------------------------------------------ KL
def kl_loss(post: Tensor, prior: Tensor, groups: int, K: int, kl_dyn: float, kl_rep: float, free_nats: float,
            regularizer: float, scale: float):
    """rows [M, 4] = (KL(post || prior) summed over the groups, (dyn + rep) max(KL, free_nats), H(post), H(prior)) and
    the gradients of coef (dyn max(KL(sg(post) || prior), free) + rep max(KL(post || sg(prior)), free)),
    coef = scale * regularizer, w.r.t. the posterior and prior logits.  The free-nats switch is fp32 torch's."""
    M = post.shape[0]
    kl_dyn, kl_rep, free_nats, coef = f32(kl_dyn), f32(kl_rep), f32(free_nats), f32(f32(scale) * f32(regularizer))
    lp32 = post.float().reshape(M, groups, K).log_softmax(-1)
    lq32 = prior.float().reshape(M, groups, K).log_softmax(-1)
    kl32 = (lp32.exp() * (lp32 - lq32)).sum((-1, -2))
    live = torch.where(kl32 > free_nats, 1.0, torch.where(kl32 == free_nats, 0.5, 0.0)).double()
    a = _d(post).reshape(M, groups, K).requires_grad_(True)
    b = _d(prior).reshape(M, groups, K).requires_grad_(True)

    def dist(logits):
        return Independent(OneHotCategorical(logits=logits), 1)

    dyn = kl_divergence(dist(a.detach()), dist(b))
    rep = kl_divergence(dist(a), dist(b.detach()))
    (coef * live * (kl_dyn * dyn + kl_rep * rep)).sum().backward()
    kl = rep.detach()
    rows = torch.stack((kl, (kl_dyn + kl_rep) * torch.maximum(kl, torch.full_like(kl, free_nats)),
                        dist(a.detach()).entropy(), dist(b.detach()).entropy()), -1)
    # bounds
    av, bv = a.detach(), b.detach()
    lpa, lqb = av - torch.logsumexp(av, -1, keepdim=True), bv - torch.logsumexp(bv, -1, keepdim=True)
    pa, pb = lpa.exp(), lqb.exp()
    Ea, Eb = lse_err(av), lse_err(bv)
    e_pa, e_pb = Ea + U * lpa.abs() + 2 * U, Eb + U * lqb.abs() + 2 * U
    dif = lpa - lqb
    E_dif = Ea + Eb + U * (lpa.abs() + lqb.abs() + dif.abs())
    t = pa * dif
    err_t = pa * (e_pa * dif.abs() + E_dif) + U * t.abs()
    GK = groups * K
    E_klg = err_t.sum(-1, keepdim=True) + tau1(K) * t.abs().sum(-1, keepdim=True)
    E_kl = err_t.sum((-1, -2)) + tau1(GK) * t.abs().sum((-1, -2))
    E_hp = (pa * (e_pa * lpa.abs() + Ea + U * lpa.abs())).sum((-1, -2)) + tau1(GK) * (pa * lpa).abs().sum((-1, -2))
    E_hq = (pb * (e_pb * lqb.abs() + Eb + U * lqb.abs())).sum((-1, -2)) + tau1(GK) * (pb * lqb).abs().sum((-1, -2))
    b_rows = torch.stack((E_kl, abs(kl_dyn + kl_rep) * E_kl + 2 * U * rows[:, 1].abs(), E_hp, E_hq), -1)
    lv = (live * coef).reshape(M, 1, 1)
    g_post, g_prior = a.grad, b.grad
    b_prior = (kl_dyn * lv).abs() * (pb * e_pb + pa * e_pa + U * (pb - pa).abs() + 2 * TINY) + 3 * U * g_prior.abs()
    delta = dif - (pa * dif).sum(-1, keepdim=True)
    b_post = (kl_rep * lv).abs() * (pa * e_pa * delta.abs() + pa * (E_dif + E_klg + U * delta.abs())
                                    + TINY * (delta.abs() + 1)) + 4 * U * g_post.abs()
    out = {"rows": rows, "d_post": g_post.reshape(M, -1), "d_prior": g_prior.reshape(M, -1)}
    return out, _safe({"rows": b_rows, "d_post": b_post.reshape(M, -1), "d_prior": b_prior.reshape(M, -1)})


def kl_rows64(post: Tensor, prior: Tensor, groups: int, K: int) -> Tensor:
    """float64 KL(post || prior) per row, for placing rows around free_nats"""
    a, b = _d(post).reshape(post.shape[0], groups, K), _d(prior).reshape(prior.shape[0], groups, K)
    la, lb = a.log_softmax(-1), b.log_softmax(-1)
    return (la.exp() * (la - lb)).sum((-1, -2))


# ------------------------------------------------------------------------------------------------ actor objectives
def uniform_mix64(x: Tensor, unimix: float) -> Tensor:
    """Actor._uniform_mix: log of the clamped (1 - unimix) softmax + unimix / K"""
    if unimix <= 0:
        return x
    probs = (1 - unimix) * x.softmax(-1) + unimix * torch.ones_like(x) / x.shape[-1]
    return torch.log(probs.clamp(FP32_EPS, 1 - FP32_EPS))


def unimix_fwd_err(x64: Tensor, unimix: float):
    """The unimix mix of the logits x64 [..., K] as an fp32 kernel forms it, with the error of each step:
    (s, E_s, pm, E_pm, l, E_l): s = softmax(x) with relative error E_s, pm = (1 - unimix) s + unimix / K with relative
    error E_pm (None, None without unimix), l = log(clamp(pm)) (x itself without unimix) with absolute error E_l.
    The clamp is continuous, so it passes pm's relative error on unchanged."""
    K = x64.shape[-1]
    s, E_s = x64.softmax(-1), _softmax_rel(x64)
    if unimix <= 0:
        return s, E_s, None, None, x64, torch.zeros_like(x64)
    pm = (1 - unimix) * s + unimix / K
    E_pm = ((1 - unimix) * s * (E_s + 2 * U) + 2 * U * unimix / K) / pm + U
    l = torch.log(pm.clamp(FP32_EPS, 1 - FP32_EPS))
    return s, E_s, pm, E_pm, l, E_pm + 2 * U * l.abs()


def unimix_bwd_err(s: Tensor, E_s: Tensor, pm: Tensor, E_pm: Tensor, gg: Tensor, E_gg: Tensor, unimix: float):
    """The chain rule through the unimix mix and its clamp: the gradient gg w.r.t. l = log(clamp(pm)) (error E_gg)
    taken to the logits, dr = s (ds - sum s ds) with ds = gg (1 - unimix) / pm inside the clamp and 0 outside.
    Returns (dr, bound of its error).  A kernel decides "inside" from its fp32 pm: an element whose float64 pm lies
    within its error of either clamp edge may take either branch, so its ds may also be the other branch's."""
    inside = ((pm >= FP32_EPS) & (pm <= 1 - FP32_EPS)).double()
    slack = E_pm * pm
    edge = (((pm - FP32_EPS).abs() <= slack) | ((pm - (1 - FP32_EPS)).abs() <= slack)).double()
    ds = inside * gg * (1 - unimix) / pm
    E_ds = (inside * (E_gg + gg.abs() * (E_pm + 3 * U))
            + edge * (gg.abs() + E_gg) * (1 + E_pm + 3 * U)) * (1 - unimix) / pm
    sds = (s * ds).sum(-1, keepdim=True)
    E_sds = (s * E_ds + (s * ds).abs() * (E_s + U)).sum(-1, keepdim=True) \
        + tau1(s.shape[-1]) * (s * ds).abs().sum(-1, keepdim=True)
    dr = s * (ds - sds)
    return dr, s * (E_ds + E_sds) + dr.abs() * (E_s + U) + (U * s + TINY) * (ds - sds).abs()


def actor_loss(raw: Tensor, actions: Tensor, lam: Tensor, val: Tensor, discount: Tensor, moments_: Tensor,
               head_dims: Sequence[int], unimix: float, ent_coef: float, scale: float):
    """The discrete objective of dreamer_v3.py: rows[m] = discount (sum_heads log_prob(action) adv + ent_coef sum_heads
    entropy) with adv = (lam - offset) / invscale - (val - offset) / invscale detached, and draw = d(-scale sum rows) /
    d raw through the unimix OneHotCategorical of each head."""
    unimix, ent_coef, scale = f32(unimix), f32(ent_coef), f32(scale)
    M = raw.shape[0]
    off, inv = float(moments_[0]), float(moments_[1])
    lm, vm, D = _d(lam).reshape(-1), _d(val).reshape(-1), _d(discount).reshape(-1)
    adv = (lm - off) / inv - (vm - off) / inv
    x = _d(raw).requires_grad_(True)
    obj = torch.zeros(M, dtype=torch.float64, device=x.device)
    ent = torch.zeros_like(obj)
    o, per_head = 0, []
    for K in head_dims:
        xh = x[:, o:o + K]
        dist = OneHotCategorical(logits=uniform_mix64(xh, unimix))
        idx = actions[:, o:o + K].float().argmax(-1)
        obj = obj + dist.log_prob(F.one_hot(idx, K).double()) * adv
        ent = ent + dist.entropy()
        per_head.append((o, K, idx))
        o += K
    rows = D * (obj + ent_coef * ent)
    (-scale * rows).sum().backward()
    g = x.grad
    # bounds
    E_adv = 3 * U * ((lm - off).abs() + (vm - off).abs()) / abs(inv) + U * adv.abs()
    E_obj, E_ent_tot = torch.zeros_like(obj), torch.zeros_like(obj)
    b_draw = torch.zeros_like(g)
    gs = (scale * D).abs().unsqueeze(-1)
    heads = []
    for o, K, idx in per_head:
        s, E_s, pm, E_pm, l, E_l = unimix_fwd_err(x.detach()[:, o:o + K], unimix)
        lg = l - torch.logsumexp(l, -1, keepdim=True)
        p = lg.exp()
        E_lg = E_l + lse_err(l) + (p * E_l).sum(-1, keepdim=True) + U * lg.abs()
        e_p = E_lg + 2 * U
        hent = -(p * lg).sum(-1, keepdim=True)
        E_ent = (p * (e_p * lg.abs() + E_lg)).sum(-1, keepdim=True) + tau1(K) * (p * lg).abs().sum(-1, keepdim=True) \
            + U * hent.abs()
        logp = lg.gather(1, idx.unsqueeze(-1)).squeeze(-1)
        E_obj += E_lg.gather(1, idx.unsqueeze(-1)).squeeze(-1) * adv.abs() + logp.abs() * E_adv \
            + 2 * U * (logp * adv).abs()
        E_ent_tot += E_ent.squeeze(-1)
        heads.append((o, K, idx, s, E_s, l, lg, p, E_lg, e_p, hent, E_ent, pm, E_pm))
    for o, K, idx, s, E_s, l, lg, p, E_lg, e_p, hent, E_ent, pm, E_pm in heads:
        dl = F.one_hot(idx, K).double() - p
        a1 = adv.unsqueeze(-1)
        dent = -p * (lg + hent)
        gg = -gs * (a1 * dl + ent_coef * dent)
        E_gg = gs * (E_adv.unsqueeze(-1) * dl.abs() + a1.abs() * p * e_p
                     + abs(ent_coef) * (p * e_p * (lg + hent).abs() + p * (E_lg + E_ent))
                     + 4 * U * ((a1 * dl).abs() + abs(ent_coef) * dent.abs())
                     + TINY * (a1.abs() + abs(ent_coef) * ((lg + hent).abs() + 1))) + 2 * U * gg.abs()
        if unimix > 0:
            b_draw[:, o:o + K] = unimix_bwd_err(s, E_s, pm, E_pm, gg, E_gg, unimix)[1]
        else:
            b_draw[:, o:o + K] = E_gg
    b_rows = D.abs() * (E_obj + abs(ent_coef) * E_ent_tot
                        + 3 * U * (obj.detach().abs() + abs(ent_coef) * ent.detach().abs()))
    return {"rows": rows.detach(), "draw": g}, _safe({"rows": b_rows, "draw": b_draw})


def cont_action(head: Tensor, eps: Tensor, min_std: float, max_std: float, init_std: float, clip: float,
                d_action: Optional[Tensor] = None, discount: Optional[Tensor] = None, ent_scale: float = 0.0):
    """The `scaled_normal` actor: std = (max - min) sigmoid(std_raw + init) + min, action = rsample of
    Normal(tanh(mean), std) with the noise eps, times the detached clip / max(clip, |action|); ent = the Independent
    Normal's entropy.  With d_action: dhead = d(sum d_action action + sum_m ent_scale discount[m] ent[m]) / d head."""
    min_std, max_std, init_std, clip, ent_scale = f32(min_std), f32(max_std), f32(init_std), f32(clip), f32(ent_scale)
    M, A = eps.shape
    h = _d(head).requires_grad_(d_action is not None)
    e = _d(eps)
    mean, sr = h[:, :A], h[:, A:]
    std = (max_std - min_std) * torch.sigmoid(sr + init_std) + min_std
    dist = Independent(Normal(torch.tanh(mean), std), 1)
    a_raw = dist.base_dist.loc + e * dist.base_dist.scale
    a = a_raw
    if clip > 0:
        c = torch.full_like(a_raw, clip)
        a = a_raw * (c / torch.maximum(c, a_raw.abs())).detach()
    ent = dist.entropy()
    out = {"action": a.detach(), "ent": ent.detach()}
    # forward bounds
    md, sd, ard, stdd = mean.detach(), sr.detach(), a_raw.detach(), std.detach()
    z = sd + init_std
    sg = torch.sigmoid(z)
    E_sg = U * z.abs() * (1 - sg) + 4 * U                                        # relative
    E_std = (max_std - min_std) * sg * (E_sg + 2 * U) + U * stdd
    th = torch.tanh(md)
    E_a = 4 * U * th.abs() + e.abs() * E_std + U * (stdd * e).abs() + U * ard.abs()
    ls = torch.log(stdd)
    E_ent = (E_std / stdd + 2 * U * ls.abs() + U * (HALF_LOG_2PI_E + ls.abs())).sum(-1) \
        + tau1(A) * (HALF_LOG_2PI_E + ls).abs().sum(-1)
    bound = {"action": E_a + 3 * U * a.detach().abs(), "ent": E_ent}
    if d_action is not None:
        dent = ent_scale * _d(discount).reshape(-1)[:M]
        ((a * _d(d_action)).sum() + (dent * ent).sum()).backward()
        out["dhead"] = h.grad
        f = (clip / torch.clamp(ard.abs(), min=clip)) if clip > 0 else torch.ones_like(ard)
        E_f = (E_a / torch.clamp(ard.abs(), min=clip) + 2 * U) if clip > 0 else torch.zeros_like(ard)
        da = _d(d_action) * f
        E_da = da.abs() * (E_f + U)
        omt = 1 - th * th
        b_mean = E_da * omt + da.abs() * (8 * U * th * th + 2 * U) + U * (da * omt).abs()
        dn = dent.unsqueeze(-1)
        dstd = da * e + dn / stdd
        E_dstd = E_da * e.abs() + U * (da * e).abs() + (dn / stdd).abs() * (E_std / stdd + 3 * U) + U * dstd.abs()
        sgsg = sg * (1 - sg)
        E_sgsg = sg * E_sg * (1 - 2 * sg).abs() + 2 * U * sgsg
        b_std = (max_std - min_std) * (E_dstd * sgsg + dstd.abs() * E_sgsg) \
            + 3 * U * (dstd * (max_std - min_std) * sgsg).abs()
        bound["dhead"] = torch.cat((b_mean, b_std), -1)
    return out, _safe(bound)


def lambda_returns_bwd(cont_logit: Tensor, discount: Tensor, moments_: Tensor, lam: Tensor, val: Tensor, ent: Tensor,
                       gamma: float, lmbda: float, ent_coef: float, scale: float):
    """The continuous objective rows [H, N] = discount (adv + ent_coef ent), adv = (lam - offset) / invscale -
    (val - offset) / invscale, and the gradients of policy_loss = -scale sum rows w.r.t. the predicted values and
    rewards [H+1, N] through compute_lambda_values (continues from the fp32 flags, continues[0] unused)."""
    gamma, lmbda, ent_coef, scale = f32(gamma), f32(lmbda), f32(ent_coef), f32(scale)
    H, N = lam.shape
    off, inv = float(moments_[0]), float(moments_[1])
    c = continues(cont_logit).reshape(H + 1, N)
    D = _d(discount).reshape(H + 1, N)
    e = _d(ent).reshape(-1)[:H * N].reshape(H, N)
    v = _d(val).reshape(H + 1, N).requires_grad_(True)
    r = torch.zeros(H + 1, N, dtype=torch.float64, device=v.device, requires_grad=True)
    lam_g = lambda_values64(r[1:], v[1:], c[1:] * gamma, lmbda)          # linear in r, v: their values do not matter
    adv_g = (lam_g - off) / inv - (v[:H] - off) / inv
    (-scale * (D[:H] * (adv_g + ent_coef * e)).sum()).backward()
    lv, vv = _d(lam), v.detach()
    adv = (lv - off) / inv - (vv[:H] - off) / inv
    rows = D[:H] * (adv + ent_coef * e)
    d_val, d_rew = v.grad, r.grad
    # bounds: G_t = d_rew[t + 1], carried forward in t
    sinv = scale / inv
    b_rows = D[:H].abs() * (3 * U * (adv).abs() + 2 * U * (ent_coef * e).abs() + U * (adv + ent_coef * e).abs()) \
        + U * rows.abs()
    b_rew, b_val = torch.zeros_like(d_rew), torch.zeros_like(d_val)
    E_G = torch.zeros(N, dtype=torch.float64, device=v.device)
    E_carry = torch.zeros_like(E_G)
    G_prev, c_prev = torch.zeros_like(E_G), torch.zeros_like(E_G)
    for t in range(H):
        dl = (sinv * D[t]).abs()
        G = d_rew[t + 1]
        E_G = (c_prev * lmbda).abs() * E_G + 3 * U * dl + 2 * U * (c_prev * lmbda * G_prev).abs() + U * G.abs()
        b_rew[t + 1] = E_G
        b_val[t] = E_carry + 3 * U * dl + U * d_val[t].abs()
        cg = c[t + 1] * gamma
        E_carry = (cg * (1 - lmbda)).abs() * E_G + 3 * U * (G * cg * (1 - lmbda)).abs()
        G_prev, c_prev = G, cg
    b_val[H] = E_carry + (c_prev * lmbda).abs() * E_G + 2 * U * (c_prev * lmbda * G_prev).abs() + U * d_val[H].abs()
    return {"rows": rows, "d_val": d_val, "d_rew": d_rew}, _safe({"rows": b_rows, "d_val": b_val, "d_rew": b_rew})


# ------------------------------------------------------------------------------------------------ reductions
def sum_rows(X: Tensor, scale: float):
    s = f32(scale)
    x = _d(X)
    out = s * x.sum(0)
    return out, SAFETY * (tau1(x.shape[0]) * abs(s) * x.abs().sum(0) + U * out.abs())


def weighted_mean(x: Tensor, w: Tensor, scale: float):
    s = f32(scale)
    xw = _d(x).reshape(-1) * _d(w).reshape(-1)
    out = s * xw.sum()
    return out, SAFETY * (tau1(xw.numel()) * abs(s) * xw.abs().sum() + U * out.abs())
