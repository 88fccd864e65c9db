"""Float64 reference of the model-free objective and sampling kernels (csrc/ppo.cu, csrc/sac.cu and the GAE scan of
csrc/replay.cu) and first-order bounds on the error of an honest fp32 implementation of each output.

Like loss_ref, every function takes fp32 tensors on any device and computes in float64 on that device.  Each forward
is written from the reference's own definitions: policy_loss / value_loss / entropy_loss (ppo/loss.py),
normalize_tensor (utils/utils.py), PPOAgent's OneHotCategorical / Normal / tanh_normal glue (ppo/agent.py), the
masking rule of ppo_recurrent.py (normalise only when more than one row is kept), A2C's per-minibatch objective,
PPOPlayer's sampling, SACActor (clamp(log_std, -5, 2), rsample with the given noise, tanh, scale / bias and the
- log(scale (1 - y^2) + 1e-6) correction), the SAC target / critic / actor / temperature losses, DroQ's mean over
critics (droq.py:147-150) and `gae` (utils/utils.py).  Every gradient is float64 autograd of that forward.

The reference's quirks are kept, because the kernels keep them:
  - `_tanh_normal` applies 2 (log 2 - a - softplus(-2 a)) to the squashed action a, not to the pre-tanh x = atanh(a).
  - safeatanh / safetanh clamp at the fp32 value of 1 - finfo(float32).resolution (SAFE_LIM, 0.99999899).
  - `gae` masks step t's bootstrap with dones[t], the step's own flag (dones[-1] at the last step), not dones[t + 1].
  - PPOPlayer.get_actions with tanh_normal (ppo_act mode 3) returns safeatanh of the Normal sample; its log-prob is
    the Normal one of the sample.

Discrete decisions are taken as fp32 torch takes them on the same inputs, on the same device: the clip branch of
torch.min(pg1, pg2) and the value branch of torch.max(u, c) (an even split on a tie), the ratio and value clamps
(which pass the gradient at their bounds), the arg-min critic (first on ties) and the ppo_act argmax of p / q.  A
ratio within its own error bound of 1 +- clip may land on either side in fp32; on such a row (`ambiguous`) the dhead
bound also covers the jump between the two branches.  Scalar hyper-parameters are the fp32 values the kernel receives
(`f32`), and the ratio clamp bounds are fp32(1 -+ clip) as the kernel forms them.

Bounds (u = 2^-24, tau1(n) = u (16 + 2 sqrt n) for an fp32 reduction of length n; expf / tanhf within 2 ulp (4u),
logf / log1pf 1 ulp (2u), atanhf 3 ulp (6u)):
  - advantage normalisation over n rows, a = (x - m) / (s + 1e-8), s the unbiased std: E_m = tau1(n) sum|x| / n +
    2u |m|; each d = x - m off by E_m + u|d|; the variance by (sum (2|d| E_d + u d^2) + tau1(n) sum d^2) / (n - 1) +
    2u v; s by E_v / 2s + u s; a by E_d / (s + eps) + |d| E_inv + u |a|.  This carries the conditioning: an offset
    vector (|m| >> s) or a near-constant one makes E_m / s, and so the bound, grow.
  - a categorical head: the logsumexp's E_lse (loss_ref.lse_err), log p off by E_lse + u |log p|, p by that plus 4u
    relative, the entropy by sum p (e_p |log p| + E_lp) + tau1(K) sum |p log p|; heads summed with tau1(heads).
  - a Normal term -(x - mu)^2 / (2 sd^2) - ls - log sqrt(2 pi): x - mu off by E_x + u |d|, the square over sd^2 by
    2 |d| E_d / sd^2 + 12u z (sd = expf(ls) squared); x = atanh(a) within 6u; the tanh correction through softplus
    within 2 (E_sp + 2u (log 2 + |a| + sp)); actions drawn in fp32 carry sd e's and mu + sd e's roundings.
  - the ratio exp(lp - old) is off by r (E_lp + u |lp - old| + 4u); every later product or sum adds u of its result,
    each reduction over rows tau1(n) of the sum of |terms|, and the 1 / n the kernel rounds one more u.
  - SAC: std = expf(clamp(ls)) 4u; x_t = mean + std e; y = tanh(x_t) off by (1 - y^2) E_x + 4u |y|; 1 - y^2 by
    2 |y| E_y + u; the correction's log(w), w = scale (1 - y^2) + 1e-6, by E_w / w.  Near saturation (1 - y^2 ~ 1e-7)
    E_w / w is large: fp32 tanh cannot resolve 1 - y^2 there, and the 1e-6 is what keeps the log finite.
  - GAE: A_t = delta_t + nnt_t gamma lambda A_{t+1} carries its bound alongside the value, E_t = gamma lambda nnt_t
    E_{t+1} + E_delta + 2u |nnt gamma A_{t+1}| + u |A_t|, as loss_ref.lambda_returns does.
Each term is the worst case of one rounding in the order the kernels apply them; the bounds returned are twice their
sum (SAFETY), floored at TINY.

Input envelope: PPO's log-std is not clamped; below about -44 fp32 exp(2 ls) underflows (in torch too), and a Normal
sample whose (x - mu) / sd is not O(1) makes the ratio overflow, so log-std stays in [-20, 5] and stored actions are
draws from the head's own distribution.  An all-zero mask in ppo_loss_masked is not reachable from the recurrent
sampler (every sequence keeps at least its first step); the kernel writes zero losses and gradients there, where
torch's mean over no rows would be NaN, and `ppo_loss` below returns the kernel's zeros for it.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch
import torch.nn.functional as F
from torch import Tensor
from torch.distributions import Independent, Normal, OneHotCategorical

from oracle.loss_ref import SAFETY, TINY, _safe, f32, lse_err
from oracle.simt_ref import U, tau1

SAFE_LIM = f32(1.0 - float(torch.finfo(torch.float32).resolution))   # safetanh / safeatanh clamp, as fp32
EPS_NORM = f32(1e-8)                                                   # normalize_tensor's eps
EPS_SAC = f32(1e-6)                                                    # SACActor's + 1e-6
C0 = 0.5 * math.log(2 * math.pi)                                       # log sqrt(2 pi)
LOG2 = math.log(2.0)
LOG_STD_MIN, LOG_STD_MAX = -5.0, 2.0


def _d(t: Optional[Tensor]) -> Optional[Tensor]:
    return None if t is None else t.detach().double()


# ------------------------------------------------------------------------------------------------ shared pieces
def _segsum(t: Tensor, sid: Tensor, n_seg: int) -> Tensor:
    return torch.zeros(n_seg, dtype=t.dtype, device=t.device).index_add(0, sid, t)


def _tau1(n: Tensor) -> Tensor:
    return U * (16.0 + 2.0 * n.sqrt())


def normalize64(x: Tensor, sid: Optional[Tensor] = None, n_seg: int = 1):
    """normalize_tensor in float64 (unbiased std, + eps outside the root) and its bound, over the rows of each segment
    (segment ids `sid`, one segment without), every segment of at least two rows"""
    x = _d(x)
    sid = torch.zeros(x.numel(), dtype=torch.long, device=x.device) if sid is None else sid
    n = _segsum(torch.ones_like(x), sid, n_seg)
    m = _segsum(x, sid, n_seg) / n
    d = x - m[sid]
    v = _segsum(d * d, sid, n_seg) / (n - 1)
    s = v.sqrt()
    den = s + EPS_NORM
    a = d / den[sid]
    E_m = _tau1(n) * _segsum(x.abs(), sid, n_seg) / n + 2 * U * m.abs()
    E_d = E_m[sid] + U * d.abs()
    E_v = (_segsum(2 * d.abs() * E_d + U * d * d, sid, n_seg) + _tau1(n) * _segsum(d * d, sid, n_seg)) / (n - 1) \
        + 2 * U * v
    E_s = torch.where(s > 0, E_v / (2 * s) + U * s, E_v.sqrt())
    E_den = E_s + U * den
    E_inv = (E_den / den + U) / den
    return a, E_d / den[sid] + d.abs() * E_inv[sid] + U * a.abs()


def logp_entropy64(h: Tensor, act: Tensor, head_dims: Sequence[int], mode: int):
    """PPOAgent.forward's log-prob of the stored action and entropy, per row, differentiable in h (float64).
    mode 0 OneHotCategorical per head, 1 Normal, 2 tanh_normal (stored actions are squashed)."""
    act = _d(act)
    if mode == 0:
        lp = ent = 0.0
        o = 0
        for K in head_dims:
            dist = OneHotCategorical(logits=h[:, o:o + K])
            lp = lp + dist.log_prob(act[:, o:o + K])
            ent = ent + dist.entropy()
            o += K
        return lp, ent
    mean, ls = torch.chunk(h, 2, -1)
    normal = Independent(Normal(mean, ls.exp()), 1)
    if mode == 1:
        return normal.log_prob(act), normal.entropy()
    x = act.clamp(-SAFE_LIM, SAFE_LIM).atanh()
    corr = 2.0 * (LOG2 - act - F.softplus(-2.0 * act)).sum(-1)          # at the squashed action, as the reference
    return normal.log_prob(x) - corr, normal.entropy()


def _lpe32(head, act, head_dims, mode):
    """logp_entropy64 in fp32 torch: the values the reference's decisions are taken on"""
    if mode == 0:
        lp = ent = 0.0
        o = 0
        for K in head_dims:
            lg = torch.log_softmax(head[:, o:o + K], -1)
            lp = lp + (lg * act[:, o:o + K]).sum(-1)
            ent = ent - (lg.exp() * lg).sum(-1)
            o += K
        return lp, ent
    mean, ls = torch.chunk(head, 2, -1)
    x = act if mode == 1 else act.clamp(-SAFE_LIM, SAFE_LIM).atanh()
    lp = (-((x - mean) ** 2) / (2 * ls.exp() ** 2) - ls - C0).sum(-1)
    if mode == 2:
        lp = lp - 2.0 * (LOG2 - act - F.softplus(-2.0 * act)).sum(-1)
    return lp, (0.5 + C0 + ls).sum(-1)


def _cat_parts(h: Tensor, K: int):
    """per head of K logits: (log p, p, E_log p, relative error of p, entropy, E_entropy), no grad"""
    E_lse = lse_err(h)
    lg = h - torch.logsumexp(h, -1, keepdim=True)
    p = lg.exp()
    E_lg = E_lse + U * lg.abs()
    e_p = E_lg + 4 * U
    hh = -(p * lg).sum(-1, keepdim=True)
    E_hh = (p * (e_p * lg.abs() + E_lg)).sum(-1, keepdim=True) + tau1(K) * (p * lg).abs().sum(-1, keepdim=True) \
        + U * hh.abs()
    return lg, p, E_lg, e_p, hh, E_hh


def _normal_parts(h: Tensor, act: Tensor, mode: int):
    """per action column: (d, sd^2, z = d^2 / sd^2, E_d, E_z, lp_j, E_lp_j, corr_j, E_corr_j), no grad"""
    A = act.shape[1]
    mu, ls = h[:, :A], h[:, A:]
    if mode == 2:
        ac = act.clamp(-SAFE_LIM, SAFE_LIM)
        x = ac.atanh()
        E_x = 6 * U * x.abs()
    else:
        x, E_x = act, torch.zeros_like(act)
    d = x - mu
    s2 = (2 * ls).exp()
    z = d * d / s2
    E_d = E_x + U * d.abs()
    E_z = 2 * d.abs() * E_d / s2 + 12 * U * z
    lpj = -z / 2 - ls - C0
    E_lpj = E_z / 2 + 3 * U * (z / 2 + ls.abs() + C0)
    if mode == 2:
        v = -2 * act
        sp = F.softplus(v)
        E_sp = 2 * U * sp + 4 * U * torch.sigmoid(v)
        corr = 2 * (LOG2 - act - sp)
        E_corr = 2 * (E_sp + 2 * U * (LOG2 + act.abs() + sp)) + 2 * U * LOG2 + U * corr.abs()
    else:
        corr, E_corr = torch.zeros_like(act), torch.zeros_like(act)
    return d, s2, z, E_d, E_z, lpj, E_lpj, corr, E_corr


def dist_bounds(h: Tensor, act: Tensor, head_dims: Sequence[int], mode: int):
    """(E_lp, E_ent) per row of the kernel's row_logp_entropy"""
    h, act = _d(h), _d(act)
    if mode == 0:
        E_lp = E_ent = 0.0
        lps, hhs = [], []
        o = 0
        for K in head_dims:
            lg, p, E_lg, e_p, hh, E_hh = _cat_parts(h[:, o:o + K], K)
            a = act[:, o:o + K]
            lps.append((lg * a).sum(-1))
            E_lp = E_lp + (E_lg * a).sum(-1)
            hhs.append(hh.squeeze(-1))
            E_ent = E_ent + E_hh.squeeze(-1)
            o += K
        H = len(head_dims)
        lp_abs = torch.stack(lps, -1).abs()
        hh_abs = torch.stack(hhs, -1).abs()
        return E_lp + U * lp_abs.sum(-1) + tau1(H) * lp_abs.sum(-1), E_ent + tau1(H) * hh_abs.sum(-1)
    A = act.shape[1]
    ls = h[:, A:]
    d, s2, z, E_d, E_z, lpj, E_lpj, corr, E_corr = _normal_parts(h, act, mode)
    lp = lpj.sum(-1) - corr.sum(-1)
    E_lp = E_lpj.sum(-1) + E_corr.sum(-1) + tau1(A) * (lpj.abs().sum(-1) + corr.abs().sum(-1)) + U * lp.abs()
    entj = 0.5 + C0 + ls
    E_ent = (2 * U * (0.5 + C0 + ls.abs())).sum(-1) + tau1(A) * entj.abs().sum(-1)
    return E_lp, E_ent


def head_grad_bound(h: Tensor, act: Tensor, head_dims: Sequence[int], mode: int, dlp: Tensor, E_dlp: Tensor,
                    dent, E_dent) -> Tensor:
    """bound of row_head_grad: dlp d(log p)/dhead + dent d(entropy)/dhead, per element (dent, E_dent: scalars or
    [rows, 1])"""
    h, act = _d(h), _d(act)
    dlp, E_dlp = dlp.unsqueeze(-1), E_dlp.unsqueeze(-1)
    ad = dent.abs() if torch.is_tensor(dent) else abs(dent)
    if mode == 0:
        out = []
        o = 0
        for K in head_dims:
            lg, p, E_lg, e_p, hh, E_hh = _cat_parts(h[:, o:o + K], K)
            a = act[:, o:o + K]
            t1, t2 = dlp * (a - p), dent * p * (lg + hh)
            out.append(E_dlp * (a - p).abs() + dlp.abs() * p * e_p
                       + ad * (p * e_p * (lg + hh).abs() + p * (E_lg + E_hh + U * (lg + hh).abs()))
                       + E_dent * p * (lg + hh).abs() + 4 * U * (t1.abs() + t2.abs()) + 2 * U * (t1 - t2).abs()
                       + TINY * (dlp.abs() + ad * ((lg + hh).abs() + 1)))
            o += K
        return torch.cat(out, -1)
    d, s2, z, E_d, E_z, *_ = _normal_parts(h, act, mode)
    g_mu = dlp * d / s2
    b_mu = E_dlp * (d / s2).abs() + dlp.abs() * (E_d / s2 + 11 * U * d.abs() / s2) + U * g_mu.abs()
    g_ls = dlp * (z - 1) + dent
    b_ls = E_dlp * (z - 1).abs() + dlp.abs() * (E_z + U * (z - 1).abs()) + E_dent + 2 * U * ((dlp * (z - 1)).abs()
                                                                                         + g_ls.abs())
    return torch.cat((b_mu, b_ls), -1)


# ------------------------------------------------------------------------------------------------ PPO
def ppo_loss(head: Tensor, actions: Tensor, old_logp: Tensor, adv: Tensor, values: Tensor, old_values: Tensor,
             returns: Tensor, head_dims: Sequence[int], mode: int, clip_vloss: bool, normalize: bool, clip_coef: float,
             vf_coef: float, ent_coef: float, mask: Optional[Tensor] = None):
    """PPO's loss = policy_loss + vf_coef value_loss + ent_coef entropy_loss over the rows with mask != 0 (all rows
    without a mask), advantages normalised when `normalize` and more than one row is kept.  Outputs dhead [B, W],
    dvalues [B] (zero on dropped rows) and losses [3] = (policy, value, entropy).  Extra key `ambiguous`: rows whose
    ratio lies within its error bound of a clip bound."""
    c, vf, ec = f32(clip_coef), f32(vf_coef), f32(ent_coef)
    lo, hi = f32(1.0 - c), f32(1.0 + c)
    B, W = head.shape
    dev = head.device
    keep = torch.ones(B, dtype=torch.bool, device=dev) if mask is None else mask.reshape(-1) != 0
    idx = keep.nonzero().reshape(-1)
    n = idx.numel()
    out = {"dhead": torch.zeros(B, W, dtype=torch.float64, device=dev),
           "dvalues": torch.zeros(B, dtype=torch.float64, device=dev),
           "losses": torch.zeros(3, dtype=torch.float64, device=dev)}
    bound = {k: torch.zeros_like(v) for k, v in out.items()}
    out["ambiguous"] = torch.zeros(B, dtype=torch.bool, device=dev)
    if n == 0:
        return out, bound
    hd, act, old = head[idx], actions[idx], old_logp.reshape(-1)[idx]
    adv_k, val, oldv, ret = (t.reshape(-1)[idx] for t in (adv, values, old_values, returns))
    # fp32 torch decisions
    with torch.no_grad():
        lp32, _ = _lpe32(hd.float(), act.float(), head_dims, mode)
        a32 = adv_k.float()
        if normalize and n > 1:
            a32 = (a32 - a32.mean()) / (a32.std() + 1e-8)
        r32 = (lp32 - old.float()).exp()
        in_r = (r32 >= lo) & (r32 <= hi)
        p1, p2 = a32 * r32, a32 * r32.clamp(lo, hi)
        lt, gt = p1 < p2, p1 > p2
        dv32 = val.float() - oldv.float()
        in_v = (dv32 >= -c) & (dv32 <= c)
        vc32 = oldv.float() + dv32.clamp(-c, c)
        u32, c32 = (val.float() - ret.float()) ** 2, (vc32 - ret.float()) ** 2
        ugt, ult = u32 > c32, u32 < c32
    # float64 forward following those decisions, autograd backward
    h = _d(hd).requires_grad_(True)
    v = _d(val).requires_grad_(True)
    lp, ent = logp_entropy64(h, act, head_dims, mode)
    if normalize and n > 1:
        a, E_a = normalize64(adv_k)
    else:
        a, E_a = _d(adv_k), torch.zeros(n, dtype=torch.float64, device=dev)
    r = (lp - _d(old)).exp()
    rc = torch.where(in_r, r, r.clamp(lo, hi).detach())
    pg1, pg2 = a * r, a * rc
    pgm = torch.where(lt, pg1, torch.where(gt, pg2, 0.5 * (pg1 + pg2)))
    pg = -pgm.mean()
    ov, rt = _d(oldv), _d(ret)
    if clip_vloss:
        dv = v - ov
        vc = ov + torch.where(in_v, dv, dv.clamp(-c, c).detach())
        uu, cc = (v - rt) ** 2, (vc - rt) ** 2
        vl = 0.5 * torch.where(ugt, uu, torch.where(ult, cc, 0.5 * (uu + cc))).mean()
    else:
        vl = ((v - rt) ** 2).mean()
    el = (-ent).mean()
    (pg + vf * vl + ec * el).backward()
    out["dhead"][idx], out["dvalues"][idx] = h.grad, v.grad
    out["losses"] = torch.stack((pg, vl, el)).detach()
    # ---- bounds
    lpd, entd, rd, ad_ = lp.detach(), ent.detach(), r.detach(), a.detach()
    E_lp, E_ent = dist_bounds(hd, act, head_dims, mode)
    E_r = rd * (E_lp + U * (lpd - _d(old)).abs() + 4 * U)
    invn = 1.0 / n
    full = (~gt).double()                                         # the kernel's pg1 <= pg2: the unclipped gradient
    dlp = -ad_ * rd * invn * full
    E_dlp = invn * (E_a * rd + ad_.abs() * E_r) * full + 3 * U * dlp.abs()
    dent, E_dent = -ec * invn, 3 * U * abs(ec * invn)
    b_h = head_grad_bound(hd, act, head_dims, mode, dlp, E_dlp, dent, E_dent)
    amb = (((rd - lo).abs() <= 2 * E_r) | ((rd - hi).abs() <= 2 * E_r)) & (ad_ != 0)
    if bool(amb.any()):                                          # either branch: add the jump |adv r / n| |dlp/dh|
        hj = _d(hd).requires_grad_(True)
        lpj, _ = logp_entropy64(hj, act, head_dims, mode)
        w = torch.where(amb, (ad_ * rd).abs() * invn + E_dlp, torch.zeros_like(rd))
        (lpj * w).sum().backward()
        b_h = b_h + hj.grad.abs()
    out["ambiguous"][idx] = amb
    rcd = rc.detach()
    pgd = pgm.detach()
    E_pg_row = E_a * rcd + ad_.abs() * E_r + 2 * U * pgd.abs()
    b_pg = (E_pg_row.sum() + tau1(n) * pgd.abs().sum()) * invn + 2 * U * pg.detach().abs()
    vd = _d(val)
    gu = vd - rt
    E_gu = U * gu.abs()
    if clip_vloss:
        dvd = vd - ov
        ind = in_v.double()
        vcd = ov + torch.where(in_v, dvd, dvd.clamp(-c, c))
        gcv = vcd - rt
        E_gc = ind * U * dvd.abs() + U * vcd.abs() + U * gcv.abs()
        E_u, E_c = 2 * gu.abs() * E_gu + U * gu * gu, 2 * gcv.abs() * E_gc + U * gcv * gcv
        rowv = 0.5 * torch.maximum(gu * gu, gcv * gcv)
        b_vl = (0.5 * (E_u + E_c).sum() + (tau1(n) + U) * rowv.sum()) * invn + 2 * U * vl.detach().abs()
        wu = torch.where(ugt, 1.0, torch.where(ult, 0.0, 0.5)).double()
        E_dvr = wu * E_gu + (1 - wu) * ind * E_gc
        b_dv = abs(vf) * invn * E_dvr + 4 * U * v.grad.abs()
    else:
        b_vl = (3 * U * (gu * gu).sum() + tau1(n) * (gu * gu).sum()) * invn + 2 * U * vl.detach().abs()
        b_dv = 5 * U * v.grad.abs()
    b_el = (E_ent.sum() + tau1(n) * entd.abs().sum()) * invn + 2 * U * el.detach().abs()
    bound["dhead"][idx], bound["dvalues"][idx] = b_h, b_dv
    bound["losses"] = torch.stack((b_pg, b_vl, b_el))
    return out, _safe(bound)


# ------------------------------------------------------------------------------------------------ A2C
def a2c_loss(head: Tensor, actions: Tensor, adv: Tensor, values: Tensor, returns: Tensor, seg: int,
             head_dims: Sequence[int], mode: int, normalize: bool, reduce_sum: bool, vf_coef: float, ent_coef: float):
    """A2C's objective per minibatch i = rows [i seg, min(N, (i + 1) seg)): pg = -(log p adv), v = (value - return)^2,
    ent = -entropy, each reduced by mean or sum, advantages normalised over the minibatch; the gradient of each
    minibatch's pg + vf v + ent_coef ent lands on its own rows.  losses [n_seg, 3]."""
    vf, ec = f32(vf_coef), f32(ent_coef)
    N, W = head.shape
    dev = head.device
    n_seg = (N + seg - 1) // seg
    sid = torch.arange(N, device=dev) // seg
    n = _segsum(torch.ones(N, dtype=torch.float64, device=dev), sid, n_seg)
    sc = torch.ones_like(n) if reduce_sum else 1.0 / n
    h = _d(head).requires_grad_(True)
    v = _d(values).reshape(-1).requires_grad_(True)
    lp, ent = logp_entropy64(h, actions, head_dims, mode)
    rt = _d(returns).reshape(-1)
    if normalize:
        a, E_a = normalize64(adv.reshape(-1), sid, n_seg)
    else:
        a, E_a = _d(adv).reshape(-1), torch.zeros(N, dtype=torch.float64, device=dev)
    pgr, vlr, elr = -(lp * a), (v - rt) ** 2, -ent
    pg, vl, el = (sc * _segsum(t, sid, n_seg) for t in (pgr, vlr, elr))
    (pg + vf * vl + ec * el).sum().backward()
    # bounds; the kernel rounds 1 / n once more under `mean`
    E_lp, E_ent = dist_bounds(head, actions, head_dims, mode)
    sr = 0.0 if reduce_sum else U
    pgd, vld, eld, lpd = pgr.detach(), vlr.detach(), elr.detach(), lp.detach()
    t1 = _tau1(n)
    b_pg = sc * (_segsum(E_lp * a.abs() + lpd.abs() * E_a + U * pgd.abs(), sid, n_seg)
                 + t1 * _segsum(pgd.abs(), sid, n_seg)) + (U + sr) * pg.detach().abs()
    b_vl = sc * (3 * U + t1) * _segsum(vld, sid, n_seg) + (U + sr) * vl.detach().abs()
    b_el = sc * (_segsum(E_ent, sid, n_seg) + t1 * _segsum(eld.abs(), sid, n_seg)) + (U + sr) * el.detach().abs()
    scr = sc[sid]
    dlp = -a * scr
    E_dlp = scr * (E_a + U * a.abs()) + 2 * U * dlp.abs()
    dent = (-ec * scr).unsqueeze(-1)
    b_h = head_grad_bound(head, actions, head_dims, mode, dlp, E_dlp, dent, 3 * U * dent.abs())
    out = {"dhead": h.grad, "dvalues": v.grad, "losses": torch.stack((pg, vl, el), -1).detach()}
    bound = {"dhead": b_h, "dvalues": 5 * U * v.grad.abs(), "losses": torch.stack((b_pg, b_vl, b_el), -1)}
    return out, _safe(bound)


# ------------------------------------------------------------------------------------------------ acting
def ppo_act_decision(head: Tensor, noise: Optional[Tensor], head_dims: Sequence[int], greedy: bool) -> Tensor:
    """the discrete actions as fp32 torch draws them: argmax of softmax / noise per head (first on ties)"""
    out, o = [], 0
    for K in head_dims:
        p = torch.log_softmax(head[:, o:o + K].float(), -1).exp()
        if not greedy and noise is not None:
            p = p / noise[:, o:o + K].float()
        out.append(F.one_hot(p.argmax(-1), K).float())
        o += K
    return torch.cat(out, -1)


def ppo_act(head: Tensor, noise: Optional[Tensor], head_dims: Sequence[int], mode: int, greedy: bool):
    """PPOPlayer: mode 0 one-hot actions (fp32 torch's decision) and their log-prob; 1 Normal sample mean + std e
    (the mean when greedy) and its log-prob; 2 tanh_normal as PPOPlayer.forward (safetanh of the sample, corrected
    log-prob); 3 tanh_normal as PPOPlayer.get_actions (safeatanh of the sample; the Normal log-prob)."""
    h = _d(head)
    if mode == 0:
        onehot = ppo_act_decision(head, noise, head_dims, greedy)
        lp, _ = logp_entropy64(h, onehot, head_dims, 0)
        E_lp, _ = dist_bounds(head, onehot, head_dims, 0)
        return {"actions": onehot.double(), "logp": lp}, {"logp": SAFETY * E_lp + TINY}
    A = sum(head_dims)
    mu, ls = h[:, :A], h[:, A:]
    sd = ls.exp()
    e = torch.zeros_like(mu) if (greedy or noise is None) else _d(noise)
    x = mu + sd * e
    lpj = -e * e / 2 - ls - C0
    sde = (sd * e).abs()
    E_x = 5 * U * sde + U * x.abs()
    E_d = E_x + U * sde
    E_lpj = sde * E_d / (sd * sd) + 11 * U * e * e / 2 + 3 * U * (e * e / 2 + ls.abs() + C0)
    lp = lpj.sum(-1)
    E_lp = E_lpj.sum(-1) + tau1(A) * lpj.abs().sum(-1)
    if mode == 1:
        a, E_a = x, E_x
    elif mode == 2:
        y = x.tanh()
        a = y.clamp(-SAFE_LIM, SAFE_LIM)
        E_a = (1 - y * y) * E_x + 4 * U * y.abs()
        v = -2 * a
        sp = F.softplus(v)
        corr = 2 * (LOG2 - a - sp)
        E_corr = 2 * (2 * torch.sigmoid(v) - 1).abs() * E_a + 2 * (2 * U * sp + 4 * U * torch.sigmoid(v)) \
            + 4 * U * (LOG2 + a.abs() + sp) + 2 * U * LOG2 + U * corr.abs()
        lp = lp - corr.sum(-1)
        E_lp = E_lp + E_corr.sum(-1) + tau1(A) * corr.abs().sum(-1)
    else:
        xc = x.clamp(-SAFE_LIM, SAFE_LIM)
        a = xc.atanh()
        inside = (x.abs() < SAFE_LIM).double()
        E_a = inside * E_x / (1 - xc * xc) + 6 * U * a.abs()
    E_lp = E_lp + U * lp.abs()
    return {"actions": a, "logp": lp}, _safe({"actions": E_a, "logp": E_lp})


# ------------------------------------------------------------------------------------------------ SAC
def sac_sample_fwd(head: Tensor, eps: Tensor, scale: Tensor, bias: Tensor):
    """SACActor.forward: action = tanh(mean + exp(clamp(ls, -5, 2)) eps) scale + bias, logp per row, and y = tanh"""
    B, A = eps.shape
    h, e, s, b = _d(head), _d(eps), _d(scale), _d(bias)
    mean, raw = h[:, :A], h[:, A:]
    lsc = raw.clamp(LOG_STD_MIN, LOG_STD_MAX)
    std = lsc.exp()
    normal = Normal(mean, std)
    xt = mean + std * e
    y = xt.tanh()
    act = y * s + b
    omy = 1 - y * y
    w = s * omy + EPS_SAC
    lp = (normal.log_prob(xt) - torch.log(w)).sum(-1)
    out = {"action": act, "logp": lp, "tanh": y}
    E_std = 4 * U * std
    E_xt = e.abs() * E_std + U * (std * e).abs() + U * xt.abs()
    E_y = omy * E_xt + 4 * U * y.abs()
    E_om = 2 * y.abs() * E_y + U * y * y + U * omy
    E_w = s.abs() * E_om + U * (s * omy).abs() + 2 * U * w
    E_d = E_xt + U * (xt - mean).abs()
    z = e * e
    E_q = (std * e).abs() * E_d / (std * std) + 11 * U * z / 2
    lw = torch.log(w)
    E_j = E_q + 4 * U + 2 * U * lsc.abs() + E_w / w + 2 * U * lw.abs() + 4 * U * (z / 2 + lsc.abs() + C0 + lw.abs())
    lpj = -z / 2 - lsc - C0 - lw
    bound = {"action": s.abs() * E_y + U * (y * s).abs() + U * act.abs(),
             "logp": E_j.sum(-1) + tau1(A) * lpj.abs().sum(-1) + U * lp.abs(),
             "tanh": E_y}
    return out, _safe(bound)


def sac_sample_bwd(head: Tensor, eps: Tensor, scale: Tensor, dact: Tensor, log_alpha: Tensor,
                   batch: Optional[int] = None):
    """dhead = d(sum dact_sum action + (alpha / batch) sum logp) / dhead through SACActor, dact_sum = sum over nets of
    dact [nets, B, A]; clamp passes the gradient on [-5, 2].  `batch` (the whole minibatch, default B) sets the 1 / B
    of the mean, so that rows can be checked a chunk at a time.  The kernel reads y = tanh(x_t) from the forward: its
    error (the first-order E_y of sac_sample_fwd) is an input error here."""
    B, A = eps.shape
    batch = B if batch is None else batch
    nets = dact.shape[0]
    h = _d(head).requires_grad_(True)
    e, s = _d(eps), _d(scale)
    alpha = math.exp(float(log_alpha.reshape(-1)[0]))
    mean, raw = h[:, :A], h[:, A:]
    std = raw.clamp(LOG_STD_MIN, LOG_STD_MAX).exp()
    xt = mean + std * e
    y = xt.tanh()
    lp = (Normal(mean, std).log_prob(xt) - torch.log(s * (1 - y * y) + EPS_SAC)).sum(-1)
    dn = _d(dact)
    da = dn.sum(0)
    ((da * (y * s)).sum() + (alpha / batch) * lp.sum()).backward()
    # bounds
    std, xt, y = std.detach(), xt.detach(), y.detach()
    dl = alpha / batch
    E_dl = 6 * U * dl
    omy = 1 - y * y
    E_xt = e.abs() * 4 * U * std + U * (std * e).abs() + U * xt.abs()
    E_y = omy * E_xt + 4 * U * y.abs()
    E_om = 2 * y.abs() * E_y + U * y * y + U * omy
    w = s * omy + EPS_SAC
    E_w = s.abs() * E_om + U * (s * omy).abs() + 2 * U * w
    E_da = tau1(nets) * dn.abs().sum(0)
    T1 = da * s * omy
    E_T1 = E_da * (s * omy).abs() + (da * s).abs() * E_om + 2 * U * T1.abs()
    num = 2 * s * y * omy
    E_num = 2 * s.abs() * (omy * E_y + y.abs() * E_om) + 3 * U * num.abs()
    T2 = dl * num / w
    E_T2 = dl * (E_num / w + num.abs() * E_w / (w * w)) + E_dl * (num / w).abs() + 2 * U * T2.abs()
    dxt = T1 + T2
    E_dxt = E_T1 + E_T2 + U * dxt.abs()
    dstd = dxt * e - dl / std
    E_dstd = E_dxt * e.abs() + U * (dxt * e).abs() + E_dl / std + 5 * U * dl / std + U * dstd.abs()
    pss = ((raw.detach() >= LOG_STD_MIN) & (raw.detach() <= LOG_STD_MAX)).double()
    b_ls = pss * (E_dstd * std + 5 * U * (dstd * std).abs())
    return {"dhead": h.grad}, _safe({"dhead": torch.cat((E_dxt, b_ls), -1)})


def sac_target(q_target: Tensor, logp: Tensor, rewards: Tensor, terminated: Tensor, log_alpha: Tensor, gamma: float):
    """SACAgent.get_next_target_q_values: r + (1 - done) gamma (min over critics - alpha logp')"""
    g = f32(gamma)
    q, lp, r, d = _d(q_target), _d(logp).reshape(-1), _d(rewards).reshape(-1), _d(terminated).reshape(-1)
    alpha = math.exp(float(log_alpha.reshape(-1)[0]))
    m = q.min(0).values
    inner = m - alpha * lp
    y = r + (1 - d) * g * inner
    E_in = 6 * U * (alpha * lp).abs() + U * inner.abs()
    E_y = ((1 - d) * g).abs() * E_in + 2 * U * ((1 - d) * g * inner).abs() + U * y.abs()
    return {"y": y}, _safe({"y": E_y})


def sac_critic_loss(q: Tensor, y: Tensor):
    """critic_loss: sum over critics of mse_loss(q_n, y), and its gradient 2 (q - y) / B"""
    nets, B = q.shape
    qq = _d(q).requires_grad_(True)
    yy = _d(y).reshape(1, -1)
    loss = sum(F.mse_loss(qq[n], yy[0]) for n in range(nets))
    loss.backward()
    dd = (qq.detach() - yy) ** 2
    return ({"loss": loss.detach().reshape(1), "dq": qq.grad},
            _safe({"loss": ((tau1(nets * B) + 3 * U) * dd.sum() / B + 2 * U * loss.detach().abs()).reshape(1),
                   "dq": 4 * U * qq.grad.abs()}))


def sac_actor_loss(q: Tensor, logp: Tensor, log_alpha: Tensor, target_entropy: float, mean_over_critics: bool):
    """policy_loss(alpha, logp, Q) with Q the min over critics (SAC; torch.min's index, first on ties) or their mean
    (DroQ), entropy_loss(log_alpha, logp, target_entropy), dq = d policy_loss / dq and dlog_alpha = d alpha_loss /
    d log_alpha"""
    nets, B = q.shape
    te = f32(target_entropy)
    qq = _d(q).requires_grad_(True)
    la = _d(log_alpha).reshape(-1)[:1].requires_grad_(True)
    lp = _d(logp).reshape(-1)
    alpha = float(la.detach().exp())
    Q = qq.mean(0) if mean_over_critics else qq.min(0).values
    actor = (alpha * lp - Q).mean()
    alpha_l = (-la * (lp + te)).mean()
    actor.backward()
    alpha_l.backward()
    Qd = Q.detach()
    E_Q = tau1(nets) * qq.detach().abs().sum(0) / nets + 2 * U * Qd.abs() if mean_over_critics else 0.0
    t = alpha * lp - Qd
    E_t = 6 * U * (alpha * lp).abs() + E_Q + U * t.abs()
    b_actor = (E_t.sum() + tau1(B) * t.abs().sum()) / B + 2 * U * actor.detach().abs()
    se = lp + te
    E_se = (U * se.abs() + tau1(B) * se.abs()).sum() / B
    dla = la.grad
    out = {"actor_loss": actor.detach().reshape(1), "alpha_loss": alpha_l.detach().reshape(1), "dlog_alpha": dla,
           "dq": qq.grad}
    bound = {"actor_loss": b_actor.reshape(1),
             "alpha_loss": (la.detach().abs() * E_se + 3 * U * alpha_l.detach().abs()).reshape(1),
             "dlog_alpha": E_se.reshape(1) + 2 * U * dla.abs(),
             "dq": 3 * U * qq.grad.abs()}
    return out, _safe(bound)


# ------------------------------------------------------------------------------------------------ GAE
def gae(rewards: Tensor, values: Tensor, dones: Tensor, next_value: Tensor, gamma: float, lmbda: float):
    """utils.gae over [T, E]: nextnonterminal = not dones[t] at every step (dones[-1] at the last), nextvalues =
    values[t + 1] or next_value; returns (returns, advantages) with the recurrence's carried bound"""
    g, lm = f32(gamma), f32(lmbda)
    r, v, d = _d(rewards), _d(values), _d(dones)
    T = r.shape[0]
    nv = _d(next_value).reshape(v[0].shape)
    nnt = 1.0 - (d != 0).double()
    adv = torch.zeros_like(r)
    E = torch.zeros_like(r)
    A_next, E_next = torch.zeros_like(nv), torch.zeros_like(nv)
    for t in reversed(range(T)):
        nxt = nv if t == T - 1 else v[t + 1]
        boot = nxt * nnt[t] * g
        delta = r[t] + boot - v[t]
        carry = nnt[t] * A_next * g * lm
        A = delta + carry
        E_delta = U * boot.abs() + U * (r[t] + boot).abs() + U * delta.abs()
        E_t = nnt[t] * g * lm * E_next + E_delta + U * (nnt[t] * A_next * g).abs() + U * carry.abs() + U * A.abs()
        adv[t], E[t] = A, E_t
        A_next, E_next = A, E_t
    ret = adv + v
    return {"returns": ret, "advantages": adv}, _safe({"returns": E + U * ret.abs(), "advantages": E})
