"""TEST INFRASTRUCTURE — executable specification (plain fp32 torch, CPU) of every C-ABI op in
`include/b200rl.h`.  One method per `b200rl_*` entry point, same argument meaning, operating on torch
tensors in place.

Two uses, both in tests only:
  * `-m gpu` tests compare each CUDA kernel against the method of the same name on seeded inputs;
  * `-m "not gpu"` tests inject this object into `sheeprl_b200.engine.DV3Engine` (test double) to
    validate the engine's hand-written backward orchestration against the autograd oracle on CPU.
The product never constructs this class: `DV3Engine` without an injected ops object loads the CUDA
library and raises if it (or a GPU) is missing.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
FP32_EPS = 1.1920928955078125e-07
ACT_NONE, ACT_SILU, ACT_TANH, ACT_RELU = 0, 1, 2, 3
SAFE_LIM = 1.0 - 1e-6        # safetanh / safeatanh clamp (sheeprl/utils/utils.py:304-313)


def _symlog(x):
    return torch.sign(x) * torch.log(1 + torch.abs(x))


def _symexp(x):
    return torch.sign(x) * (torch.exp(torch.abs(x)) - 1)


class EmulOps:
    name = "emul"

    # ---------------------------------------------------------------- GEMM family
    def gemm(self, A: Tensor, B: Tensor, C: Tensor, transA: bool, transB: bool,
             bias: Optional[Tensor] = None, accumulate: bool = False):
        """C[M,N] = op(A) @ op(B) (+bias[N]) (+C).  A: [M,K] or [K,M] if transA; B: [K,N] or [N,K] if
        transB.  2-D views with unit inner stride."""
        a = A.t() if transA else A
        b = B.t() if transB else B
        r = a @ b
        if bias is not None:
            r = r + bias
        if accumulate:
            C.add_(r)
        else:
            C.copy_(r)

    def col_sum(self, X: Tensor, out: Tensor, accumulate: bool = False):
        r = X.sum(0)
        out.add_(r) if accumulate else out.copy_(r)

    # ---------------------------------------------------------------- LayerNorm (+SiLU)
    def ln_act_fwd(self, X: Tensor, gamma: Tensor, beta: Tensor, eps: float, act: int, Y: Tensor):
        y = F.layer_norm(X, (X.shape[-1],), gamma, beta, eps)
        if act == ACT_SILU:
            y = F.silu(y)
        elif act == ACT_TANH:
            y = torch.tanh(y)
        elif act == ACT_RELU:
            y = torch.relu(y)
        Y.copy_(y)

    def ln_act_bwd(self, X: Tensor, gamma: Tensor, beta: Tensor, eps: float, act: int, dY: Tensor,
                   dX: Tensor, dgamma: Optional[Tensor], dbeta: Optional[Tensor], accumulate: bool = False):
        """Recomputes LN from X.  dX may alias dY.  dgamma/dbeta (+)= column sums (None: skipped)."""
        mu = X.mean(-1, keepdim=True)
        var = ((X - mu) ** 2).mean(-1, keepdim=True)
        rstd = torch.rsqrt(var + eps)
        xh = (X - mu) * rstd
        ln = xh * gamma + beta
        if act == ACT_SILU:
            s = torch.sigmoid(ln)
            dln = dY * (s * (1 + ln * (1 - s)))
        elif act == ACT_TANH:
            dln = dY * (1 - torch.tanh(ln) ** 2)
        elif act == ACT_RELU:
            dln = dY * (ln > 0).to(dY.dtype)
        else:
            dln = dY.clone()
        if dgamma is not None:
            dg, db = (dln * xh).sum(0), dln.sum(0)
            if accumulate:
                dgamma.add_(dg), dbeta.add_(db)
            else:
                dgamma.copy_(dg), dbeta.copy_(db)
        dxh = dln * gamma
        dX.copy_(rstd * (dxh - dxh.mean(-1, keepdim=True) - xh * (dxh * xh).mean(-1, keepdim=True)))

    # ---------------------------------------------------------------- stride-2 k4 p1 convolutions (NHWC)
    def obs_prep(self, obs: Tensor, out: Tensor):
        """obs [N,C,H,W] uint8 or float (0..255) -> out [N,H,W,C] fp32 = obs/255 - 0.5."""
        out.copy_((obs.float() / 255.0 - 0.5).permute(0, 2, 3, 1))

    def transpose_batched(self, X: Tensor, Y: Tensor):
        """X [N,a,b] -> Y [N,b,a]."""
        Y.copy_(X.transpose(1, 2))

    def conv_down(self, big: Tensor, W: Tensor, small: Tensor):
        """small[n,y,x,cs] = sum_{ky,kx,cb} big[n,2y-1+ky,2x-1+kx,cb] * W[cs,cb,ky,kx]."""
        r = F.conv2d(big.permute(0, 3, 1, 2), W, None, stride=2, padding=1)
        small.copy_(r.permute(0, 2, 3, 1))

    def conv_up(self, small: Tensor, W: Tensor, big: Tensor, bias: Optional[Tensor] = None):
        """big[n,Y,X,cb] = sum_{cs,(y,ky):2y-1+ky=Y,(x,kx):2x-1+kx=X} small[n,y,x,cs]*W[cs,cb,ky,kx] (+bias)."""
        r = F.conv_transpose2d(small.permute(0, 3, 1, 2), W, bias, stride=2, padding=1)
        big.copy_(r.permute(0, 2, 3, 1))

    def conv_wgrad(self, small: Tensor, big: Tensor, dW: Tensor, accumulate: bool = False):
        """dW[cs,cb,ky,kx] (+)= sum_{n,y,x} small[n,y,x,cs] * big[n,2y-1+ky,2x-1+kx,cb]."""
        N, h, w, Cs = small.shape
        Cb = big.shape[-1]
        bp = F.pad(big, (0, 0, 1, 1, 1, 1))                       # pad H and W by 1
        r = torch.empty(Cs, Cb, 4, 4)
        sm = small.reshape(-1, Cs)
        for ky in range(4):
            for kx in range(4):
                patch = bp[:, ky:ky + 2 * h:2, kx:kx + 2 * w:2, :].reshape(-1, Cb)
                r[:, :, ky, kx] = sm.t() @ patch
        dW.add_(r) if accumulate else dW.copy_(r)

    # ---------------------------------------------------------------- RSSM element-wise pieces
    def gru_gate_fwd(self, G: Tensor, Hin: Tensor, Hout: Tensor):
        """G [M,3R] post-LayerNorm (reset|cand|update), Hin/Hout [M,R]."""
        r, c, u = torch.chunk(G, 3, -1)
        c = torch.tanh(torch.sigmoid(r) * c)
        u = torch.sigmoid(u - 1)
        Hout.copy_(u * c + (1 - u) * Hin)

    def gru_gate_bwd(self, G: Tensor, Hin: Tensor, dH: Tensor, dG: Tensor, dHin: Tensor):
        """dH: grad wrt gate output.  dG [M,3R] grad wrt post-LN G; dHin = dH*(1-u) (written, not added)."""
        gr, gc, gu = torch.chunk(G, 3, -1)
        r = torch.sigmoid(gr)
        c = torch.tanh(r * gc)
        u = torch.sigmoid(gu - 1)
        du = dH * (c - Hin)
        drc = dH * u * (1 - c * c)
        dG.copy_(torch.cat((drc * gc * r * (1 - r), drc * r, du * u * (1 - u)), -1))
        dHin.copy_(dH * (1 - u))

    def mask_mix(self, prev: Tensor, init: Tensor, first: Tensor, out: Tensor):
        """out[m,:] = (1-f[m])*prev[m,:] + f[m]*init[:]   (init is a single row; prev None -> zeros)."""
        f = first.reshape(-1, 1)
        p = prev if prev is not None else torch.zeros_like(out)
        out.copy_((1 - f) * p + f * init.reshape(1, -1))

    def mask_rows(self, X: Tensor, first: Tensor, out: Tensor):
        """out = (1-f[m]) * X[m,:]"""
        out.copy_((1 - first.reshape(-1, 1)) * X)

    def mask_bwd(self, dIn: Tensor, first: Tensor, dPrev: Tensor, dInit: Tensor):
        """dPrev = (1-f)*dIn ;  dInit[:] += sum_m f[m]*dIn[m,:]"""
        f = first.reshape(-1, 1)
        dPrev.copy_((1 - f) * dIn)
        if dInit is not None:
            dInit.add_((f * dIn).sum(0))

    def cat_sample(self, raw: Tensor, noise: Optional[Tensor], unimix: float, groups: int, classes: int,
                   onehot: Tensor, mix_out: Optional[Tensor] = None):
        """raw [M,groups*classes] logits -> unimix log-probs (optionally stored) -> one-hot sample
        argmax(p / q) per group (q=None: mode)."""
        M = raw.shape[0]
        x = raw.reshape(M, groups, classes)
        if unimix > 0:
            pr = (1 - unimix) * torch.softmax(x, -1) + unimix / classes
            x = torch.log(pr.clamp(FP32_EPS, 1 - FP32_EPS))
        if mix_out is not None:
            mix_out.copy_(x.reshape(M, -1))
        p = torch.softmax(x - torch.logsumexp(x, -1, keepdim=True), -1)
        if noise is not None:
            p = p / noise.reshape(M, groups, classes)
        if onehot is not None:
            onehot.copy_(F.one_hot(p.argmax(-1), classes).float().reshape(M, -1))

    def cat_sample_bwd(self, raw: Tensor, dz: Optional[Tensor], dmix: Optional[Tensor], unimix: float, groups: int,
                       classes: int, draw: Tensor):
        """Gradient wrt raw logits given (a) dz: grad wrt the straight-through sample (= grad wrt the
        normalised probs) and (b) dmix: grad wrt the unimix log-probs (from the KL).  Either may be None."""
        M = raw.shape[0]
        x = raw.reshape(M, groups, classes)
        s = torch.softmax(x, -1)
        if unimix > 0:
            pm = (1 - unimix) * s + unimix / classes
            pmc = pm.clamp(FP32_EPS, 1 - FP32_EPS)
            mix = torch.log(pmc)
        else:
            mix = x
        g = torch.zeros_like(x)
        if dmix is not None:
            g = g + dmix.reshape(M, groups, classes)
        if dz is not None:
            p = torch.softmax(mix - torch.logsumexp(mix, -1, keepdim=True), -1)
            d = dz.reshape(M, groups, classes)
            g = g + p * (d - (p * d).sum(-1, keepdim=True))
        if unimix > 0:
            inside = (pm >= FP32_EPS) & (pm <= 1 - FP32_EPS)
            ds = torch.where(inside, g * (1 - unimix) / pmc, torch.zeros_like(g))
            g = s * (ds - (s * ds).sum(-1, keepdim=True))
        draw.copy_(g.reshape(M, -1))

    # ---------------------------------------------------------------- losses (forward value + seed gradient)
    def kl_loss_grad(self, post_mix: Tensor, prior_mix: Tensor, groups: int, classes: int, kl_dyn: float,
                     kl_rep: float, free_nats: float, regularizer: float, scale: float,
                     d_post: Tensor, d_prior: Tensor, rows: Tensor):
        """Per row m: kl = KL(post||prior) summed over groups (torch Categorical semantics).
        loss_state = dyn*max(kl,free)+rep*max(kl,free).  rows[m] = (kl, loss_state, H(post), H(prior)).
        d_post / d_prior: gradient of `scale * regularizer * loss_state` wrt the unimix log-probs."""
        M = post_mix.shape[0]
        lp = post_mix.reshape(M, groups, classes)
        lq = prior_mix.reshape(M, groups, classes)
        lp = lp - torch.logsumexp(lp, -1, keepdim=True)
        lq = lq - torch.logsumexp(lq, -1, keepdim=True)
        pp, pq = torch.exp(lp), torch.exp(lq)
        t = pp * (lp - lq)
        klg = t.sum(-1)                                     # [M, groups]
        kl = klg.sum(-1)
        rows[:, 0] = kl
        rows[:, 1] = (kl_dyn + kl_rep) * torch.clamp(kl, min=free_nats)
        rows[:, 2] = -(pp * lp).sum(-1).sum(-1)
        rows[:, 3] = -(pq * lq).sum(-1).sum(-1)
        live = (kl > free_nats).float().reshape(M, 1, 1) * (scale * regularizer)
        d_prior.copy_((kl_dyn * live * (pq - pp)).reshape(M, -1))
        d_post.copy_((kl_rep * live * pp * ((lp - lq) - klg.unsqueeze(-1))).reshape(M, -1))

    def mse_loss_grad(self, pred: Tensor, target: Tensor, scale: float, loss_row: Tensor, grad: Tensor):
        """pred/target [M,P]; loss_row[m] = sum (pred-target)^2 ; grad = 2*(pred-target)*scale (may alias pred)."""
        d = pred - target
        loss_row.copy_((d * d).sum(-1))
        grad.copy_(2 * scale * d)

    def twohot_loss_grad(self, logits: Tensor, x: Tensor, weight: Optional[Tensor], scale: float, low: float,
                         high: float, loss_row: Tensor, dlogits: Tensor, accumulate: bool = False):
        """loss_row[m] (+)= -TwoHot(logits).log_prob(x[m]);  dlogits (+)= (softmax - target)*scale*weight[m]."""
        nb = logits.shape[-1]
        bins = torch.linspace(low, high, nb)
        xs = _symlog(x.reshape(-1, 1))
        below = (bins <= xs).to(torch.int32).sum(-1, keepdim=True) - 1
        above = torch.clamp(below + 1, max=nb - 1)
        below = torch.clamp(below, min=0)
        same = below == above
        d_lo = torch.where(same, torch.ones_like(xs), (bins[below] - xs).abs())
        d_hi = torch.where(same, torch.ones_like(xs), (bins[above] - xs).abs())
        tot = d_lo + d_hi
        target = torch.zeros_like(logits)
        target.scatter_add_(1, below.long(), d_hi / tot)
        target.scatter_add_(1, above.long(), d_lo / tot)
        logp = logits - torch.logsumexp(logits, -1, keepdim=True)
        w = torch.ones(logits.shape[0]) if weight is None else weight.reshape(-1)
        lr = -(target * logp).sum(-1)
        g = (torch.exp(logp) * target.sum(-1, keepdim=True) - target) * (scale * w).unsqueeze(-1)
        if accumulate:
            loss_row.add_(lr), dlogits.add_(g)
        else:
            loss_row.copy_(lr), dlogits.copy_(g)

    def bce_loss_grad(self, logit: Tensor, target: Tensor, loss_scale: float, scale: float, loss_row: Tensor,
                      dlogit: Tensor):
        l, y = logit.reshape(-1), target.reshape(-1)
        loss_row.copy_(loss_scale * F.binary_cross_entropy_with_logits(l, y, reduction="none"))
        dlogit.reshape(-1).copy_(loss_scale * scale * (torch.sigmoid(l) - y))

    def twohot_mean(self, logits: Tensor, low: float, high: float, out: Tensor):
        bins = torch.linspace(low, high, logits.shape[-1])
        out.reshape(-1).copy_(_symexp((torch.softmax(logits, -1) * bins).sum(-1)))

    def lambda_returns(self, rew: Tensor, val: Tensor, cont_logit: Tensor, true_cont: Tensor, gamma: float,
                       lmbda: float, lam: Tensor, discount: Tensor):
        """rew/val/cont_logit [H+1,N]; true_cont [N]; lam [H,N]; discount [H+1,N].
        (dreamer_v3.py:246-260, utils.py:66-77)"""
        H = rew.shape[0] - 1
        cont = (torch.sigmoid(cont_logit) > 0.5).float()
        cont = torch.cat((true_cont.reshape(1, -1), cont[1:]), 0)
        c = cont[1:] * gamma
        interm = rew[1:] + c * val[1:] * (1 - lmbda)
        nxt = val[-1]
        for t in reversed(range(H)):
            nxt = interm[t] + c[t] * lmbda * nxt
            lam[t] = nxt
        discount.copy_(torch.cumprod(cont * gamma, 0) / gamma)

    def moments_update(self, x: Tensor, state: Tensor, decay: float, max_: float, p_low: float, p_high: float,
                       out: Tensor):
        """x: flat values (already all-gathered); state[0:2] = (low, high) EMA buffers (updated in place);
        out[0:2] = (offset, invscale).  torch.quantile 'linear' interpolation."""
        v = x.flatten()
        lo = torch.quantile(v, p_low)
        hi = torch.quantile(v, p_high)
        state[0] = decay * state[0] + (1 - decay) * lo
        state[1] = decay * state[1] + (1 - decay) * hi
        out[0] = state[0]
        out[1] = torch.maximum(torch.tensor(1.0 / max_), state[1] - state[0])

    def actor_loss_grad(self, raw: Tensor, actions: Tensor, lam: Tensor, val: Tensor, discount: Tensor,
                        moments: Tensor, head_dims, unimix: float, ent_coef: float, scale: float,
                        rows: Tensor, draw: Tensor):
        """Discrete policy loss (dreamer_v3.py:272-297) for M = H*N rows.
        raw [M,sumA] raw head logits, actions [M,sumA] one-hot, lam/val/discount [M], moments=(offset,invscale).
        rows[m] = discount*(logp*adv + ent_coef*ent)  (policy_loss = -scale * sum rows with scale=1/M);
        draw = d(policy_loss)/d raw."""
        M = raw.shape[0]
        adv = (lam - moments[0]) / moments[1] - (val - moments[0]) / moments[1]
        obj = torch.zeros(M)
        ent_tot = torch.zeros(M)
        off = 0
        for ad in head_dims:
            x = raw[:, off:off + ad]
            s = torch.softmax(x, -1)
            if unimix > 0:
                pm = (1 - unimix) * s + unimix / ad
                pmc = pm.clamp(FP32_EPS, 1 - FP32_EPS)
                mix = torch.log(pmc)
            else:
                mix = x
            lg = mix - torch.logsumexp(mix, -1, keepdim=True)
            p = torch.exp(lg)
            a_idx = actions[:, off:off + ad].argmax(-1, keepdim=True)
            logp = lg.gather(-1, a_idx).squeeze(-1)
            ent = -(p * lg).sum(-1)
            obj = obj + logp * adv
            ent_tot = ent_tot + ent
            dlogp = F.one_hot(a_idx.squeeze(-1), ad).float() - p
            dent = -p * (lg + ent.unsqueeze(-1))
            g = (-(scale * discount)).unsqueeze(-1) * (adv.unsqueeze(-1) * dlogp + ent_coef * dent)
            if unimix > 0:
                inside = (pm >= FP32_EPS) & (pm <= 1 - FP32_EPS)
                ds = torch.where(inside, g * (1 - unimix) / pmc, torch.zeros_like(g))
                g = s * (ds - (s * ds).sum(-1, keepdim=True))
            draw[:, off:off + ad] = g
            off += ad
        rows.copy_(discount * (obj + ent_coef * ent_tot))

    # ---------------------------------------------------------------- reductions / optimiser
    def sum_rows(self, X: Tensor, out: Tensor, scale: float):
        """out[c] = scale * sum_m X[m,c]  (X [M,C] -> out [C]); used for metric means."""
        out.copy_(scale * X.reshape(X.shape[0], -1).sum(0))

    def weighted_mean(self, x: Tensor, w: Tensor, scale: float, out: Tensor):
        out.copy_(scale * (x.flatten() * w.flatten()).sum())

    def sumsq(self, x: Tensor, out: Tensor):
        """out (float64 scalar tensor) = sum x^2"""
        out.copy_((x.double() ** 2).sum())

    def adam_step(self, p: Tensor, g: Tensor, m: Tensor, v: Tensor, normsq: Tensor, max_norm: float, lr: float,
                  b1: float, b2: float, eps: float, step_t: Tensor, norm_out: Tensor):
        """clip_grad_norm_(max_norm) folded into torch.optim.Adam's update.  normsq: float64 scalar
        (sum g^2 over the whole group).  norm_out[0] = pre-clip L2 norm (fp32)."""
        step = int(step_t.item())
        total = torch.sqrt(normsq).float()
        norm_out.copy_(total)
        coef = torch.clamp(max_norm / (total + 1e-6), max=1.0) if max_norm > 0 else torch.tensor(1.0)
        gg = g * coef
        m.lerp_(gg, 1 - b1)
        v.mul_(b2).addcmul_(gg, gg, value=1 - b2)
        bc1 = 1 - b1 ** step
        bc2 = 1 - b2 ** step
        denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
        p.addcdiv_(m, denom, value=-lr / bc1)

    def ema(self, target: Tensor, src: Tensor, tau: float):
        target.mul_(1 - tau).add_(src, alpha=tau)

    def fill_exponential(self, out: Tensor, seed: int, stream_id: int, counter: Optional[Tensor] = None):
        c = int(counter.item()) if counter is not None else 0
        g = torch.Generator().manual_seed(seed * 1000003 + stream_id * 7919 + c)
        out.exponential_(1.0, generator=g)

    def increment(self, step_t: Tensor):
        step_t.add_(1)

    def affine(self, x: Tensor, out: Tensor, alpha: float, beta: float):
        out.copy_(alpha * x + beta)

    def zero(self, x: Tensor):
        x.zero_()

    def copy(self, src: Tensor, dst: Tensor):
        dst.copy_(src)

    def axpy(self, x: Tensor, y: Tensor, alpha: float = 1.0):
        y.add_(x, alpha=alpha)

    def symlog(self, x: Tensor, y: Tensor):
        y.copy_(_symlog(x))

    def tanh_fwd(self, x: Tensor, y: Tensor):
        y.copy_(torch.tanh(x))

    def tanh_bwd(self, y: Tensor, dy: Tensor, dx: Tensor, accumulate: bool = False):
        r = dy * (1 - y * y)
        dx.add_(r) if accumulate else dx.copy_(r)

    # ---- replay storage (csrc/replay.cu)
    def replay_gather(self, storage: Tensor, idx: Tensor, out: Tensor, n_samples: int, batch: int, seq_len: int):
        rows = storage[idx.long()].reshape(n_samples, batch, seq_len, *storage.shape[1:])
        out.view(n_samples, seq_len, batch, *storage.shape[1:]).copy_(rows.transpose(1, 2))

    def replay_scatter(self, src: Tensor, dst_rows: Tensor, storage: Tensor):
        storage[dst_rows.long()] = src

    # ---- SAC / PPO dense layers (csrc/mlp.cu)
    def bgemm(self, A: Tensor, B: Tensor, C: Tensor, bias=None, aux=None, rsum=None, epi: str = "none",
              accumulate: bool = False):
        v = torch.matmul(A, B)
        if bias is not None:
            v = v + bias.unsqueeze(1)
        if epi == "relu":
            v = torch.relu(v)
        elif epi == "tanh":
            v = torch.tanh(v)
        elif epi == "drelu":
            v = v * (aux > 0)
        elif epi == "dtanh":
            v = v * (1 - aux * aux)
        C.add_(v) if accumulate else C.copy_(v)
        if rsum is not None:
            r = A.sum(-1).expand(C.shape[0], -1)
            rsum.add_(r) if accumulate else rsum.copy_(r)

    # ---- SAC element-wise stages (csrc/sac.cu)
    def sac_sample_fwd(self, head, eps, scale, abias, action, logp, tanh_out=None):
        A = eps.shape[1]
        mean, ls = head[:, :A], head[:, A:].clamp(-5.0, 2.0)
        std = ls.exp()
        xt = mean + std * eps
        y = torch.tanh(xt)
        action.copy_(y * scale + abias)
        lp = -((xt - mean) ** 2) / (2 * std * std) - std.log() - math.log(math.sqrt(2 * math.pi))
        lp = lp - torch.log(scale * (1 - y * y) + 1e-6)
        logp.copy_(lp.sum(-1))
        if tanh_out is not None:
            tanh_out.copy_(y)

    def sac_sample_bwd(self, head, eps, tanh_y, scale, dact, log_alpha, dhead):
        B, A = eps.shape
        raw = head[:, A:]
        std = raw.clamp(-5.0, 2.0).exp()
        dlogp = log_alpha.exp() / B
        om = 1 - tanh_y * tanh_y
        dxt = dact.sum(0) * scale * om + dlogp * (2 * scale * tanh_y * om) / (scale * om + 1e-6)
        dstd = dxt * eps - dlogp / std
        dhead[:, :A] = dxt
        dhead[:, A:] = torch.where((raw >= -5.0) & (raw <= 2.0), dstd * std, torch.zeros_like(std))

    def sac_target(self, q_target, logp, rewards, terminated, log_alpha, gamma, y):
        y.copy_(rewards + (1 - terminated) * gamma * (q_target.min(0)[0] - log_alpha.exp() * logp))

    def sac_critic_loss(self, q, y, dq, loss_out):
        d = q - y.unsqueeze(0)
        loss_out.copy_((d * d).mean(1).sum().reshape(1))
        dq.copy_(2 * d / q.shape[1])

    def sac_actor_loss(self, q, logp, log_alpha, target_entropy, dq, actor_loss, alpha_loss, dlog_alpha):
        B = q.shape[1]
        m, arg = q.min(0)
        dq.zero_()
        dq.scatter_(0, arg.unsqueeze(0), -1.0 / B)
        actor_loss.copy_((log_alpha.exp() * logp - m).mean().reshape(1))
        s = (logp + target_entropy).mean()
        alpha_loss.copy_((-log_alpha * s).reshape(1))
        dlog_alpha.copy_((-s).reshape(1))

    def fill_normal(self, out: Tensor, seed: int, stream_id: int, counter: Optional[Tensor] = None):
        c = int(counter.item()) if counter is not None else 0
        g = torch.Generator().manual_seed(seed * 1000003 + stream_id * 7919 + c)
        out.normal_(generator=g)

    # ---- PPO (csrc/ppo.cu)
    def im2col(self, x: Tensor, col: Tensor, k: int, stride: int):
        B, H, W, C = x.shape
        p = x.unfold(1, k, stride).unfold(2, k, stride)          # [B, Ho, Wo, C, ky, kx]
        col.copy_(p.permute(0, 1, 2, 4, 5, 3).reshape(col.shape))

    def col2im(self, dcol: Tensor, act, dx: Tensor, k: int, stride: int):
        B, H, W, C = dx.shape
        Ho, Wo = (H - k) // stride + 1, (W - k) // stride + 1
        d = dcol.reshape(B, Ho * Wo, k, k, C).permute(0, 4, 2, 3, 1).reshape(B, C * k * k, Ho * Wo)
        out = F.fold(d, (H, W), kernel_size=k, stride=stride).permute(0, 2, 3, 1)
        dx.copy_(out * (act > 0) if act is not None else out)

    def ppo_loss(self, head, actions, old_logp, adv, values, old_values, returns, dhead, dvalues, losses, head_dims,
                 is_continuous, clip_vloss, normalize_adv, clip_coef, vf_coef, ent_coef):
        h = head.detach().clone().requires_grad_(True)
        v = values.detach().clone().requires_grad_(True)
        if is_continuous:
            mean, ls = h.chunk(2, -1)
            sd = ls.exp()
            corr = 0.0
            if int(is_continuous) == 2:          # tanh_normal: stored actions are squashed (ppo/agent.py:194-206)
                corr = 2.0 * (math.log(2.0) - actions - F.softplus(-2.0 * actions)).sum(-1)
                actions = torch.atanh(actions.clamp(-SAFE_LIM, SAFE_LIM))
            lp = (-((actions - mean) ** 2) / (2 * sd * sd) - ls - math.log(math.sqrt(2 * math.pi))).sum(-1) - corr
            ent = (0.5 + 0.5 * math.log(2 * math.pi) + ls).sum(-1)
        else:
            lp, ent, off = 0.0, 0.0, 0
            for n in head_dims:
                logp = torch.log_softmax(h[:, off:off + n], -1)
                lp = lp + (logp * actions[:, off:off + n]).sum(-1)
                ent = ent - (logp.exp() * logp).sum(-1)
                off += n
        a = adv
        if normalize_adv:
            a = (a - a.mean()) / (a.std() + 1e-8)
        ratio = (lp - old_logp).exp()
        pg = -torch.min(a * ratio, a * ratio.clamp(1 - clip_coef, 1 + clip_coef)).mean()
        if clip_vloss:
            vc = old_values + (v - old_values).clamp(-clip_coef, clip_coef)
            vl = 0.5 * torch.max((v - returns) ** 2, (vc - returns) ** 2).mean()
        else:
            vl = ((v - returns) ** 2).mean()
        el = (-ent).mean()
        gh, gv = torch.autograd.grad(pg + vf_coef * vl + ent_coef * el, [h, v], allow_unused=True)
        dhead.copy_(gh)
        dvalues.copy_(gv)
        losses.copy_(torch.stack([pg, vl, el]).detach())

    # ---- imagination: Linear([one-hot z, a]) as a gather-sum (csrc/rssm.cu)
    def transpose2d(self, X: Tensor, Y: Tensor):
        Y.copy_(X.t())

    def onehot_linear_supported(self, groups: int, classes: int, A: int, N: int) -> bool:
        return groups <= 64 and A <= 32

    def onehot_linear(self, z: Tensor, act: Tensor, WT: Tensor, out: Tensor, groups: int, classes: int):
        Z = groups * classes
        out.copy_(z @ WT[:Z] + act @ WT[Z:])

    # ---- fused imagination ops: exact compositions of the ops above (b200rl_gemm_ln, b200rl_onehot_linear_ln,
    # b200rl_head_sample); having them here lets the CPU engine tests walk the same fused schedule as the GPU
    def gemm_ln_supported(self, A: Tensor, W: Tensor, mode: int = 0) -> bool:
        N = W.shape[0]
        return A.shape[0] >= 32 and N % 4 == 0 and N <= 1536 and (mode == 0 or N % 384 == 0)

    def gemm_ln_act(self, A: Tensor, W: Tensor, gamma: Tensor, beta: Tensor, eps: float, act: int, out: Tensor,
                    pre: Optional[Tensor] = None):
        tmp = torch.empty(A.shape[0], W.shape[0])
        self.gemm(A, W, tmp, False, True)
        if pre is not None:
            pre.copy_(tmp)
        self.ln_act_fwd(tmp, gamma, beta, eps, act, out)

    def gemm_ln_gru(self, A: Tensor, W: Tensor, gamma: Tensor, beta: Tensor, eps: float, h_prev: Tensor, h_out: Tensor,
                    h_out2: Optional[Tensor] = None, g_pre: Optional[Tensor] = None, g_ln: Optional[Tensor] = None):
        """h_out2 may alias the left half of A (the next step's [h | x] buffer): everything is computed before it is written."""
        tmp = torch.empty(A.shape[0], W.shape[0])
        self.gemm(A, W, tmp, False, True)
        ln = torch.empty_like(tmp)
        self.ln_act_fwd(tmp, gamma, beta, eps, ACT_NONE, ln)
        h = torch.empty(A.shape[0], W.shape[0] // 3)
        self.gru_gate_fwd(ln, h_prev, h)
        if g_pre is not None:
            g_pre.copy_(tmp)
        if g_ln is not None:
            g_ln.copy_(ln)
        h_out.copy_(h)
        if h_out2 is not None:
            h_out2.copy_(h)

    def onehot_linear_ln_supported(self, WT: Tensor, out: Tensor, pre: Optional[Tensor] = None) -> bool:
        return 128 <= WT.shape[1] <= 1024 and WT.shape[1] % 128 == 0

    def onehot_linear_ln(self, z: Tensor, act: Tensor, WT: Tensor, gamma: Tensor, beta: Tensor, eps: float, out: Tensor,
                         groups: int, classes: int, pre: Optional[Tensor] = None):
        tmp = torch.empty(z.shape[0], WT.shape[1])
        self.onehot_linear(z, act, WT, tmp, groups, classes)
        if pre is not None:
            pre.copy_(tmp)
        self.ln_act_fwd(tmp, gamma, beta, eps, ACT_SILU, out)

    def head_sample_supported(self, X: Tensor, W: Tensor) -> bool:
        return W.shape[0] <= 32 and X.shape[1] <= 1024 and X.shape[1] % 4 == 0

    def head_sample(self, X: Tensor, W: Tensor, bias: Optional[Tensor], noise: Optional[Tensor], unimix: float, raw: Tensor,
                    onehot: Tensor):
        tmp = torch.empty(X.shape[0], W.shape[0])
        self.gemm(X, W, tmp, False, True, bias=bias)
        raw.copy_(tmp)
        self.cat_sample(tmp, noise, unimix, 1, W.shape[0], onehot)

    # ---- Dreamer-V3 continuous actions (csrc/dv3_cont.cu)
    def cont_action_fwd(self, head, eps, action, ent, min_std, max_std, init_std, clip):
        A = eps.shape[1]
        std = (max_std - min_std) * torch.sigmoid(head[:, A:] + init_std) + min_std
        a = torch.tanh(head[:, :A]) + std * eps
        if clip > 0:
            a = a * (clip / torch.clamp(a.abs(), min=clip))
        action.copy_(a)
        if ent is not None:
            ent.copy_((0.5 + 0.5 * math.log(2 * math.pi) + std.log()).sum(-1))

    def cont_action_bwd(self, head, eps, d_action, discount, dhead, min_std, max_std, init_std, clip, ent_scale):
        M, A = eps.shape
        sg = torch.sigmoid(head[:, A:] + init_std)
        std = (max_std - min_std) * sg + min_std
        th = torch.tanh(head[:, :A])
        a_raw = th + std * eps
        f = clip / torch.clamp(a_raw.abs(), min=clip) if clip > 0 else torch.ones_like(a_raw)
        da = d_action * f
        dstd = da * eps + (ent_scale * discount.reshape(-1)[:M]).unsqueeze(-1) / std
        dhead[:, :A] = da * (1 - th * th)
        dhead[:, A:] = dstd * (max_std - min_std) * sg * (1 - sg)

    def lambda_returns_bwd(self, cont_logit, discount, moments, lam, val, ent, gamma, lmbda, ent_coef, scale, d_val,
                           d_rew, rows):
        H, N = lam.shape
        inv = 1.0 / moments[1]
        c = (torch.sigmoid(cont_logit.reshape(H + 1, N)) > 0.5).float() * gamma
        D, v, e = discount.reshape(H + 1, N), val.reshape(H + 1, N), ent.reshape(-1)[: H * N].reshape(H, N)
        rows.reshape(H, N).copy_(D[:H] * ((lam - v[:H]) * inv + ent_coef * e))
        dv, dr = d_val.reshape(H + 1, N), d_rew.reshape(H + 1, N)
        dv.zero_(), dr.zero_()
        G = torch.zeros(N)
        for t in range(H):
            G = -scale * D[t] * inv + (c[t] * lmbda * G if t > 0 else 0.0)
            dr[t + 1] = G
            dv[t] += scale * D[t] * inv
            dv[t + 1] += G * c[t + 1] * (1 - lmbda)
        dv[H] += c[H] * lmbda * G

    def twohot_mean_bwd(self, logits, d_mean, low, high, d_logits):
        nb = logits.shape[-1]
        bins = torch.linspace(low, high, nb)
        p = torch.softmax(logits, -1)
        m = (p * bins).sum(-1, keepdim=True)
        d_logits.copy_(d_mean.reshape(-1, 1) * torch.exp(m.abs()) * p * (bins - m))

    def ppo_act(self, head, noise, actions, logp, head_dims, is_continuous, greedy):
        if is_continuous:
            A = sum(head_dims)
            mean, ls = head[:, :A], head[:, A:]
            a = mean if (greedy or noise is None) else mean + ls.exp() * noise
            lp = (-((a - mean) ** 2) / (2 * (ls.exp() ** 2)) - ls - math.log(math.sqrt(2 * math.pi))).sum(-1)
            if int(is_continuous) == 2:          # PPOPlayer.forward with tanh_normal (ppo/agent.py:257-268)
                a = torch.tanh(a).clamp(-SAFE_LIM, SAFE_LIM)
                lp = lp - 2.0 * (math.log(2.0) - a - F.softplus(-2.0 * a)).sum(-1)
            elif int(is_continuous) == 3:        # PPOPlayer.get_actions with tanh_normal (ppo/agent.py:306-311)
                a = torch.atanh(a.clamp(-SAFE_LIM, SAFE_LIM))
            actions.copy_(a)
            logp.copy_(lp)
            return
        off, lp = 0, 0.0
        for n in head_dims:
            lg = torch.log_softmax(head[:, off:off + n], -1)
            p = lg.exp()
            if not greedy and noise is not None:
                p = p / noise[:, off:off + n]
            idx = p.argmax(-1)
            actions[:, off:off + n] = F.one_hot(idx, n).float()
            lp = lp + lg.gather(-1, idx.unsqueeze(-1)).squeeze(-1)
            off += n
        logp.copy_(lp)
