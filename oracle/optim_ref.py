"""Float64 reference of the optimiser family (csrc/optim.cu: clip + Adam with optional L2 decay, clip + RMSprop, the
target-critic EMA, the sum of squares behind the clip) and first-order bounds on the error of an fp32 implementation
that evaluates the same expressions.

Like ln_ref / loss_ref, every function takes fp32 (or fp64) tensors on any device and computes in float64 on that
device.  The scalar hyperparameters are the values the kernels receive: the C-ABI passes lr, betas, alpha, eps,
momentum, weight decay, max_norm and tau as `float`, so a caller hands this module those values rounded to fp32
(`f32`).  torch.optim keeps them in double; that gap (1 - 0.999f is 1.3e-5 off 0.001) is a property of the ABI, checked
separately, never folded into a bound here.

Bounds are per element, first order in u = 2^-24, evaluated on the float64 magnitudes: one u per rounding of each
operation on the magnitude it rounds, the clip coefficient's own rounding carried into every element, and an absolute
term for products that land among the fp32 subnormals (the library is built without --use_fast_math, so they are
kept, each rounding off by at most half the smallest subnormal).  A NaN or inf input makes the bound NaN / inf in the
elements it reaches; callers compare the finite elements and check the non-finite ones separately.
"""
from __future__ import annotations

import math
import numpy as np
import torch
from torch import Tensor

from oracle.simt_ref import U

TINY = 2.0 ** -149        # smallest fp32 subnormal: bounds one rounding that underflows (half of it, kept whole here)
F64 = torch.float64
COEF_ERR = 4 * U          # relative error of the fp32 clip coefficient: sqrt rounded to fp32, + 1e-6f, the division


def f32(x: float) -> float:
    """x as the kernels receive it (a C `float`)"""
    return float(np.float32(x))


def _d(t) -> Tensor:
    return t.detach().to(F64) if torch.is_tensor(t) else torch.tensor(t, dtype=F64)


def sumsq64(x: Tensor) -> float:
    """sum of x^2, exactly: the squares of fp32 values are exact in double and math.fsum adds them without rounding"""
    a = x.detach().cpu().double().numpy().ravel()
    return math.fsum(a * a)


def clip_coef64(normsq, max_norm: float) -> tuple[Tensor, Tensor]:
    """(coef, total) of torch.nn.utils.clip_grad_norm_: total = sqrt(normsq), coef = clamp(max_norm / (total + 1e-6),
    max=1), so a NaN total gives a NaN coefficient (torch.clamp propagates NaN) and an inf total gives 0.  max_norm <= 0
    is no clipping (the engines skip clip_gradients then): coef = 1, NaN or not."""
    total = _d(normsq).sqrt()
    if max_norm <= 0:
        return torch.ones((), dtype=F64, device=total.device), total
    return torch.clamp(max_norm / (total + 1e-6), max=1.0), total


def _sqrt_err(a: Tensor, e_a: Tensor) -> Tensor:
    """error of sqrtf(a~) where |a~ - a| <= e_a: propagated (|sqrt(a+e) - sqrt(a)| <= min(e / 2 sqrt(a), sqrt(e)))
    plus the rounding of the root"""
    a = a.clamp_min(0.0)
    r = a.sqrt()
    return torch.minimum(e_a / (2 * r), e_a.sqrt()) + U * r


def _clipped_grad(p: Tensor, g: Tensor, coef: Tensor, weight_decay: float):
    """grad = g * coef (+ weight_decay * p) and its error bound"""
    gc = g * coef
    e = (1 + COEF_ERR / U) * U * gc.abs()                 # the product's rounding and the coefficient's
    if weight_decay != 0:
        wp = weight_decay * p
        gc = gc + wp
        e = e + U * wp.abs() + U * gc.abs()
    return gc, e


def adam_step64(p, g, m, v, normsq, step: int, max_norm: float, lr: float, b1: float, b2: float, eps: float,
                weight_decay: float = 0.0) -> dict:
    """clip_grad_norm_(max_norm) then torch.optim.Adam's single-tensor step (torch/optim/adam.py, foreach=False) at step
    count `step`: grad = g coef (+ weight_decay p); m.lerp_(grad, 1 - b1); v.mul_(b2).addcmul_(grad, grad, 1 - b2);
    p.addcdiv_(m, sqrt(v) / sqrt(1 - b2^t) + eps, value=-lr / (1 - b1^t)).  Returns p, m, v, coef, total and the bounds
    err_p, err_m, err_v."""
    p, g, m, v = _d(p), _d(g), _d(m), _d(v)
    coef, total = clip_coef64(normsq, max_norm)
    coef, total = coef.to(p.device), total.to(p.device)
    gr, e_g = _clipped_grad(p, g, coef, weight_decay)
    omb1, omb2 = 1.0 - b1, 1.0 - b2                       # exact in fp32 for betas in [0.5, 1] (Sterbenz)
    d = gr - m
    m1 = m + omb1 * d
    e_m = omb1 * (e_g + U * d.abs()) + U * (omb1 * d).abs() + U * m1.abs() + TINY
    gg = omb2 * gr * gr
    v1 = v * b2 + gg
    e_v = 2 * omb2 * gr.abs() * e_g + 2 * U * gg + U * (v * b2).abs() + U * v1.abs() + 4 * TINY
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    step_size, bc2_sqrt = lr / bc1, math.sqrt(bc2)
    s = v1.sqrt() / bc2_sqrt
    den = s + eps
    q = m1 / den
    p1 = p - step_size * q
    e_s = _sqrt_err(v1, e_v) / bc2_sqrt + 2 * U * s       # the root, fp32 sqrt(bc2) and the division
    e_den = e_s + U * den
    e_q = e_m / den + q.abs() * e_den / den + U * q.abs()
    e_p = step_size * e_q + 2 * U * (step_size * q).abs() + U * p1.abs() + TINY   # fp32 step size, product, difference
    return dict(p=p1, m=m1, v=v1, coef=coef, total=total, err_p=e_p, err_m=e_m, err_v=e_v)


def rmsprop_step64(p, g, square_avg, normsq, max_norm: float, lr: float, alpha: float, eps: float,
                   weight_decay: float = 0.0, momentum: float = 0.0, momentum_buf=None, grad_avg=None) -> dict:
    """clip_grad_norm_(max_norm) then torch.optim.RMSprop's single-tensor step (torch/optim/rmsprop.py, foreach=False):
    grad (+ weight_decay p); sq.mul_(alpha).addcmul_(grad, grad, 1 - alpha); centered (grad_avg given):
    grad_avg.lerp_(grad, 1 - alpha), avg = sqrt(sq - grad_avg^2) + eps, else avg = sqrt(sq) + eps; momentum > 0:
    buf = buf momentum + grad / avg, p -= lr buf; else p -= lr grad / avg.  A negative centered variance gives NaN, as in
    torch.  Returns p, sq, buf, gavg (None where unused), coef, total and the bounds err_*."""
    p, g, sq = _d(p), _d(g), _d(square_avg)
    coef, total = clip_coef64(normsq, max_norm)
    coef, total = coef.to(p.device), total.to(p.device)
    gr, e_g = _clipped_grad(p, g, coef, weight_decay)
    oma = 1.0 - alpha
    gg = oma * gr * gr
    sq1 = sq * alpha + gg
    e_sq = 2 * oma * gr.abs() * e_g + 2 * U * gg + U * (sq * alpha).abs() + U * sq1.abs() + 4 * TINY
    out = dict(coef=coef, total=total, sq=sq1, err_sq=e_sq, buf=None, err_buf=None, gavg=None, err_gavg=None)
    if grad_avg is not None:
        ga = _d(grad_avg)
        d = gr - ga
        ga1 = ga + oma * d
        e_ga = oma * (e_g + U * d.abs()) + U * (oma * d).abs() + U * ga1.abs() + TINY
        var = sq1 - ga1 * ga1
        e_var = e_sq + 2 * ga1.abs() * e_ga + U * ga1 * ga1 + U * var.abs() + TINY
        root = var.sqrt()                                 # NaN where the variance is negative, as in torch
        e_root = _sqrt_err(var, e_var)
        out.update(gavg=ga1, err_gavg=e_ga, var=var, err_var=e_var)
    else:
        root = sq1.sqrt()
        e_root = _sqrt_err(sq1, e_sq)
    avg = root + eps
    e_avg = e_root + U * avg
    q = gr / avg
    e_q = e_g / avg + q.abs() * e_avg / avg + U * q.abs()
    if momentum > 0:
        buf = _d(momentum_buf)
        b1 = buf * momentum + q
        e_b = e_q + U * (buf * momentum).abs() + U * b1.abs() + TINY
        p1 = p - lr * b1
        e_p = lr * e_b + U * (lr * b1).abs() + U * p1.abs() + TINY
        out.update(buf=b1, err_buf=e_b)
    else:
        p1 = p - lr * q
        e_p = lr * e_q + U * (lr * q).abs() + U * p1.abs() + TINY
    out.update(p=p1, err_p=e_p)
    return out


def ema64(target, src, tau: float) -> tuple[Tensor, Tensor]:
    """tau src + (1 - tau) target (dreamer_v3.py:680) and the bound of target (1 - tau) + tau src in fp32: 1 - tau
    rounded, two products, one sum"""
    t, s = _d(target), _d(src)
    a, b = t * (1.0 - tau), tau * s
    r = a + b
    return r, 3 * U * (a.abs() + b.abs()) + U * r.abs() + TINY
