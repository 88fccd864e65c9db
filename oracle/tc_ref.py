"""Float64 reference of the tensor-core product family (csrc/gemm_tc.cu, csrc/conv.cu): GEMM in all four layouts,
the stride-2 k4 p1 convolutions and their weight gradient, and the fused product + LayerNorm (+ SiLU) / + GRU gate.

Every function takes fp32 (or fp64) tensors on any device, computes in float64 on that device, and returns the result
together with the elementwise magnitude  sum_k |a_k| |b_k|  (+ |bias|, + |C0|): the scale a per-element rounding-error
bound is stated against.  Layouts are the library's: NHWC images, conv weights [Cs, Cb, 4, 4] (Conv2d: big Cb -> small
Cs; ConvTranspose2d: small Cs -> big Cb), GEMM operands as passed to `CudaOps.gemm` (A [M, K] or [K, M] if transA,
B [K, N] or [N, K] if transB).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import Tensor


def _d(t: Optional[Tensor]) -> Optional[Tensor]:
    return None if t is None else t.detach().double()


def gemm64(A: Tensor, B: Tensor, transA: bool, transB: bool, bias: Optional[Tensor] = None,
           C0: Optional[Tensor] = None):
    """C = op(A) op(B) (+ bias[N]) (+ C0); returns (C, magnitude)."""
    a, b = _d(A), _d(B)
    a = a.t() if transA else a
    b = b.t() if transB else b
    c, mag = a @ b, a.abs() @ b.abs()
    if bias is not None:
        c, mag = c + _d(bias), mag + _d(bias).abs()
    if C0 is not None:
        c, mag = c + _d(C0), mag + _d(C0).abs()
    return c, mag


def _nchw(x: Tensor) -> Tensor:
    return x.permute(0, 3, 1, 2)


def _nhwc(x: Tensor) -> Tensor:
    return x.permute(0, 2, 3, 1).contiguous()


def conv_down64(big: Tensor, W: Tensor, bias: Optional[Tensor] = None):
    """Conv2d(k4, s2, p1): big [NB, 2h, 2w, Cb] -> small [NB, h, w, Cs] (+ bias[Cs]); returns (small, magnitude)."""
    x, w, b = _nchw(_d(big)), _d(W), _d(bias)
    out = F.conv2d(x, w, b, stride=2, padding=1)
    mag = F.conv2d(x.abs(), w.abs(), None if b is None else b.abs(), stride=2, padding=1)
    return _nhwc(out), _nhwc(mag)


def conv_up64(small: Tensor, W: Tensor, bias: Optional[Tensor] = None):
    """ConvTranspose2d(k4, s2, p1): small [NB, h, w, Cs] -> big [NB, 2h, 2w, Cb] (+ bias[Cb]); returns (big, magnitude)."""
    x, w, b = _nchw(_d(small)), _d(W), _d(bias)
    out = F.conv_transpose2d(x, w, b, stride=2, padding=1)
    mag = F.conv_transpose2d(x.abs(), w.abs(), None if b is None else b.abs(), stride=2, padding=1)
    return _nhwc(out), _nhwc(mag)


def conv_wgrad64(small: Tensor, big: Tensor, dW0: Optional[Tensor] = None):
    """Weight gradient of conv_down: dW[cs, cb, ky, kx] = sum_{n,y,x} small[n,y,x,cs] big[n,2y-1+ky,2x-1+kx,cb]
    (+ dW0, the accumulate form); returns (dW, magnitude)."""
    s, x = _nchw(_d(small)), _nchw(_d(big))
    shape = (s.shape[1], x.shape[1], 4, 4)
    dw = torch.nn.grad.conv2d_weight(x, shape, s, stride=2, padding=1)
    mag = torch.nn.grad.conv2d_weight(x.abs(), shape, s.abs(), stride=2, padding=1)
    if dW0 is not None:
        dw, mag = dw + _d(dW0), mag + _d(dW0).abs()
    return dw, mag


def _layer_norm(x: Tensor, gamma: Tensor, beta: Tensor, eps: float) -> Tensor:
    return F.layer_norm(x, (x.shape[-1],), _d(gamma), _d(beta), eps)


def gemm_ln64(A: Tensor, W: Tensor, gamma: Tensor, beta: Tensor, eps: float, act: int):
    """Fused product + LayerNorm, mode 0: out = act(LN(A W^T)), act 0 = identity, 1 = SiLU.
    Returns (out, magnitude of the product, pre = A W^T)."""
    pre, mag = gemm64(A, W, False, True)
    out = _layer_norm(pre, gamma, beta, eps)
    if act == 1:
        out = F.silu(out)
    return out, mag, pre


def gru_gate64(ln: Tensor, h_prev: Tensor) -> Tensor:
    """LayerNormGRUCell gate on the normalised (reset | cand | update) thirds."""
    r, c, u = torch.chunk(ln, 3, -1)
    r = torch.sigmoid(r)
    c = torch.tanh(r * c)
    u = torch.sigmoid(u - 1.0)
    return u * c + (1.0 - u) * _d(h_prev)


def gemm_ln_gru64(A: Tensor, W: Tensor, gamma: Tensor, beta: Tensor, eps: float, h_prev: Tensor):
    """Fused product + LayerNorm + GRU gate, mode 1.  Returns (h, magnitude of the product, pre = A W^T, ln = LN(pre))."""
    pre, mag = gemm64(A, W, False, True)
    ln = _layer_norm(pre, gamma, beta, eps)
    return gru_gate64(ln, h_prev), mag, pre, ln
