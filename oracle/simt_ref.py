"""Float64 references of the CUDA-core (FFMA) product family that oracle/tc_ref.py does not already cover: the batched
MLP product of csrc/mlp.cu with its epilogues and row sums, and the LSTM recurrence of csrc/lstm.cu, forward one step at
a time (teacher-forced) and backward through time with a propagated first-order error bound.

Like tc_ref, every function takes fp32 (or fp64) tensors on any device and computes in float64 on that device.  GEMM
and convolutions are tc_ref.gemm64 / conv_down64 / conv_up64 / conv_wgrad64.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

U = 2.0 ** -24          # unit roundoff of fp32


def tau1(K: int) -> float:
    """Error bound of one fp32 FFMA reduction of length K, relative to sum |a||b|: 2^-24 (16 + 2 sqrt(K)).  A sequential
    chain of round-to-nearest FMAs reaches ~1.0 sqrt(K) u on positive operands and a few u on mixed signs; split-K,
    tiles and paired FMAs only shorten the chain."""
    return U * (16.0 + 2.0 * K ** 0.5)


def _d(t: Optional[Tensor]) -> Optional[Tensor]:
    return None if t is None else t.double()          # keeps the autograd graph: the CPU test differentiates lstm_step64


def bgemm64(A: Tensor, B: Tensor, bias: Optional[Tensor] = None, aux: Optional[Tensor] = None, epi: str = "none",
            C0: Optional[Tensor] = None):
    """C[n] = C0[n] + epi(A[n] B[n] + bias[n]) for the 3-D views `CudaOps.bgemm` takes (A [n|1, M, K], B [n|1, K, N],
    bias [n|1, N], aux / C0 [n, M, N]; a leading dim of 1 broadcasts).  epi: none / relu / tanh, or drelu / dtanh,
    which multiply by ReLU'(aux) = (aux > 0) / Tanh'(aux) = 1 - aux^2.

    Returns (C, magnitude, rsum): magnitude = sum_k |a||b| + |bias| + |C0| (before the epilogue), rsum = sum_k A[n, m, k]
    broadcast to [n, M]."""
    a, b = _d(A), _d(B)
    pre, mag = torch.matmul(a, b), torch.matmul(a.abs(), b.abs())
    if bias is not None:
        pre, mag = pre + _d(bias).unsqueeze(1), mag + _d(bias).abs().unsqueeze(1)
    if epi == "relu":
        v = pre.clamp_min(0.0)
    elif epi == "tanh":
        v = torch.tanh(pre)
    elif epi == "drelu":
        v = pre * (_d(aux) > 0)
    elif epi == "dtanh":
        v = pre * (1.0 - _d(aux) ** 2)
    else:
        assert epi == "none", epi
        v = pre
    if C0 is not None:
        v, mag = v + _d(C0), mag + _d(C0).abs()
    nets = max(A.shape[0], B.shape[0])
    rsum = a.sum(-1).expand(nets, -1)
    return v, mag, rsum


def _gate_acts(z: Tensor) -> Tensor:
    H = z.shape[-1] // 4
    i, f, g, o = torch.split(z, H, -1)
    return torch.cat((torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)), -1)


def lstm_step64(xw_t: Tensor, W: Tensor, h_prev: Tensor, c_prev: Tensor):
    """One LSTM step (torch gate order i, f, g, o) on rows [..., 4H] / [..., H]: z = xw_t + h_prev W^T.

    Returns (gates, c, h, mag) in float64: the activated gates [..., 4H], the new cell and hidden state [..., H], and
    mag = |xw_t| + |h_prev| |W|^T, the scale of the pre-activation's rounding error."""
    xw, w, hp, cp = _d(xw_t), _d(W), _d(h_prev), _d(c_prev)
    z = xw + hp @ w.t()
    mag = xw.abs() + hp.abs() @ w.abs().t()
    gates = _gate_acts(z)
    H = hp.shape[-1]
    i, f, g, o = torch.split(gates, H, -1)
    c = f * cp + i * g
    h = o * torch.tanh(c)
    return gates, c, h, mag


def _carry_dc(dc: Tensor, f: Tensor) -> Tensor:
    """the cell-state gradient handed to step t-1"""
    return dc * f


def lstm_bwd64(d_out: Tensor, W: Tensor, gates: Tensor, cs: Tensor, c0: Tensor, lengths: Tensor):
    """Backward through time of the LSTM forward that saved `gates` [T, B, 4H] (activated) and `cs` [T, B, H], in
    float64 on those saved values (so only the backward's own arithmetic is referenced).  Padded steps (t >= lengths[b])
    get zero gradients and carry nothing.

    Returns (d_gates, bound), both [T, B, 4H]: d_gates w.r.t. the pre-activation gates, and a first-order bound on the
    error of an fp32 implementation that forms each step like csrc/lstm.cu: the carried state gradients are propagated
    through the same recurrence,
        E_dh(t-1) = |W|^T E_dg(t) + tau1(4H) sum_j |dg_j| |W_jk|
        E_dc(t-1) = |f| E_dc(t) + u |dc f|
    and E_dg(t) follows from E_dh(t), E_dc(t) through each gate's coefficient, plus the rounding of that coefficient
    (tanhf and expf within 2 ulp = 4u relative, every other operation u)."""
    do, w, gt, ct, c00 = _d(d_out), _d(W), _d(gates), _d(cs), _d(c0)
    T, B, G = gt.shape
    H = G // 4
    valid = torch.arange(T, device=gt.device).unsqueeze(1) < lengths.to(gt.device).long().reshape(1, -1)
    dgates, bound = torch.zeros_like(gt), torch.zeros_like(gt)
    dh_c, dc_c = torch.zeros(B, H, dtype=gt.dtype, device=gt.device), torch.zeros(B, H, dtype=gt.dtype, device=gt.device)
    e_dh_c, e_dc_c = torch.zeros_like(dh_c), torch.zeros_like(dc_c)
    wa, t4 = w.abs(), tau1(4 * H)
    u = U
    for t in reversed(range(T)):
        v = valid[t].unsqueeze(-1)
        i, f, g, o = torch.split(gt[t], H, -1)
        c = ct[t]
        cp = ct[t - 1] if t > 0 else c00
        tc = torch.tanh(c)
        s = o * (1 - tc * tc)
        dh = do[t] + dh_c
        dc = dc_c + dh * s
        a_i, a_f, a_g, a_o = g * i * (1 - i), cp * f * (1 - f), i * (1 - g * g), tc * o * (1 - o)
        dg = torch.cat((dc * a_i, dc * a_f, dc * a_g, dh * a_o), -1)
        dg = torch.where(v, dg, torch.zeros_like(dg))
        # error bounds of this step
        e_dh = e_dh_c + u * dh.abs()
        e_s = 12 * u * o.abs()                                   # o (1 - tanhf(c)^2): tanhf 4u, square, subtract, multiply
        e_dc = e_dc_c + s.abs() * e_dh + dh.abs() * e_s + 2 * u * (dc_c.abs() + (dh * s).abs())
        # (1 - x) and (1 - x^2) of a gate in [0, 1] / [-1, 1] cost at most 2u absolute; three products 3u relative
        e_i = a_i.abs() * e_dc + dc.abs() * (2 * u * (g * i).abs() + 3 * u * a_i.abs())
        e_f = a_f.abs() * e_dc + dc.abs() * (2 * u * (cp * f).abs() + 3 * u * a_f.abs())
        e_g = a_g.abs() * e_dc + dc.abs() * (2 * u * i.abs() + 3 * u * a_g.abs())
        e_o = a_o.abs() * e_dh + dh.abs() * (2 * u * (tc * o).abs() + 4 * u * (o * (1 - o)).abs() * tc.abs()
                                             + 3 * u * a_o.abs())
        e_dg = torch.where(v, torch.cat((e_i, e_f, e_g, e_o), -1), torch.zeros_like(dg))
        dgates[t], bound[t] = dg, e_dg
        # carried to step t - 1
        dc_c = torch.where(v, _carry_dc(dc, f), torch.zeros_like(dc))
        e_dc_c = torch.where(v, f.abs() * e_dc + u * (dc * f).abs(), torch.zeros_like(dc))
        dh_c = dg @ w
        e_dh_c = e_dg @ wa + t4 * (dg.abs() @ wa)
    return dgates, bound
