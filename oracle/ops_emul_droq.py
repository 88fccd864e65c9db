"""TEST INFRASTRUCTURE — executable specification (plain fp32 torch, CPU) of the DroQ C-ABI ops in `include/b200rl.h`
(`b200rl_droq_actor_loss`, `b200rl_dropout_mask`, `b200rl_dropout_ln_relu_fwd` / `_bwd`), on top of the
`oracle/ops_emul.py::EmulOps` specification of every other op.  Same two uses: `-m gpu` tests compare each CUDA kernel
against the method of the same name, and `-m "not gpu"` tests inject this object into `DroQEngine` (test double) to walk
the engine's schedule on a GPU-less host.  The product never constructs it.
"""
from __future__ import annotations

import torch

from oracle.ops_emul import EmulOps


def mask_words(H: int) -> int:
    return (H + 31) // 32


def pack_masks(keep: torch.Tensor) -> torch.Tensor:
    """bool keep masks [..., H] -> int32 words [..., ceil(H/32)], bit j of word k = column 32k + j (padding bits 0)"""
    H = keep.shape[-1]
    W = mask_words(H)
    bits = torch.zeros(*keep.shape[:-1], W * 32, dtype=torch.int64, device=keep.device)
    bits[..., :H] = keep.to(torch.int64)
    words = (bits.view(*keep.shape[:-1], W, 32) << torch.arange(32, device=keep.device)).sum(-1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def unpack_masks(words: torch.Tensor, H: int) -> torch.Tensor:
    """int32 words [..., W] -> bool keep masks [..., H] (padding bits ignored)"""
    w = words.to(torch.int64) & 0xFFFFFFFF
    bits = (w.unsqueeze(-1) >> torch.arange(32, device=words.device)) & 1
    return bits.reshape(*words.shape[:-1], words.shape[-1] * 32)[..., :H].bool()


def dropout_scale(p: float) -> torch.Tensor:
    """torch's dropout multiplies by mask / (1-p) computed in fp32"""
    return torch.tensor(1.0, dtype=torch.float32) / (1.0 - p)


class DroQEmulOps(EmulOps):
    name = "emul_droq"

    def droq_actor_loss(self, q, logp, log_alpha, target_entropy, dq, actor_loss, alpha_loss, dlog_alpha):
        nets, B = q.shape
        dq.fill_(-1.0 / (nets * B))
        actor_loss.copy_((log_alpha.exp() * logp - q.mean(0)).mean().reshape(1))
        s = (logp + target_entropy).mean()
        alpha_loss.copy_((-log_alpha * s).reshape(1))
        dlog_alpha.copy_((-s).reshape(1))

    def dropout_mask(self, mask, p: float, seed: int, stream_id: int, counter=None):
        """the bits are Bernoulli(1-p); the stream differs from the CUDA kernel's (tests inject masks where they matter)"""
        c = int(counter.item()) if counter is not None else 0
        g = torch.Generator().manual_seed(seed * 1000003 + stream_id * 7919 + c)
        keep = torch.rand(*mask.shape, 32, generator=g) >= p
        mask.copy_(pack_masks(keep.reshape(*mask.shape[:-1], mask.shape[-1] * 32)))

    def dropout_ln_relu_supported(self, H: int) -> bool:
        return 1 <= H <= 1024

    @staticmethod
    def _dropped(z, mask, p):
        if mask is None:
            return z
        return z * unpack_masks(mask, z.shape[-1]).to(z.dtype) * dropout_scale(p).to(z.dtype)

    def dropout_ln_relu_fwd(self, z, mask, p: float, gamma, beta, eps: float, y, stats):
        x = self._dropped(z, mask, p)
        mean = x.mean(-1, keepdim=True)
        rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + eps)
        y.copy_(torch.relu((x - mean) * rstd * gamma.unsqueeze(1) + beta.unsqueeze(1)))
        stats.copy_(torch.cat([mean, rstd], -1))

    def dropout_ln_relu_bwd(self, dy, y, z, mask, p: float, stats, gamma, dz, dgamma=None, dbeta=None):
        """gradient of relu(LN(dropout(z))) w.r.t. z (and gamma, beta), from the forward's row statistics"""
        mean, rstd = stats[..., :1], stats[..., 1:]
        xhat = (self._dropped(z, mask, p) - mean) * rstd
        g = dy * (y > 0).to(dy.dtype)
        dxh = g * gamma.unsqueeze(1)
        dx = rstd * (dxh - dxh.mean(-1, keepdim=True) - xhat * (dxh * xhat).mean(-1, keepdim=True))
        dz.copy_(self._dropped(dx, mask, p))
        if dgamma is not None:
            dgamma.copy_((g * xhat).sum(1))
            dbeta.copy_(g.sum(1))
