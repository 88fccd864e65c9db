"""TEST INFRASTRUCTURE — writes tests/golden/dv3_rssm_ref.pt by running the REAL REFERENCE's RSSM pieces in float64 with
autograd, on a few hundred small rows:

    python -m oracle.make_golden_rssm_ref

RSSM._uniform_mix and Actor._uniform_mix with OneHotCategoricalStraightThrough (its mode, its probabilities and the
gradient of rsample for given dz and dmix), and LayerNormGRUCell with layer_norm_cls = nn.Identity, bias = False and the
linear weight [0 | I_3R]: the cell's input is cat(hx, input), so its pre-activation is exactly G and the reference's own
forward computes the gate of gru_gate_fwd / _bwd.  The inputs stay clear of argmax near-ties and of the unimix clamp,
where the float64 reference and an fp32 kernel may differ by design.  tests/test_rssm_ref_cpu.py compares
oracle/rssm_ref.py with the fixture.
"""
from __future__ import annotations

import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import ref_harness  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "dv3_rssm_ref.pt")

# (owner, groups, classes, unimix): the RSSM's latent groups and the actor's heads
CAT_CASES = (("rssm", 4, 5, 0.01), ("rssm", 2, 33, 0.01), ("rssm", 3, 7, 0.0), ("actor", 1, 6, 0.01),
             ("actor", 1, 4, 0.5), ("actor", 1, 9, 0.0))


def f32(v):
    """scalar parameters are the fp32 values the kernels receive, so they are fp32-exact here"""
    return float(torch.tensor(v, dtype=torch.float32))


def clear_rows(logits, G, K, unimix, margin=1e-3):
    """rows whose every group has a relative gap of at least `margin` between its two largest probabilities"""
    x = logits.double().view(-1, G, K)
    if unimix > 0:
        x = torch.log((1 - unimix) * x.softmax(-1) + unimix / K)
    top = x.softmax(-1).topk(min(2, K), -1).values
    gap = (top[..., 0] - top[..., -1]) / top[..., 0] if K > 1 else torch.ones_like(top[..., 0])
    return logits[(gap > margin).all(-1)]


def make():
    ref_harness.install()
    from torch import nn
    from torch.distributions import OneHotCategoricalStraightThrough

    from sheeprl.algos.dreamer_v3.agent import RSSM, Actor
    from sheeprl.models.models import LayerNormGRUCell

    g = torch.Generator().manual_seed(7)
    fx = {}
    for owner, G, K, unimix in CAT_CASES:
        unimix = f32(unimix)
        M = 64
        raw = clear_rows(torch.randn(2 * M, G * K, generator=g) * 2, G, K, unimix)[:M].contiguous()
        dz, dmix = torch.randn(M, G * K, generator=g), torch.randn(M, G * K, generator=g)
        out = {}
        for name, a, b in (("dz", dz, None), ("dmix", None, dmix), ("both", dz, dmix)):
            x = raw.double().requires_grad_(True)
            if owner == "rssm":
                me = types.SimpleNamespace(unimix=unimix, discrete=K)
                mix = RSSM._uniform_mix(me, x.view(1, M, G * K)).view(M, G, K)
            else:
                mix = Actor._uniform_mix(types.SimpleNamespace(_unimix=unimix), x).view(M, G, K)
            dist = OneHotCategoricalStraightThrough(logits=mix)
            z = dist.rsample()
            loss = torch.zeros((), dtype=torch.float64)
            if a is not None:
                loss = loss + (z * a.double().view(M, G, K)).sum()
            if b is not None:
                loss = loss + (mix * b.double().view(M, G, K)).sum()
            loss.backward()
            out[f"draw_{name}"] = x.grad
            out["mix"], out["mode"], out["probs"] = mix.detach().reshape(M, -1), dist.mode.reshape(M, -1), \
                dist.probs.detach()
        fx[f"cat_{owner}_G{G}_K{K}_u{unimix}"] = {"args": dict(raw=raw, dz=dz, dmix=dmix, groups=G, K=K,
                                                               unimix=unimix), "out": out}
    # ---- LayerNormGRUCell's gate through the reference's own forward
    for R, scale in ((5, 1.0), (16, 30.0)):
        M = 48
        cell = LayerNormGRUCell(3 * R, R, bias=False, batch_first=False, layer_norm_cls=nn.Identity).double()
        with torch.no_grad():
            cell.linear.weight.zero_()
            cell.linear.weight[:, R:] = torch.eye(3 * R, dtype=torch.float64)
        G = torch.randn(M, 3 * R, generator=g) * scale
        Hin, dH = torch.randn(M, R, generator=g), torch.randn(M, R, generator=g)
        gi, hi = G.double().requires_grad_(True), Hin.double().requires_grad_(True)
        h = cell(gi, hi)
        (h * dH.double()).sum().backward()
        fx[f"gru_R{R}_s{scale}"] = {"args": dict(G=G, Hin=Hin, dH=dH),
                                    "out": dict(h=h.detach(), dG=gi.grad, dHin=hi.grad)}
    return fx


if __name__ == "__main__":
    torch.save(make(), OUT)
    print(OUT)
