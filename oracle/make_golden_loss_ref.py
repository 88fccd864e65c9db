"""TEST INFRASTRUCTURE — writes tests/golden/dv3_loss_ref.pt by running the REAL REFERENCE's distributions and objective
pieces in float64 with autograd, on a few hundred small rows:

    python -m oracle.make_golden_loss_ref

TwoHotEncodingDistribution.log_prob / .mean, MSEDistribution, BernoulliSafeMode, the KL of loss.py with free nats,
compute_lambda_values with BernoulliSafeMode.mode continues and the discount cumprod, Moments (at decay 0, where the
state is torch.quantile itself), Actor._uniform_mix with OneHotCategoricalStraightThrough for the discrete objective,
and Actor.forward's `scaled_normal` branch with its detached clip for the continuous actor.  The inputs stay clear of the
discrete decisions (bin edges, sigmoid(l) = 0.5, KL = free nats), where the float64 reference and the fp32 decisions
of oracle/loss_ref.py may differ by design.  tests/test_loss_ref_cpu.py compares oracle/loss_ref.py with the fixture.
"""
from __future__ import annotations

import os
import sys
import types
from unittest import mock

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import ref_harness  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "dv3_loss_ref.pt")
LOW, HIGH = -20.0, 20.0


def _g(seed):
    return torch.Generator().manual_seed(seed)


def f32(v):
    """scalar parameters are the fp32 values the kernels receive, so they are fp32-exact here"""
    return float(torch.tensor(v, dtype=torch.float32))


def make():
    ref_harness.install()
    from torch.distributions import Independent, OneHotCategoricalStraightThrough
    from torch.distributions.kl import kl_divergence

    from sheeprl.algos.dreamer_v3.agent import Actor
    from sheeprl.algos.dreamer_v3.utils import Moments, compute_lambda_values
    from sheeprl.utils.distribution import BernoulliSafeMode, MSEDistribution, TwoHotEncodingDistribution

    def d64(t):
        return t.detach().double().requires_grad_(True)

    fx = {}
    # ---- two-hot log_prob and mean
    g = _g(1)
    M, nb = 200, 63
    logits = torch.randn(M, nb, generator=g) * 2
    x = torch.sign(torch.randn(M, generator=g)) * (torch.exp(torch.rand(M, generator=g) * 12) - 1)
    weight = torch.rand(M, generator=g) + 0.5
    d_mean = torch.randn(M, generator=g)
    l = d64(logits)
    loss = -TwoHotEncodingDistribution(l, dims=1, low=LOW, high=HIGH).log_prob(x.double().unsqueeze(-1))
    (0.25 * weight.double() * loss).sum().backward()
    lm = d64(logits)
    mean = TwoHotEncodingDistribution(lm, dims=1, low=LOW, high=HIGH).mean.squeeze(-1)
    (mean * d_mean.double()).sum().backward()
    fx["twohot"] = {"args": dict(logits=logits, x=x, weight=weight, scale=0.25, d_mean=d_mean),
                    "out": dict(loss=loss.detach(), grad=l.grad, mean=mean.detach(), mean_grad=lm.grad)}
    # ---- MSE
    pred, target = torch.randn(100, 9, generator=g), torch.randn(100, 9, generator=g)
    p = d64(pred)
    loss = -MSEDistribution(p, dims=1).log_prob(target.double())
    (0.125 * loss).sum().backward()
    fx["mse"] = {"args": dict(pred=pred, target=target, scale=0.125), "out": dict(loss=loss.detach(), grad=p.grad)}
    # ---- Bernoulli continue head
    logit = torch.cat([torch.randn(300, generator=g) * 4, torch.tensor([25.0, -25.0, 30.0, -30.0])])
    tgt = (torch.rand(logit.numel(), generator=g) > 0.3).double()
    lo = d64(logit)
    loss = -1.0 * BernoulliSafeMode(logits=lo).log_prob(tgt)
    (0.5 * loss).sum().backward()
    fx["bce"] = {"args": dict(logit=logit, target=tgt.float(), loss_scale=1.0, scale=0.5),
                 "out": dict(loss=loss.detach(), grad=lo.grad)}
    # ---- KL with free nats (loss.py)
    M, G, K = 64, 4, 5
    post, prior = torch.randn(M, G * K, generator=g) * 1.5, torch.randn(M, G * K, generator=g) * 1.5
    a, b = d64(post), d64(prior)

    def dist(z):
        return Independent(OneHotCategoricalStraightThrough(logits=z.view(M, G, K)), 1)

    kl = kl_divergence(dist(a.detach()), dist(b.detach()))
    srt = kl.sort().values
    free = float(torch.tensor(float(srt[M // 2 - 1] + srt[M // 2]) / 2, dtype=torch.float32))
    dyn = kl_divergence(dist(a.detach()), dist(b))
    rep = kl_divergence(dist(a), dist(b.detach()))
    fr = torch.full_like(dyn, free)
    kl_loss = 0.5 * torch.maximum(dyn, fr) + f32(0.1) * torch.maximum(rep, fr)
    (0.25 * 1.0 * kl_loss).sum().backward()
    rows = torch.stack((kl, (0.5 + f32(0.1)) * torch.maximum(kl, fr), dist(a.detach()).entropy(),
                        dist(b.detach()).entropy()), -1)
    fx["kl"] = {"args": dict(post=post, prior=prior, groups=G, K=K, free=free, scale=0.25),
                "out": dict(rows=rows, d_post=a.grad, d_prior=b.grad)}
    # ---- lambda values, discount (dreamer_v3.py), and the continuous objective's gradient through them
    H, N = 6, 50
    gamma, lmbda, ent_coef = f32(0.997), 0.75, 0.0625
    rew, val = torch.randn(H + 1, N, generator=g), torch.randn(H + 1, N, generator=g) * 3
    cl = torch.randn(H + 1, N, generator=g) * 4
    cl = torch.where(cl.abs() < 0.1, torch.full_like(cl, 0.5), cl)
    tc = (torch.rand(N, generator=g) > 0.2).float()
    mom = torch.tensor([0.25, 2.0])
    ent = torch.randn(H * N, generator=g)
    c = BernoulliSafeMode(logits=cl.double()).mode
    c = torch.cat((tc.double().reshape(1, -1), c[1:]))
    lam = compute_lambda_values(rew.double()[1:], val.double()[1:], c[1:] * gamma, lmbda=lmbda)
    disc = torch.cumprod(c * gamma, 0) / gamma
    fx["lambda"] = {"args": dict(rew=rew, val=val, cont_logit=cl, true_cont=tc, gamma=gamma, lmbda=lmbda,
                                 moments=mom, ent=ent, ent_coef=ent_coef, scale=1.0 / 64),
                    "out": dict(lam=lam, discount=disc)}
    r, v = d64(rew), d64(val)
    lam_g = compute_lambda_values(r[1:], v[1:], c[1:] * gamma, lmbda=lmbda)
    lam32, disc32 = lam.float().double(), disc.float().double()
    off, inv = float(mom[0]), float(mom[1])
    adv = (lam_g - off) / inv - (v[:-1] - off) / inv
    (-(1.0 / 64) * (disc32[:-1] * (adv + ent_coef * ent.double().view(H, N))).sum()).backward()
    rows = disc32[:-1] * ((lam32 - off) / inv - (val.double()[:-1] - off) / inv + ent_coef * ent.double().view(H, N))
    r_grad = r.grad.clone()
    r_grad[0] = 0.0
    fx["lambda"]["out"].update(rows=rows, d_val=v.grad, d_rew=r_grad)
    # ---- Moments at decay 0: the state is torch.quantile of the values
    xs = torch.randn(1001, generator=g) * 3
    m = Moments(decay=0.0, max_=1e8, percentile_low=0.05, percentile_high=0.95)
    low, _ = m(xs, ref_harness.FakeFabric())
    fx["moments"] = {"args": dict(x=xs, state=torch.zeros(2), decay=0.0, max=1e8),
                     "out": dict(state=torch.stack((m.low, m.high)).double())}
    # ---- discrete objective with unimix (dreamer_v3.py:272-297)
    ent_coef = f32(3e-4)
    for unimix in (0.0, f32(0.01)):
        M, heads = 120, (3, 7, 2)
        raw = torch.randn(M, sum(heads), generator=g) * 2
        idx = [torch.randint(0, k, (M,), generator=g) for k in heads]
        acts = torch.cat([F.one_hot(i, k).float() for i, k in zip(idx, heads)], 1)
        lamv, valv, dsc = torch.randn(M, generator=g), torch.randn(M, generator=g), torch.rand(M, generator=g)
        x = d64(raw)
        me = types.SimpleNamespace(_unimix=unimix)
        adv = (lamv.double() - off) / inv - (valv.double() - off) / inv
        obj, entr, o = 0.0, 0.0, 0
        for k in heads:
            pd = OneHotCategoricalStraightThrough(logits=Actor._uniform_mix(me, x[:, o:o + k]))
            obj = obj + pd.log_prob(acts[:, o:o + k].double()) * adv
            entr = entr + pd.entropy()
            o += k
        rows = dsc.double() * (obj + ent_coef * entr)
        (-f32(1.0 / M) * rows).sum().backward()
        fx[f"actor_u{unimix}"] = {"args": dict(raw=raw, actions=acts, lam=lamv, val=valv, discount=dsc, moments=mom,
                                               heads=heads, unimix=unimix, ent_coef=ent_coef, scale=f32(1.0 / M)),
                                  "out": dict(rows=rows.detach(), draw=x.grad)}
    # ---- the scaled_normal actor (agent.py Actor.forward) with its detached clip factor
    M, A = 150, 4
    head, eps = torch.randn(M, 2 * A, generator=g) * 2, torch.randn(M, A, generator=g) * 1.5
    dact, dsc = torch.randn(M, A, generator=g), torch.rand(M, generator=g)
    cfg = (f32(0.1), 1.0, 2.0, 1.0)
    me = types.SimpleNamespace(model=lambda s: s, mlp_heads=[lambda s: s], is_continuous=True,
                               distribution="scaled_normal", min_std=cfg[0], max_std=cfg[1], init_std=cfg[2],
                               _action_clip=cfg[3])
    h = d64(head)
    with mock.patch("torch.distributions.normal._standard_normal", lambda shape, dtype, device: eps.to(dtype)):
        actions, dists = Actor.forward(me, h)
    ent_scale = f32(-0.01)
    ((actions[0] * dact.double()).sum() + (ent_scale * dsc.double() * dists[0].entropy()).sum()).backward()
    fx["cont"] = {"args": dict(head=head, eps=eps, cfg=cfg, d_action=dact, discount=dsc, ent_scale=ent_scale),
                  "out": dict(action=actions[0].detach(), ent=dists[0].entropy().detach(), dhead=h.grad)}
    return fx


if __name__ == "__main__":
    torch.save(make(), OUT)
    print(OUT)
