"""TEST INFRASTRUCTURE — writes tests/golden/mf_loss_ref.pt by running the REAL REFERENCE's model-free objective and
sampling code in float64 with autograd, on a few hundred small rows:

    python -m oracle.make_golden_mf_loss_ref

policy_loss / value_loss (both branches) / entropy_loss (ppo/loss.py) and normalize_tensor over PPOAgent.forward's
OneHotCategorical (three heads), Normal and tanh_normal log-probs and entropies, with the recurrent rule (normalise
only when more than one row is kept) on a masked batch; normalize_tensor alone; SACActor.forward with its rsample noise
given; SACAgent.get_next_target_q_values; the SAC critic_loss / policy_loss / entropy_loss; and `gae`.

The inputs stay clear of the discrete decisions (ratios at 1 +- clip, value-clip ties), where the float64 reference and
the fp32 decisions of oracle/mf_loss_ref.py may differ by design, and the scalars are fp32-exact (clip 0.25,
ent_coef 2^-7).  SACActor's `+ 1e-6` is a float64 1e-6 here and fp32's in mf_loss_ref (the value a kernel adds); the
SAC rows stay clear of tanh saturation, where that difference would show.  `_tanh_normal` casts the stored actions
with `.float()`; here that cast is the identity, so the run stays in float64, and its clamp
(1 - finfo(dtype).resolution) is then float64's: the stored actions stay inside +-(1 - 1e-6), where either clamp is inactive.
tests/test_mf_loss_ref_cpu.py compares oracle/mf_loss_ref.py with the fixture.
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

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "mf_loss_ref.pt")
CLIP, VF, ENT = 0.25, 0.5, 2.0 ** -7


def f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _ppo_inputs(g, B, mode, dims):
    """heads, stored actions drawn from them, old log-probs giving ratios near 1 or far outside the clip, advantages,
    and values inside / outside the value clip"""
    if mode == 0:
        head = 2 * torch.randn(B, sum(dims), generator=g)
        acts, o = [], 0
        for K in dims:
            acts.append(F.one_hot(torch.multinomial(torch.softmax(head[:, o:o + K], -1), 1, generator=g).reshape(-1),
                                  K).float())
            o += K
        acts = torch.cat(acts, -1)
    else:
        A = dims[0]
        mu, ls = torch.randn(B, A, generator=g), torch.rand(B, A, generator=g) * 3 - 2
        x = mu + ls.exp() * torch.randn(B, A, generator=g)
        acts = x if mode == 1 else torch.tanh(x).clamp(-0.9999, 0.9999)
        head = torch.cat((mu, ls), -1)
    far = torch.where(torch.rand(B, generator=g) < 0.5, 0.4, 2.5)
    target = torch.where(torch.rand(B, generator=g) < 0.6, torch.exp(0.05 * torch.randn(B, generator=g)), far)
    old_lp = torch.randn(B, generator=g)                       # replaced by the caller once the log-probs are known
    adv = torch.randn(B, generator=g) * 2 + 0.3
    old_v = torch.randn(B, generator=g)
    vals = old_v + torch.where(torch.rand(B, generator=g) < 0.5, 0.1, 0.6) * torch.randn(B, generator=g)
    ret = vals + torch.randn(B, generator=g)
    return head, acts, old_lp, adv, vals, old_v, ret, target


def make():
    ref_harness.install()
    from sheeprl.algos.ppo.agent import PPOAgent
    from sheeprl.algos.ppo.loss import entropy_loss, policy_loss, value_loss
    from sheeprl.algos.sac.agent import SACActor, SACAgent
    from sheeprl.algos.sac.loss import critic_loss
    from sheeprl.algos.sac.loss import entropy_loss as sac_entropy_loss
    from sheeprl.algos.sac.loss import policy_loss as sac_policy_loss
    from sheeprl.utils.utils import gae, normalize_tensor

    g = torch.Generator().manual_seed(7)
    fx = {}

    def agent_logp_ent(h, acts, dims, mode):
        me = types.SimpleNamespace(is_continuous=mode > 0, distribution={1: "normal", 2: "tanh_normal"}.get(mode),
                                   feature_extractor=lambda obs: obs, critic=lambda feat: feat)
        if mode == 0:
            me.actor = lambda feat: list(torch.split(h, list(dims), -1))
            actions = list(torch.split(acts.double(), list(dims), -1))
        else:
            me.actor = lambda feat: [h]
            actions = [acts.double()]
        me._normal = types.MethodType(PPOAgent._normal, me)
        me._tanh_normal = types.MethodType(PPOAgent._tanh_normal, me)
        with mock.patch.object(torch.Tensor, "float", lambda self: self):
            _, lp, ent, _ = PPOAgent.forward(me, None, actions)
        return lp.squeeze(-1), ent.squeeze(-1)

    # ---- PPO: three distributions, both value branches, with and without normalisation; a masked (recurrent) batch
    for name, mode, dims, clip_v, norm, masked in (("ppo_cat", 0, (3, 3, 2), True, True, False),
                                                   ("ppo_normal", 1, (4,), False, True, False),
                                                   ("ppo_tanh", 2, (3,), True, False, False),
                                                   ("ppo_masked", 0, (5,), True, True, True)):
        B = 200
        head, acts, _, adv, vals, old_v, ret, target = _ppo_inputs(g, B, mode, dims)
        with torch.no_grad():
            lp0, _ = agent_logp_ent(head.double(), acts, dims, mode)
        old_lp = (lp0 - torch.log(target.double())).float()
        mask = (torch.rand(B, generator=g) < 0.6).float() if masked else None
        keep = torch.ones(B, dtype=torch.bool) if mask is None else mask != 0
        h = head.double().requires_grad_(True)
        v = vals.double().requires_grad_(True)
        lp, ent = agent_logp_ent(h, acts, dims, mode)
        a = adv.double()[keep]
        if norm and len(a) > 1:
            a = normalize_tensor(a)
        pg = policy_loss(lp[keep], old_lp.double()[keep], a, CLIP)
        vl = value_loss(v[keep], old_v.double()[keep], ret.double()[keep], CLIP, clip_v)
        el = entropy_loss(ent[keep])
        (pg + VF * vl + ENT * el).backward()
        args = dict(head=head, actions=acts, old_logp=old_lp, adv=adv, values=vals, old_values=old_v, returns=ret,
                    dims=dims, mode=mode, clip_vloss=clip_v, normalize=norm, clip=CLIP, vf=VF, ent=ENT)
        if masked:
            args["mask"] = mask
        fx[name] = {"args": args, "out": dict(dhead=h.grad, dvalues=v.grad,
                                              losses=torch.stack((pg, vl, el)).detach())}
    # ---- normalize_tensor alone, on an offset vector
    x = torch.randn(300, generator=g) * 0.01 + 50.0
    fx["normalize"] = {"args": dict(x=x), "out": dict(adv=normalize_tensor(x.double()))}
    # ---- SACActor.forward with the rsample noise given, and the actor's gradient
    B, A, nets = 150, 5, 2
    head = torch.cat((torch.randn(B, A, generator=g) * 0.5, torch.rand(B, A, generator=g) * 10 - 7), -1)
    eps = torch.randn(B, A, generator=g) * 0.05                # |x_t| < 3: the fp32 1e-6 moves log(w) by < 1e-12
    scale, bias = torch.rand(A, generator=g) + 0.5, torch.randn(A, generator=g) * 0.2
    dact = torch.randn(nets, B, A, generator=g)
    log_alpha = torch.tensor([-0.75])
    h = head.double().requires_grad_(True)
    me = types.SimpleNamespace(model=lambda o: o, fc_mean=lambda x: x[:, :A], fc_logstd=lambda x: x[:, A:],
                               action_scale=scale.double(), action_bias=bias.double())
    me._get_actions_and_log_probs = types.MethodType(SACActor._get_actions_and_log_probs, me)
    with mock.patch("torch.distributions.normal._standard_normal", lambda shape, dtype, device: eps.to(dtype)):
        action, logp = SACActor.forward(me, h)
    alpha = float(log_alpha.double().exp())
    ((dact.double().sum(0) * action).sum() + (alpha / B) * logp.sum()).backward()
    fx["sac_sample"] = {"args": dict(head=head, eps=eps, scale=scale, bias=bias, dact=dact, log_alpha=log_alpha),
                        "out": dict(action=action.detach(), logp=logp.detach().squeeze(-1), dhead=h.grad)}
    # ---- SACAgent.get_next_target_q_values
    gamma = f32(0.99)
    q = torch.randn(nets, B, generator=g) * 3
    lp_next, rew = torch.randn(B, generator=g) * 2, torch.randn(B, generator=g)
    term = (torch.rand(B, generator=g) < 0.3).float()
    me = types.SimpleNamespace(get_actions_and_log_probs=lambda o: (None, lp_next.double().unsqueeze(-1)),
                               get_target_q_values=lambda o, a: q.double().t(), alpha=alpha)
    y = SACAgent.get_next_target_q_values(me, None, rew.double().unsqueeze(-1), term.double().unsqueeze(-1), gamma)
    fx["sac_target"] = {"args": dict(q=q, logp=lp_next, rewards=rew, terminated=term, log_alpha=log_alpha,
                                     gamma=gamma), "out": dict(y=y.squeeze(-1))}
    # ---- the SAC losses (sac.py train: critic_loss, policy_loss over the min critic, entropy_loss)
    qv = torch.randn(nets, B, generator=g) * 3
    ytgt, lp = torch.randn(B, generator=g) * 3, torch.randn(B, generator=g) * 2
    te = -float(A)
    qc = qv.double().t().contiguous().requires_grad_(True)
    critic_loss(qc, ytgt.double().unsqueeze(-1), nets).backward()
    qa = qv.double().t().contiguous().requires_grad_(True)
    la = log_alpha.double().requires_grad_(True)
    lpd = lp.double().unsqueeze(-1)
    actor = sac_policy_loss(alpha, lpd, torch.min(qa, dim=-1, keepdim=True)[0])
    actor.backward()
    alpha_l = sac_entropy_loss(la, lpd, torch.tensor(te, dtype=torch.float64))
    alpha_l.backward()
    fx["sac_losses"] = {"args": dict(q=qv, y=ytgt, logp=lp, log_alpha=log_alpha, target_entropy=te),
                        "out": dict(critic_loss=critic_loss(qc.detach(), ytgt.double().unsqueeze(-1), nets).reshape(1),
                                    dq_critic=qc.grad.t(), actor_loss=actor.detach().reshape(1), dq_actor=qa.grad.t(),
                                    alpha_loss=alpha_l.detach().reshape(1), dlog_alpha=la.grad)}
    # ---- gae (utils.py), dones in every pattern
    T, E = 9, 6
    r, v = torch.randn(T, E, generator=g), torch.randn(T, E, generator=g) * 2
    d = (torch.rand(T, E, generator=g) < 0.3).float()
    d[:, 0], d[:, 1] = 0.0, 1.0
    d[::2, 2] = 1.0
    nv = torch.randn(1, E, generator=g)
    gm, lm = f32(0.99), f32(0.95)
    ret, adv = gae(r.double(), v.double(), d.double(), nv.double(), T, gm, lm)
    fx["gae"] = {"args": dict(rewards=r, values=v, dones=d, next_value=nv, gamma=gm, lmbda=lm),
                 "out": dict(returns=ret, advantages=adv)}
    return fx


if __name__ == "__main__":
    torch.save(make(), OUT)
    print(OUT)
