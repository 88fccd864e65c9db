"""TEST INFRASTRUCTURE (oracle) — NOT part of the product path.

CPU restatement, in plain fp32 PyTorch, of the reference's Dreamer-V3 update step
(`sheeprl/algos/dreamer_v3/dreamer_v3.py:48-357`).  It is written functionally over state-dict
shaped parameter dictionaries (the key names are the reference's own, SURVEY.md §8b) so that the
same weights can be fed to the reference, to this oracle and to the CUDA engine.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may
import this module.  The product package `sheeprl_b200` never does.

Parity status: PINNED against the executed reference — `tests/test_oracle_pin.py` runs the unmodified
reference `build_agent` + `train()` (imported through `oracle/ref_harness.py`, container only) on
the same weights / batch / injected sampling noise and compares every post-step parameter and the
13 logged metrics; `oracle/make_golden.py` freezes the same comparison into `tests/golden/`.

Stochastic nodes draw from *injected* noise (SURVEY.md §0 F8): a categorical sample is
`argmax(probs / q)`, q ~ Exp(1), which is what `torch.multinomial(p, 1, True)` computes on CPU.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
FP32_EPS = torch.finfo(torch.float32).eps


# --------------------------------------------------------------------------------------------------
# small pieces
# --------------------------------------------------------------------------------------------------
def symlog(x: Tensor) -> Tensor:  # reference: sheeprl/utils/utils.py:148
    return torch.sign(x) * torch.log(1 + torch.abs(x))


def symexp(x: Tensor) -> Tensor:  # reference: sheeprl/utils/utils.py:152
    return torch.sign(x) * (torch.exp(torch.abs(x)) - 1)


def layer_norm(x: Tensor, w: Tensor, b: Tensor, eps: float) -> Tensor:
    return F.layer_norm(x, (x.shape[-1],), w, b, eps)


def dense_stack(p: Dict[str, Tensor], prefix: str, x: Tensor, n_hidden: int, eps: float, final: bool) -> Tensor:
    """`n_hidden` x [Linear(no bias) -> LayerNorm -> SiLU] (+ final Linear with bias).

    Reference: MLP built by `miniblock` (sheeprl/models/models.py:16-119, utils/model.py:34-88);
    Sequential indices: 3i = Linear, 3i+1 = LayerNorm, 3i+2 = SiLU, 3*n_hidden = output Linear."""
    for i in range(n_hidden):
        x = F.linear(x, p[f"{prefix}{3 * i}.weight"])
        x = F.silu(layer_norm(x, p[f"{prefix}{3 * i + 1}.weight"], p[f"{prefix}{3 * i + 1}.bias"], eps))
    if final:
        x = F.linear(x, p[f"{prefix}{3 * n_hidden}.weight"], p[f"{prefix}{3 * n_hidden}.bias"])
    return x


def unimix_logits(raw: Tensor, groups: int, classes: int, unimix: float) -> Tensor:
    """log(clamp((1-u)*softmax + u/K)) per K-way group.  Reference: agent.py:437-449, :839-845;
    torch.distributions.utils.probs_to_logits (clamp to [eps, 1-eps])."""
    shp = raw.shape
    x = raw.reshape(*shp[:-1], groups, classes)
    if unimix > 0.0:
        pr = torch.softmax(x, -1)
        pr = (1 - unimix) * pr + unimix / classes
        x = torch.log(pr.clamp(FP32_EPS, 1 - FP32_EPS))
    return x.reshape(shp)


def categorical_normalise(logits: Tensor) -> Tuple[Tensor, Tensor]:
    """torch Categorical(logits=...) ctor: logits - logsumexp, probs = softmax (categorical.py)."""
    lg = logits - torch.logsumexp(logits, -1, keepdim=True)
    return lg, torch.softmax(lg, -1)


def st_sample(logits_mix: Tensor, groups: int, classes: int, q: Optional[Tensor],
              condition_margin: float = 0.0) -> Tensor:
    """OneHotCategoricalStraightThrough.rsample with injected Exp(1) noise `q` (None -> mode).

    Reference: dreamer_v2/utils.py:44-61; torch one_hot_categorical.py:140-143 (value = one-hot +
    probs - probs.detach()).  When `condition_margin` > 0 near-ties (top-2 ratio within the margin) are
    removed by shrinking the winner's q in place, which leaves the drawn index unchanged: tests use
    this so that 1-ulp differences in `probs` cannot flip a sample."""
    shp = logits_mix.shape
    lg, pr = categorical_normalise(logits_mix.reshape(*shp[:-1], groups, classes))
    if q is None:
        idx = pr.argmax(-1)
        return F.one_hot(idx, classes).to(pr.dtype).reshape(shp)
    qv = q.reshape(pr.shape)
    ratio = pr.detach() / qv
    if condition_margin > 0.0:
        top2 = ratio.topk(2, -1)
        tight = top2.values[..., 0] < top2.values[..., 1] * (1.0 + condition_margin)
        if bool(tight.any()):
            win = top2.indices[..., 0:1]
            cur = qv.gather(-1, win)
            qv.scatter_(-1, win, torch.where(tight.unsqueeze(-1), cur * 0.25, cur))
            ratio = pr.detach() / qv
    idx = ratio.argmax(-1)
    hot = F.one_hot(idx, classes).to(pr.dtype)
    return (hot + pr - pr.detach()).reshape(shp)


def twohot_log_prob(logits: Tensor, x: Tensor, low: float = -20.0, high: float = 20.0) -> Tensor:
    """TwoHotEncodingDistribution(logits, dims=1).log_prob(x), x [...,1] -> [...].
    Reference: sheeprl/utils/distribution.py:224-276."""
    nb = logits.shape[-1]
    bins = torch.linspace(low, high, nb, device=logits.device)
    x = symlog(x)
    below = (bins <= x).to(torch.int32).sum(-1, keepdim=True) - 1
    above = torch.clamp(below + 1, max=nb - 1)
    below = torch.clamp(below, min=0)
    same = below == above
    d_lo = torch.where(same, torch.ones_like(x), (bins[below] - x).abs())
    d_hi = torch.where(same, torch.ones_like(x), (bins[above] - x).abs())
    tot = d_lo + d_hi
    target = (F.one_hot(below.long(), nb) * (d_hi / tot)[..., None]
              + F.one_hot(above.long(), nb) * (d_lo / tot)[..., None]).squeeze(-2)
    logp = logits - torch.logsumexp(logits, -1, keepdim=True)
    return (target * logp).sum(-1)


def twohot_mean(logits: Tensor, low: float = -20.0, high: float = 20.0) -> Tensor:
    """TwoHotEncodingDistribution.mean (distribution.py:245-247): symexp(sum softmax*bins), keepdim."""
    bins = torch.linspace(low, high, logits.shape[-1], device=logits.device)
    return symexp((torch.softmax(logits, -1) * bins).sum(-1, keepdim=True))


def categorical_kl(post_mix: Tensor, prior_mix: Tensor, groups: int, classes: int) -> Tensor:
    """kl_divergence(Independent(OHC(post),1), Independent(OHC(prior),1)) -> [...]
    Reference: torch kl.py `_kl_categorical_categorical` (+inf / 0 masks) summed over groups."""
    lp, pp = categorical_normalise(post_mix.reshape(*post_mix.shape[:-1], groups, classes))
    lq, pq = categorical_normalise(prior_mix.reshape(*prior_mix.shape[:-1], groups, classes))
    t = pp * (lp - lq)
    t = torch.where(pq == 0, torch.full_like(t, math.inf), t)
    t = torch.where(pp == 0, torch.zeros_like(t), t)
    return t.sum(-1).sum(-1)


def categorical_entropy(logits_mix: Tensor, groups: int, classes: int) -> Tensor:
    """Independent(OneHotCategorical(logits), 1).entropy() (categorical.py:159-163)."""
    lg, pr = categorical_normalise(logits_mix.reshape(*logits_mix.shape[:-1], groups, classes))
    lg = torch.clamp(lg, min=torch.finfo(lg.dtype).min)
    return -(lg * pr).sum(-1).sum(-1)


# --------------------------------------------------------------------------------------------------
# networks
# --------------------------------------------------------------------------------------------------
def vec_dims(cfg) -> Dict[str, int]:
    """{vector observation key: dimension} — the reference reads these from the observation space; the synthetic
    configs of the tests / bench carry them under cfg.env.mlp_dims"""
    return dict(cfg.env.get("mlp_dims", {}) or {})


def mlp_encoder_forward(wm: Dict[str, Tensor], data: Dict[str, Tensor], keys: Sequence[str], n_hidden: int, eps: float):
    """MLPEncoder (agent.py:100-152): symlog of the concatenated vectors -> n x [Linear nobias -> LN -> SiLU].
    Returns (features, symlog inputs per key)."""
    xs = [symlog(data[k].float()) for k in keys]
    return dense_stack(wm, "encoder.mlp_encoder.model._model.", torch.cat(xs, -1), n_hidden, eps, False), xs


def mlp_decoder_loss(wm: Dict[str, Tensor], latent: Tensor, targets: Sequence[Tensor], n_hidden: int, eps: float) -> Tensor:
    """MLPDecoder (agent.py:229-278) + SymlogDistribution.log_prob (utils/distribution.py:177-192, dist "mse", agg "sum",
    tol 1e-8): sum over keys of sum_d (head_k(x) - symlog(obs_k))^2, squared distances below tol zeroed."""
    hid = dense_stack(wm, "observation_model.mlp_decoder.model._model.", latent, n_hidden, eps, False)
    loss = 0.0
    for i, tgt in enumerate(targets):
        rec = F.linear(hid, wm[f"observation_model.mlp_decoder.heads.{i}.weight"], wm[f"observation_model.mlp_decoder.heads.{i}.bias"])
        dist = (rec - tgt) ** 2
        dist = torch.where(dist < 1e-8, torch.zeros_like(dist), dist)
        loss = loss + dist.sum(-1)
    return loss


def encoder_forward(wm: Dict[str, Tensor], obs: Tensor, stages: int, eps: float) -> Tensor:
    """CNNEncoder (agent.py:42-97): stages x [Conv2d k4 s2 p1 nobias -> LN(channel) -> SiLU] -> flatten CHW.
    obs: [T,B,C,H,W] already normalised."""
    lead = obs.shape[:-3]
    x = obs.reshape(-1, *obs.shape[-3:])
    pre = "encoder.cnn_encoder.model.0._model."
    for i in range(stages):
        x = F.conv2d(x, wm[f"{pre}{3 * i}.weight"], None, stride=2, padding=1)
        x = layer_norm(x.permute(0, 2, 3, 1), wm[f"{pre}{3 * i + 1}.weight"], wm[f"{pre}{3 * i + 1}.bias"], eps)
        x = F.silu(x.permute(0, 3, 1, 2))
    return x.reshape(*lead, -1)


def decoder_forward(wm: Dict[str, Tensor], latent: Tensor, stages: int, eps: float, out_shape) -> Tensor:
    """CNNDecoder (agent.py:154-226): Linear -> (C,4,4) -> (stages-1) x [ConvT k4 s2 p1 nobias, LN, SiLU]
    -> ConvT(+bias)."""
    lead = latent.shape[:-1]
    x = latent.reshape(-1, latent.shape[-1])
    pre = "observation_model.cnn_decoder.model."
    x = F.linear(x, wm[f"{pre}0.weight"], wm[f"{pre}0.bias"])
    x = x.reshape(x.shape[0], -1, 4, 4)
    for i in range(stages - 1):
        x = F.conv_transpose2d(x, wm[f"{pre}2._model.{3 * i}.weight"], None, stride=2, padding=1)
        x = layer_norm(x.permute(0, 2, 3, 1), wm[f"{pre}2._model.{3 * i + 1}.weight"],
                       wm[f"{pre}2._model.{3 * i + 1}.bias"], eps)
        x = F.silu(x.permute(0, 3, 1, 2))
    j = 3 * (stages - 1)
    x = F.conv_transpose2d(x, wm[f"{pre}2._model.{j}.weight"], wm[f"{pre}2._model.{j}.bias"], stride=2, padding=1)
    return x.reshape(*lead, *out_shape)


def recurrent_step(wm: Dict[str, Tensor], z: Tensor, a: Tensor, h: Tensor, eps: float,
                   saves: Optional[Dict[str, Tensor]] = None) -> Tensor:
    """RecurrentModel.forward (agent.py:328-341) + LayerNormGRUCell (models.py:370-410):
    x = SiLU(LN(W_in [z,a])); g = LN(W_g [h,x]); r,c,u = chunk(g); h' = u'*tanh(sig(r)*c) + (1-u')*h,
    u' = sig(u - 1).  `saves`: if given, receives the intermediates x_pre, x_act, g_pre, g_ln (graph nodes)."""
    p = "rssm.recurrent_model."
    x_pre = F.linear(torch.cat((z, a), -1), wm[p + "mlp._model.0.weight"])
    x = F.silu(layer_norm(x_pre, wm[p + "mlp._model.1.weight"], wm[p + "mlp._model.1.bias"], eps))
    g_pre = F.linear(torch.cat((h, x), -1), wm[p + "rnn.linear.weight"])
    g = layer_norm(g_pre, wm[p + "rnn.layer_norm.weight"], wm[p + "rnn.layer_norm.bias"], eps)
    if saves is not None:
        saves.update(x_pre=x_pre, x_act=x, g_pre=g_pre, g_ln=g)
    r, c, u = torch.chunk(g, 3, -1)
    c = torch.tanh(torch.sigmoid(r) * c)
    u = torch.sigmoid(u - 1)
    return u * c + (1 - u) * h


def transition_logits(wm, h, S, D, unimix, eps):  # agent.py:467-480
    raw = dense_stack(wm, "rssm.transition_model._model.", h, 1, eps, True)
    return unimix_logits(raw, S, D, unimix)


def representation_logits(wm, h, e, S, D, unimix, eps):  # agent.py:451-465 (input order [h, embed])
    raw = dense_stack(wm, "rssm.representation_model._model.", torch.cat((h, e), -1), 1, eps, True)
    return unimix_logits(raw, S, D, unimix)


def actor_logits(actor: Dict[str, Tensor], x: Tensor, n_hidden: int, actions_dim: Sequence[int],
                 unimix: float, eps: float) -> List[Tensor]:
    """Actor.forward, discrete branch (agent.py:783-845): MLP trunk, one Linear head per action
    dimension, unimix per head."""
    hdn = dense_stack(actor, "model._model.", x, n_hidden, eps, False)
    out = []
    for i, ad in enumerate(actions_dim):
        raw = F.linear(hdn, actor[f"mlp_heads.{i}.weight"], actor[f"mlp_heads.{i}.bias"])
        out.append(unimix_logits(raw, 1, ad, unimix))
    return out


# --------------------------------------------------------------------------------------------------
# optimiser restatement
# --------------------------------------------------------------------------------------------------
def clip_grad_norm(grads: Sequence[Tensor], max_norm: float) -> Tensor:
    """torch.nn.utils.clip_grad_norm_ (norm_type=2): returns pre-clip norm, scales in place."""
    total = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(g) for g in grads]))
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for g in grads:
        g.mul_(coef)
    return total


class AdamState:
    """torch.optim.Adam(betas=(0.9,0.999), weight_decay=0, amsgrad=False) restated; per-parameter
    state {step, exp_avg, exp_avg_sq} like torch's."""

    def __init__(self, params: Dict[str, Tensor], lr: float, eps: float, betas=(0.9, 0.999)):
        self.lr, self.eps, self.b1, self.b2 = lr, eps, betas[0], betas[1]
        self.step_count = 0
        self.m = {k: torch.zeros_like(v) for k, v in params.items()}
        self.v = {k: torch.zeros_like(v) for k, v in params.items()}

    @torch.no_grad()
    def step(self, params: Dict[str, Tensor], grads: Dict[str, Tensor]):
        self.step_count += 1
        t = self.step_count
        bc1 = 1 - self.b1 ** t
        bc2 = 1 - self.b2 ** t
        for k, p in params.items():
            g = grads[k]
            self.m[k].lerp_(g, 1 - self.b1)
            self.v[k].mul_(self.b2).addcmul_(g, g, value=1 - self.b2)
            denom = (self.v[k].sqrt() / math.sqrt(bc2)).add_(self.eps)
            p.addcdiv_(self.m[k], denom, value=-self.lr / bc1)


# --------------------------------------------------------------------------------------------------
# the update step
# --------------------------------------------------------------------------------------------------
def draw_noise(T: int, B: int, H: int, S: int, D: int, actions_dim: Sequence[int], seed: int,
               is_continuous: bool = False) -> Dict[str, Tensor]:
    """Exp(1) noise for every categorical draw; continuous actions: one N(0,1) tensor [H+1, N, sum(A)] consumed by
    Normal.rsample (agent.py:817)."""
    g = torch.Generator().manual_seed(seed)
    N = T * B

    def exp1(*shape):
        return torch.empty(*shape).exponential_(1.0, generator=g)

    return {
        "prior": exp1(T, B, S, D),       # consumed by the reference, discarded by training (agent.py:433)
        "post": exp1(T, B, S, D),
        "img_state": exp1(H, N, S, D),
        "img_action": ([torch.randn(H + 1, N, int(sum(actions_dim)), generator=g)] if is_continuous
                       else [exp1(H + 1, N, ad) for ad in actions_dim]),
    }


def continuous_action(head: Tensor, eps_n: Tensor, acfg):
    """Actor.forward, continuous `scaled_normal` branch (agent.py:803-825): returns (clipped action, entropy)."""
    mean, std = torch.chunk(head, 2, -1)
    std = (acfg.max_std - acfg.min_std) * torch.sigmoid(std + acfg.init_std) + acfg.min_std
    act = torch.tanh(mean) + std * eps_n
    if acfg.action_clip > 0.0:
        clip = torch.full_like(act, acfg.action_clip)
        act = act * (clip / torch.maximum(clip, act.abs())).detach()
    ent = (0.5 + 0.5 * math.log(2 * math.pi) + torch.log(std)).sum(-1)
    return act, ent


def reference_normal_order(noise: Dict[str, Tensor], H: int) -> List[Tensor]:
    """N(0,1) tensors in the order the reference calls Normal.rsample with continuous actions: one per imagination
    step (dreamer_v3.py:219,240) and one (discarded) for the re-evaluation on the whole trajectory (:273)."""
    e = noise["img_action"][0]
    return [e[i] for i in range(H + 1)] + [torch.zeros_like(e)]


def reference_noise_order(noise: Dict[str, Tensor], T: int, H: int, n_heads: int) -> List[Tensor]:
    """Flatten `noise` in the order the reference's train() calls torch.multinomial
    (prior then posterior per step: agent.py:433-434; actor then transition per imagination step:
    dreamer_v3.py:219,236-240)."""
    out = []
    for t in range(T):
        out += [noise["prior"][t], noise["post"][t]]
    out += [noise["img_action"][k][0] for k in range(n_heads)]
    for i in range(1, H + 1):
        out.append(noise["img_state"][i - 1])
        out += [noise["img_action"][k][i] for k in range(n_heads)]
    # the reference re-evaluates the actor on the whole trajectory (dreamer_v3.py:273); that forward
    # also draws (discarded) action samples, one multinomial call per head over (H+1)*N rows
    out += [torch.ones(noise["img_action"][k].shape).reshape(-1, noise["img_action"][k].shape[-1])
            for k in range(n_heads)]
    return out


def world_model_phase(cfg, wm: Dict[str, Tensor], opt_wm: "AdamState", data: Dict[str, Tensor], noise: Dict[str, Tensor],
                      condition_margin: float, keep: bool, out: Dict[str, Tensor], detach_heads: bool = False):
    """Dynamic learning (dreamer_v3.py:98-200; identical in p2e_dv3_exploration.py:113-205): encoder, RSSM scan, heads,
    reconstruction loss, backward, clip, Adam on `wm` (which must already require grad).  Fills the 9 world-model
    metrics into `out`; returns (zs [T,B,Z], hs [T,B,R], cont_target [T,B,1]).  detach_heads: the reward / continue
    heads read `latent.detach()` (p2e_dv3_exploration.py:157,160: their losses do not shape the latent state)."""
    a = cfg.algo
    w = a.world_model
    T, B = a.per_rank_sequence_length, a.per_rank_batch_size
    S, D = w.stochastic_size, w.discrete_size
    Z, R = S * D, w.recurrent_model.recurrent_state_size
    eps = a.mlp_layer_norm.kw.eps
    ceps = a.cnn_layer_norm.kw.eps
    um = a.unimix
    stages = int(round(math.log2(cfg.env.screen_size) - 2))
    cnn_keys, vkeys = list(a.cnn_keys.encoder), list(a.mlp_keys.encoder)
    n_hid = a.mlp_layers

    # ---- dreamer_v3.py:98-104
    # several image keys are concatenated on the channel axis (CNNEncoder.forward agent.py:96); the decoder's per-key
    # MSE terms (CNNDecoder splits its output, agent.py:226) add up to the MSE over the concatenated image
    obs = torch.cat([data[k].float() for k in cnn_keys], -3) / 255.0 - 0.5 if cnn_keys else None
    is_first = data["is_first"].float().clone()
    is_first[0] = 1.0
    actions = torch.cat((torch.zeros_like(data["actions"][:1]), data["actions"][:-1]), 0).float()
    rewards = data["rewards"].float()
    cont_target = 1 - data["terminated"].float()

    # ---- encoder + RSSM scan (dreamer_v3.py:113-146; agent.py:396-435)
    embs, vtargets = [], []
    if cnn_keys:
        embs.append(encoder_forward(wm, obs, stages, ceps))
    if vkeys:                                  # MultiEncoder: cnn features first, then the vector features (models.py:466-475)
        vemb, vtargets = mlp_encoder_forward(wm, data, vkeys, w.encoder.mlp_layers, w.encoder.mlp_layer_norm.kw.eps)
        embs.append(vemb)
    emb = torch.cat(embs, -1)
    h = torch.zeros(B, R, device=emb.device)
    z = torch.zeros(B, Z, device=emb.device)
    hs, zs, post_l, prior_l = [], [], [], []
    h0_raw = wm["rssm.initial_recurrent_state"]
    if not w.get("learnable_initial_recurrent_state", True):     # a buffer, not a parameter (agent.py:382-389)
        h0_raw = h0_raw.detach()
    h0 = torch.tanh(h0_raw).expand(B, R)
    for t in range(T):
        f = is_first[t]
        act = (1 - f) * actions[t]
        z0 = st_sample(transition_logits(wm, h0, S, D, um, eps), S, D, None)
        h = (1 - f) * h + f * h0
        z = (1 - f) * z + f * z0
        h = recurrent_step(wm, z, act, h, eps)
        pl = transition_logits(wm, h, S, D, um, eps)
        ql = representation_logits(wm, h, emb[t], S, D, um, eps)
        z = st_sample(ql, S, D, noise["post"][t], condition_margin)
        hs.append(h), zs.append(z), post_l.append(ql), prior_l.append(pl)
    hs, zs = torch.stack(hs), torch.stack(zs)
    post_l, prior_l = torch.stack(post_l), torch.stack(prior_l)
    latent = torch.cat((zs, hs), -1)

    # ---- heads + losses (dreamer_v3.py:149-190, loss.py:9-88)
    obs_loss, recon = 0.0, None
    if cnn_keys:
        recon = decoder_forward(wm, latent, stages, ceps, obs.shape[-3:])
        obs_loss = ((recon - obs) ** 2).sum((-3, -2, -1))
    if vkeys:
        obs_loss = obs_loss + mlp_decoder_loss(wm, latent, vtargets, w.observation_model.mlp_layers,
                                               w.observation_model.mlp_layer_norm.kw.eps)
    head_in = latent.detach() if detach_heads else latent
    rew_logits = dense_stack(wm, "reward_model._model.", head_in, n_hid, eps, True)
    reward_loss = -twohot_log_prob(rew_logits, rewards)
    cont_logit = dense_stack(wm, "continue_model._model.", head_in, n_hid, eps, True)
    continue_loss = w.continue_scale_factor * F.binary_cross_entropy_with_logits(
        cont_logit, cont_target, reduction="none").sum(-1)
    kl = categorical_kl(post_l.detach(), prior_l, S, D)
    dyn = w.kl_dynamic * torch.clamp(kl, min=w.kl_free_nats)
    rep = w.kl_representation * torch.clamp(categorical_kl(post_l, prior_l.detach(), S, D), min=w.kl_free_nats)
    kl_loss = dyn + rep
    rec_loss = (w.kl_regularizer * kl_loss + obs_loss + reward_loss + continue_loss).mean()
    rec_loss.backward()
    for v in wm.values():
        if v.grad is None:
            v.grad = torch.zeros_like(v)                         # buffers: no gradient, Adam leaves them untouched
    with torch.no_grad():
        wm_norm = clip_grad_norm([v.grad for v in wm.values()], w.clip_gradients)
        if keep:
            out["grads/wm"] = {k: v.grad.clone() for k, v in wm.items()}
        opt_wm.step(wm, {k: v.grad for k, v in wm.items()})
    out.update({
        "Loss/world_model_loss": rec_loss.detach(), "Loss/observation_loss": obs_loss.mean().detach(),
        "Loss/reward_loss": reward_loss.mean().detach(), "Loss/state_loss": kl_loss.mean().detach(),
        "Loss/continue_loss": continue_loss.mean().detach(), "State/kl": kl.mean().detach(),
        "State/post_entropy": categorical_entropy(post_l.detach(), S, D).mean(),
        "State/prior_entropy": categorical_entropy(prior_l.detach(), S, D).mean(),
        "Grads/world_model": wm_norm,
    })
    if keep:
        out.update({"emb": emb.detach(), "latent": latent.detach(), "post_logits": post_l.detach(),
                    "prior_logits": prior_l.detach(), "recon": None if recon is None else recon.detach(),
                    "reward_logits": rew_logits.detach(), "continue_logit": cont_logit.detach()})

    return zs, hs, cont_target


def dv3_train_step(
    cfg,
    wm: Dict[str, Tensor],
    actor: Dict[str, Tensor],
    critic: Dict[str, Tensor],
    target_critic: Dict[str, Tensor],
    opt_wm: AdamState,
    opt_actor: AdamState,
    opt_critic: AdamState,
    data: Dict[str, Tensor],
    noise: Dict[str, Tensor],
    moments_state: Dict[str, Tensor],
    actions_dim: Sequence[int],
    condition_margin: float = 0.0,
    keep: bool = False,
    is_continuous: bool = False,
) -> Dict[str, Tensor]:
    """One Dreamer-V3 update (discrete actions, or continuous `scaled_normal` actions with is_continuous=True: the
    policy gradient then flows through the imagined rollout, dreamer_v3.py:283-284).  Mutates the parameter dicts, optimiser states and
    `moments_state` ("low","high") in place like the reference mutates its modules; returns the 13
    metrics of dreamer_v3.py:330-352 plus (keep=True) the intermediates named in SURVEY.md §8a."""
    a = cfg.algo
    w = a.world_model
    T, B = a.per_rank_sequence_length, a.per_rank_batch_size
    S, D = w.stochastic_size, w.discrete_size
    Z, R = S * D, w.recurrent_model.recurrent_state_size
    H = a.horizon
    N = T * B
    eps = a.mlp_layer_norm.kw.eps
    um = a.unimix
    n_hid = a.mlp_layers
    out: Dict[str, Tensor] = {}

    for d in (wm, actor, critic):
        for v in d.values():
            v.requires_grad_(True)
            v.grad = None

    zs, hs, cont_target = world_model_phase(cfg, wm, opt_wm, data, noise, condition_margin, keep, out)

    # ---- imagination with the UPDATED world model (dreamer_v3.py:203-241); discrete actions: the policy
    # loss does not back-propagate through the rollout (SURVEY.md App. E), so it runs without grad.
    with torch.set_grad_enabled(is_continuous):
        # world model / critic act as constants here (their gradients from the policy loss are discarded by the reference)
        wm_c = {k: v.detach() for k, v in wm.items()}
        critic_c = {k: v.detach() for k, v in critic.items()}
        zi = zs.detach().reshape(N, Z)
        hi = hs.detach().reshape(N, R)
        traj = [torch.cat((zi, hi), -1)]
        acts = []

        ents = []

        def act_sample(state, i):
            if is_continuous:      # the actor always sees a detached state (dreamer_v3.py:219,240)
                hdn = dense_stack(actor, "model._model.", state.detach(), n_hid, eps, False)
                head = F.linear(hdn, actor["mlp_heads.0.weight"], actor["mlp_heads.0.bias"])
                act, ent = continuous_action(head, noise["img_action"][0][i], a.actor)
                ents.append(ent)
                return act
            ls = actor_logits(actor, state, n_hid, actions_dim, um, eps)
            return torch.cat([st_sample(l, 1, ad, noise["img_action"][k][i], condition_margin)
                              for k, (l, ad) in enumerate(zip(ls, actions_dim))], -1)

        acts.append(act_sample(traj[0], 0))
        for i in range(1, H + 1):
            hi = recurrent_step(wm_c, zi, acts[-1], hi, eps)
            zi = st_sample(transition_logits(wm_c, hi, S, D, um, eps), S, D, noise["img_state"][i - 1],
                           condition_margin)
            traj.append(torch.cat((zi, hi), -1))
            acts.append(act_sample(traj[-1], i))
        traj = torch.stack(traj)          # [H+1, N, L]
        acts = torch.stack(acts)          # [H+1, N, sum(A)]

        # ---- dreamer_v3.py:244-260
        values = twohot_mean(dense_stack(critic_c, "_model.", traj, n_hid, eps, True))
        rew = twohot_mean(dense_stack(wm_c, "reward_model._model.", traj, n_hid, eps, True))
        cont = (torch.sigmoid(dense_stack(wm_c, "continue_model._model.", traj, n_hid, eps, True)) > 0.5).float()
        cont = torch.cat((cont_target.reshape(1, N, 1), cont[1:]), 0)
        # compute_lambda_values (dreamer_v3/utils.py:66-77)
        c = cont[1:] * a.gamma
        interm = rew[1:] + c * values[1:] * (1 - a.lmbda)
        nxt = values[-1]
        lam = []
        for t in reversed(range(H)):
            nxt = interm[t] + c[t] * a.lmbda * nxt
            lam.append(nxt)
        lam = torch.stack(list(reversed(lam)))                       # [H, N, 1]
        discount = torch.cumprod(cont * a.gamma, 0) / a.gamma        # [H+1, N, 1]

        # ---- Moments (dreamer_v3/utils.py:56-63)
        mo = a.actor.moments
        lo = torch.quantile(lam.detach().flatten(), mo.percentile.low)
        hi_q = torch.quantile(lam.detach().flatten(), mo.percentile.high)
        moments_state["low"] = mo.decay * moments_state["low"] + (1 - mo.decay) * lo
        moments_state["high"] = mo.decay * moments_state["high"] + (1 - mo.decay) * hi_q
        invscale = torch.maximum(torch.tensor(1.0 / mo.max, device=lam.device), moments_state["high"] - moments_state["low"])
        offset = moments_state["low"]
        advantage = (lam - offset) / invscale - (values[:-1] - offset) / invscale

    # ---- actor loss (dreamer_v3.py:272-304)
    if is_continuous:
        # objective = advantage, differentiated through lambda-values AND the baseline into the rollout; the entropy
        # comes from the reference's second actor evaluation on the detached trajectory, numerically the same heads
        objective = advantage
        ent = torch.stack(ents)                                          # [H+1, N]
    else:
        ls = actor_logits(actor, traj, n_hid, actions_dim, um, eps)
        logp = 0.0
        ent = 0.0
        for l, av in zip(ls, torch.split(acts, list(actions_dim), -1)):
            lg, pr = categorical_normalise(l)
            logp = logp + lg.gather(-1, av.argmax(-1, keepdim=True))     # [H+1,N,1]
            ent = ent + (-(torch.clamp(lg, min=torch.finfo(lg.dtype).min) * pr).sum(-1))
        objective = logp[:-1] * advantage
    entropy = a.actor.ent_coef * ent
    policy_loss = -torch.mean(discount[:-1].detach() * (objective + entropy.unsqueeze(-1)[:-1]))
    policy_loss.backward()
    with torch.no_grad():
        actor_norm = clip_grad_norm([v.grad for v in actor.values()], a.actor.clip_gradients)
        if keep:
            out["grads/actor"] = {k: v.grad.clone() for k, v in actor.items()}
        opt_actor.step(actor, {k: v.grad for k, v in actor.items()})

    # ---- critic loss (dreamer_v3.py:307-327)
    traj, lam, acts = traj.detach(), lam.detach(), acts.detach()
    values, rew, discount, advantage = values.detach(), rew.detach(), discount.detach(), advantage.detach()
    qv_logits = dense_stack(critic, "_model.", traj[:-1], n_hid, eps, True)
    with torch.no_grad():
        tgt_vals = twohot_mean(dense_stack(target_critic, "_model.", traj[:-1], n_hid, eps, True))
    value_loss = -twohot_log_prob(qv_logits, lam) - twohot_log_prob(qv_logits, tgt_vals)
    value_loss = torch.mean(value_loss * discount[:-1].squeeze(-1))
    value_loss.backward()
    with torch.no_grad():
        critic_norm = clip_grad_norm([v.grad for v in critic.values()], a.critic.clip_gradients)
        if keep:
            out["grads/critic"] = {k: v.grad.clone() for k, v in critic.items()}
        opt_critic.step(critic, {k: v.grad for k, v in critic.items()})

    out.update({"Loss/policy_loss": policy_loss.detach(), "Loss/value_loss": value_loss.detach(),
                "Grads/actor": actor_norm, "Grads/critic": critic_norm})
    if keep:
        out.update({"traj": traj, "imagined_actions": acts, "values": values, "lambda_values": lam,
                    "discount": discount, "advantage": advantage, "pred_rewards": rew, "continues": cont})
    for d in (wm, actor, critic):
        for v in d.values():
            v.grad = None
            v.requires_grad_(False)
    return out


# --------------------------------------------------------------------------------------------------
# parameter construction (oracle-side init: statistically the reference's, not bit-identical;
# pinned runs copy the reference's own state_dict instead)
# --------------------------------------------------------------------------------------------------
def _trunc_normal(shape, fan_in, fan_out, g, limit_in_std=True):
    std = math.sqrt(1.0 / ((fan_in + fan_out) / 2.0)) / 0.87962566103423978
    t = torch.empty(*shape)
    lim = 2.0 * std if limit_in_std else 2.0
    torch.nn.init.trunc_normal_(t, 0.0, std, -lim, lim, generator=g)
    return t


def _uniform(shape, fan_in, fan_out, scale, g):
    if scale == 0.0:
        return torch.zeros(*shape)
    lim = math.sqrt(3 * scale / ((fan_in + fan_out) / 2.0))
    return (torch.rand(*shape, generator=g) * 2 - 1) * lim


def init_params(cfg, actions_dim: Sequence[int], in_channels: int = 3, seed: int = 0, is_continuous: bool = False):
    """Parameter dicts with the reference's state-dict keys/shapes (SURVEY.md §8b) and the reference's
    initialisation distributions (dreamer_v3/utils.py:143-186, agent.py:1170-1180)."""
    g = torch.Generator().manual_seed(seed)
    a, w = cfg.algo, cfg.algo.world_model
    S, D = w.stochastic_size, w.discrete_size
    Z, R = S * D, w.recurrent_model.recurrent_state_size
    L = Z + R
    du, nh = a.dense_units, a.mlp_layers
    mult = w.encoder.cnn_channels_multiplier
    stages = int(round(math.log2(cfg.env.screen_size) - 2))
    A = int(sum(actions_dim))
    wm: Dict[str, Tensor] = {}

    def lin(d, name, o, i, bias, uni=None):
        d[name + ".weight"] = _trunc_normal((o, i), i, o, g) if uni is None else _uniform((o, i), i, o, uni, g)
        if bias:
            d[name + ".bias"] = torch.zeros(o)

    def ln(d, name, n):
        d[name + ".weight"] = torch.ones(n)
        d[name + ".bias"] = torch.zeros(n)

    def mlp(d, prefix, i, hidden, n_hidden, o, uni):
        for k in range(n_hidden):
            lin(d, f"{prefix}{3 * k}", hidden, i if k == 0 else hidden, False)
            ln(d, f"{prefix}{3 * k + 1}", hidden)
        if o is not None:
            lin(d, f"{prefix}{3 * n_hidden}", o, hidden, True, uni)

    has_cnn, vd = len(a.cnn_keys.encoder) > 0, vec_dims(cfg)
    vkeys = list(a.mlp_keys.encoder)
    chans = [in_channels] + [mult * 2 ** i for i in range(stages)]
    E = 0
    if has_cnn:
        for i in range(stages):
            ci, co = chans[i], chans[i + 1]
            wm[f"encoder.cnn_encoder.model.0._model.{3 * i}.weight"] = _trunc_normal((co, ci, 4, 4), 16 * ci, 16 * co, g, False)
            ln(wm, f"encoder.cnn_encoder.model.0._model.{3 * i + 1}", co)
        E = chans[-1] * 16
    if vkeys:
        mlp(wm, "encoder.mlp_encoder.model._model.", sum(vd[k] for k in vkeys), w.encoder.dense_units, w.encoder.mlp_layers, None, None)
        E += w.encoder.dense_units
    wm["rssm.initial_recurrent_state"] = torch.zeros(R)
    lin(wm, "rssm.recurrent_model.mlp._model.0", w.recurrent_model.dense_units, Z + A, False)
    ln(wm, "rssm.recurrent_model.mlp._model.1", w.recurrent_model.dense_units)
    lin(wm, "rssm.recurrent_model.rnn.linear", 3 * R, R + w.recurrent_model.dense_units, False)
    ln(wm, "rssm.recurrent_model.rnn.layer_norm", 3 * R)
    mlp(wm, "rssm.representation_model._model.", R + E, w.representation_model.hidden_size, 1, Z, 1.0)
    mlp(wm, "rssm.transition_model._model.", R, w.transition_model.hidden_size, 1, Z, 1.0)
    dch = [chans[-1]] + [mult * 2 ** i for i in reversed(range(stages - 1))] + [in_channels]
    if has_cnn:
        lin(wm, "observation_model.cnn_decoder.model.0", chans[-1] * 16, L, True)
    for i in range(stages if has_cnn else 0):
        ci, co = dch[i], dch[i + 1]
        last = i == stages - 1
        name = f"observation_model.cnn_decoder.model.2._model.{3 * i}"
        wm[name + ".weight"] = _trunc_normal((ci, co, 4, 4), 16 * ci, 16 * co, g, False)
        if last:
            wm[name + ".bias"] = torch.zeros(co)
        else:
            ln(wm, f"observation_model.cnn_decoder.model.2._model.{3 * i + 1}", co)
    if a.mlp_keys.decoder:
        om = w.observation_model
        mlp(wm, "observation_model.mlp_decoder.model._model.", L, om.dense_units, om.mlp_layers, None, None)
        for i, k in enumerate(a.mlp_keys.decoder):
            lin(wm, f"observation_model.mlp_decoder.heads.{i}", vd[k], om.dense_units, True, 1.0)
    mlp(wm, "reward_model._model.", L, du, nh, w.reward_model.bins, 0.0)
    mlp(wm, "continue_model._model.", L, du, nh, 1, 1.0)
    actor: Dict[str, Tensor] = {}
    mlp(actor, "model._model.", L, du, nh, None, None)
    if is_continuous:
        lin(actor, "mlp_heads.0", 2 * A, du, True, 1.0)
    else:
        for i, ad in enumerate(actions_dim):
            lin(actor, f"mlp_heads.{i}", ad, du, True, 1.0)
    critic: Dict[str, Tensor] = {}
    mlp(critic, "_model.", L, du, nh, a.critic.bins, 0.0)
    target = {k: v.clone() for k, v in critic.items()}
    return wm, actor, critic, target


def make_batch(cfg, actions_dim: Sequence[int], seed: int = 1, in_channels: int = 3,
               as_uint8: bool = False, is_continuous: bool = False) -> Dict[str, Tensor]:
    """Synthetic replay batch of SURVEY.md §8d: uniform uint8 pixels, one-hot actions, N(0,1) rewards,
    Bernoulli(0.01) terminated, Bernoulli(0.02) is_first."""
    g = torch.Generator().manual_seed(seed)
    T, B = cfg.algo.per_rank_sequence_length, cfg.algo.per_rank_batch_size
    sz = cfg.env.screen_size
    cch = dict(cfg.env.get("cnn_channels", {}) or {})
    first = cfg.algo.cnn_keys.encoder[0] if cfg.algo.cnn_keys.encoder else None
    rgb = torch.randint(0, 256, (T, B, cch.get(first, in_channels) if len(cch) > 1 else in_channels, sz, sz), generator=g,
                        dtype=torch.uint8)
    acts = []
    for ad in actions_dim:
        if is_continuous:
            acts.append(torch.rand(T, B, ad, generator=g) * 2 - 1)
        else:
            idx = torch.randint(0, ad, (T, B), generator=g)
            acts.append(F.one_hot(idx, ad).float())
    obs = {cfg.algo.cnn_keys.encoder[0]: rgb if as_uint8 else rgb.float()} if cfg.algo.cnn_keys.encoder else {}
    out = {
        **obs,
        "actions": torch.cat(acts, -1),
        "rewards": torch.randn(T, B, 1, generator=g),
        "terminated": (torch.rand(T, B, 1, generator=g) < 0.01).float(),
        "truncated": torch.zeros(T, B, 1),
        "is_first": (torch.rand(T, B, 1, generator=g) < 0.02).float(),
    }
    for k, d in vec_dims(cfg).items():               # vector observations, heavy-tailed enough to exercise symlog
        out[k] = torch.randn(T, B, d, generator=g) * 3.0
    for k in list(cfg.algo.cnn_keys.encoder)[1:]:    # further image keys (drawn last: older fixtures keep their streams)
        img = torch.randint(0, 256, (T, B, cch[k], sz, sz), generator=g, dtype=torch.uint8)
        out[k] = img if as_uint8 else img.float()
    return out
