"""TEST INFRASTRUCTURE (oracle) — NOT part of the product path.

The Dreamer-V3 oracle (`oracle/dv3_oracle.py`) with decoders over a subset of the encoded keys
(`cnn_keys.decoder` / `mlp_keys.decoder`, in their own order).  The reference's train() builds the reconstruction
targets from the decoder keys (dreamer_v3.py:148-160): the CNN decoder's output is split per decoder key on the channel
axis (agent.py:226) and each key contributes an MSE sum, the MLP decoder has one head per decoder key with a symlog MSE
sum, and either decoder may be missing.  Only the reconstruction part of `world_model_phase` depends on those keys, so
`world_model_phase` below is the coupled oracle's with that part rewritten; `decoder_keys()` installs it in the
Dreamer-V3 and Plan2Explore oracles for the duration of a `with` block.  With decoder keys equal to the encoder's it
computes the same thing as the original.
"""
from __future__ import annotations

import contextlib
import math
from typing import Dict

import torch
import torch.nn.functional as F

from oracle import dv3_oracle as O

Tensor = O.Tensor


def world_model_phase(cfg, wm: Dict[str, Tensor], opt_wm: "O.AdamState", data: Dict[str, Tensor], noise: Dict[str, Tensor],
                      condition_margin: float, keep: bool, out: Dict[str, Tensor], detach_heads: bool = False):
    """`O.world_model_phase` with the reconstruction terms over the decoder keys"""
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
    cnn_dec, vec_dec = list(a.cnn_keys.decoder or []), list(a.mlp_keys.decoder or [])
    n_hid = a.mlp_layers

    # ---- dreamer_v3.py:98-104: every image key normalised; the encoder sees them concatenated in encoder order
    pix = {k: data[k].float() / 255.0 - 0.5 for k in cnn_keys}
    obs = torch.cat([pix[k] for k in cnn_keys], -3) if cnn_keys else None
    is_first = data["is_first"].float().clone()
    is_first[0] = 1.0
    actions = torch.cat((torch.zeros_like(data["actions"][:1]), data["actions"][:-1]), 0).float()
    rewards = data["rewards"].float()
    cont_target = 1 - data["terminated"].float()

    embs = []
    if cnn_keys:
        embs.append(O.encoder_forward(wm, obs, stages, ceps))
    if vkeys:
        vemb, _ = O.mlp_encoder_forward(wm, data, vkeys, w.encoder.mlp_layers, w.encoder.mlp_layer_norm.kw.eps)
        embs.append(vemb)
    emb = torch.cat(embs, -1)
    h = torch.zeros(B, R, device=emb.device)
    z = torch.zeros(B, Z, device=emb.device)
    hs, zs, post_l, prior_l = [], [], [], []
    h0_raw = wm["rssm.initial_recurrent_state"]
    if not w.get("learnable_initial_recurrent_state", True):
        h0_raw = h0_raw.detach()
    h0 = torch.tanh(h0_raw).expand(B, R)
    for t in range(T):
        f = is_first[t]
        act = (1 - f) * actions[t]
        z0 = O.st_sample(O.transition_logits(wm, h0, S, D, um, eps), S, D, None)
        h = (1 - f) * h + f * h0
        z = (1 - f) * z + f * z0
        h = O.recurrent_step(wm, z, act, h, eps)
        pl = O.transition_logits(wm, h, S, D, um, eps)
        ql = O.representation_logits(wm, h, emb[t], S, D, um, eps)
        z = O.st_sample(ql, S, D, noise["post"][t], condition_margin)
        hs.append(h), zs.append(z), post_l.append(ql), prior_l.append(pl)
    hs, zs = torch.stack(hs), torch.stack(zs)
    post_l, prior_l = torch.stack(post_l), torch.stack(prior_l)
    latent = torch.cat((zs, hs), -1)

    # ---- reconstruction over the decoder keys (dreamer_v3.py:148-160, loss.py:61)
    obs_loss, recon = 0.0, None
    if cnn_dec:
        chans = [pix[k].shape[-3] for k in cnn_dec]
        recon = O.decoder_forward(wm, latent, stages, ceps, (sum(chans),) + tuple(pix[cnn_dec[0]].shape[-2:]))
        for k, rk in zip(cnn_dec, torch.split(recon, chans, -3)):
            obs_loss = obs_loss + ((rk - pix[k]) ** 2).sum((-3, -2, -1))
    if vec_dec:
        obs_loss = obs_loss + O.mlp_decoder_loss(wm, latent, [O.symlog(data[k].float()) for k in vec_dec],
                                                 w.observation_model.mlp_layers, w.observation_model.mlp_layer_norm.kw.eps)
    head_in = latent.detach() if detach_heads else latent
    rew_logits = O.dense_stack(wm, "reward_model._model.", head_in, n_hid, eps, True)
    reward_loss = -O.twohot_log_prob(rew_logits, rewards)
    cont_logit = O.dense_stack(wm, "continue_model._model.", head_in, n_hid, eps, True)
    continue_loss = w.continue_scale_factor * F.binary_cross_entropy_with_logits(
        cont_logit, cont_target, reduction="none").sum(-1)
    kl = O.categorical_kl(post_l.detach(), prior_l, S, D)
    dyn = w.kl_dynamic * torch.clamp(kl, min=w.kl_free_nats)
    rep = w.kl_representation * torch.clamp(O.categorical_kl(post_l, prior_l.detach(), S, D), min=w.kl_free_nats)
    kl_loss = dyn + rep
    rec_loss = (w.kl_regularizer * kl_loss + obs_loss + reward_loss + continue_loss).mean()
    rec_loss.backward()
    for v in wm.values():
        if v.grad is None:
            v.grad = torch.zeros_like(v)
    with torch.no_grad():
        wm_norm = O.clip_grad_norm([v.grad for v in wm.values()], w.clip_gradients)
        if keep:
            out["grads/wm"] = {k: v.grad.clone() for k, v in wm.items()}
        opt_wm.step(wm, {k: v.grad for k, v in wm.items()})
    out.update({
        "Loss/world_model_loss": rec_loss.detach(), "Loss/observation_loss": obs_loss.mean().detach(),
        "Loss/reward_loss": reward_loss.mean().detach(), "Loss/state_loss": kl_loss.mean().detach(),
        "Loss/continue_loss": continue_loss.mean().detach(), "State/kl": kl.mean().detach(),
        "State/post_entropy": O.categorical_entropy(post_l.detach(), S, D).mean(),
        "State/prior_entropy": O.categorical_entropy(prior_l.detach(), S, D).mean(),
        "Grads/world_model": wm_norm,
    })
    if keep:
        out.update({"emb": emb.detach(), "latent": latent.detach(), "post_logits": post_l.detach(),
                    "prior_logits": prior_l.detach(), "recon": None if recon is None else recon.detach(),
                    "reward_logits": rew_logits.detach(), "continue_logit": cont_logit.detach()})
    return zs, hs, cont_target


@contextlib.contextmanager
def decoder_keys():
    """inside the block the Dreamer-V3 and Plan2Explore oracles reconstruct the decoder keys"""
    from oracle import p2e_continuous_oracle, p2e_oracle

    mods = (O, p2e_oracle, p2e_continuous_oracle)
    orig = [m.world_model_phase for m in mods]
    for m in mods:
        m.world_model_phase = world_model_phase
    try:
        yield
    finally:
        for m, f in zip(mods, orig):
            m.world_model_phase = f
