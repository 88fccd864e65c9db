"""TEST INFRASTRUCTURE (oracle) — functional fp32 torch restatement of the recurrent PPO update.

Reference: `train` sheeprl/algos/ppo_recurrent/ppo_recurrent.py:31-116, RecurrentPPOAgent / RecurrentModel
ppo_recurrent/agent.py:18-262, losses ppo/loss.py.  Parity PINNED: tests/golden/ppo_rec_*.pt come from the executed
reference `train()` (oracle/make_golden_ppo_recurrent.py), run with torch's distribution argument validation off.

spec = the PPO oracle spec (ppo_oracle.ppo_param_shapes) plus rnn = dict(hidden=H, pre=None | (dense, layer_norm),
post=None | (dense, layer_norm)); discrete actions only.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

from oracle import ppo_oracle as PO
from oracle.dv3_oracle import AdamState  # noqa: F401

RNN_LN_EPS = 1e-3


def param_shapes(spec) -> "Dict[str, tuple]":
    base = PO.ppo_param_shapes(spec)
    out = {k: v for k, v in base.items() if k.startswith("feature_extractor.")}
    feat = (spec["cnn_features"] if spec["cnn_channels"] else 0) + (spec["mlp_features"] if spec["mlp_dim"] else 0)
    d_in = feat + sum(spec["actions_dim"])
    r = spec["rnn"]
    H = r["hidden"]
    if r.get("pre"):
        dense, ln = r["pre"]
        out["rnn._pre_mlp._model.0.weight"], out["rnn._pre_mlp._model.0.bias"] = (dense, d_in), (dense,)
        if ln:
            out["rnn._pre_mlp._model.1.weight"], out["rnn._pre_mlp._model.1.bias"] = (dense,), (dense,)
        d_in = dense
    out["rnn._lstm.weight_ih_l0"], out["rnn._lstm.weight_hh_l0"] = (4 * H, d_in), (4 * H, H)
    out["rnn._lstm.bias_ih_l0"], out["rnn._lstm.bias_hh_l0"] = (4 * H,), (4 * H,)
    if r.get("post"):
        dense, ln = r["post"]
        out["rnn._post_mlp._model.0.weight"], out["rnn._post_mlp._model.0.bias"] = (dense, H), (dense,)
        if ln:
            out["rnn._post_mlp._model.1.weight"], out["rnn._post_mlp._model.1.bias"] = (dense,), (dense,)
    for k, v in base.items():
        if k.startswith(("critic.", "actor.")):
            out[k] = (v[0], H) if k.endswith("._model.0.weight") else v
    return out


def _dense(p, prefix, x, cfg, act):
    dense, ln = cfg
    x = F.linear(x, p[f"{prefix}._model.0.weight"], p[f"{prefix}._model.0.bias"])
    if ln:
        x = F.layer_norm(x, (dense,), p[f"{prefix}._model.1.weight"], p[f"{prefix}._model.1.bias"], RNN_LN_EPS)
    return act(x)


def features(p, spec, obs):
    act = torch.tanh if spec.get("act", "tanh") == "tanh" else torch.relu
    feats = []
    if spec["cnn_channels"]:
        x = obs["rgb"]
        for i, (k, st) in enumerate(PO.CONVS):
            pre = f"feature_extractor.cnn_encoder.model._model.{2 * i}"
            x = torch.relu(F.conv2d(x, p[f"{pre}.weight"], p[f"{pre}.bias"], stride=st))
        feats.append(torch.relu(F.linear(x.flatten(1), p["feature_extractor.cnn_encoder.model.fc.weight"],
                                         p["feature_extractor.cnn_encoder.model.fc.bias"])))
    if spec["mlp_dim"]:
        feats.append(PO._mlp(p, "feature_extractor.mlp_encoder.model", obs["state"], PO.net_cfg(spec, "encoder"), act))
    return torch.cat(feats, -1)


def lstm(p, x, h, c, lengths):
    """x [T, B, D]; (h, c) [B, H]; packed-sequence semantics: out 0 and state kept for t >= lengths[b]."""
    H = h.shape[-1]
    outs = []
    for t in range(x.shape[0]):
        z = F.linear(x[t], p["rnn._lstm.weight_ih_l0"], p["rnn._lstm.bias_ih_l0"]) + \
            F.linear(h, p["rnn._lstm.weight_hh_l0"], p["rnn._lstm.bias_hh_l0"])
        i, f, g, o = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.tanh(z[:, 2 * H:3 * H]), torch.sigmoid(z[:, 3 * H:])
        cn = f * c + i * g
        hn = o * torch.tanh(cn)
        valid = (t < lengths).unsqueeze(-1)
        c, h = torch.where(valid, cn, c), torch.where(valid, hn, h)
        outs.append(torch.where(valid, hn, torch.zeros_like(hn)))
    return torch.stack(outs), (h, c)


def forward(p, spec, obs, prev_actions, h0, c0, lengths):
    """RecurrentPPOAgent.forward up to the heads: (list of logits per head, values), each [T, B, *].  obs values
    [T, B, ...] (images already normalised)."""
    T, B = prev_actions.shape[:2]
    act = torch.tanh if spec.get("act", "tanh") == "tanh" else torch.relu
    flat = {k: v.reshape(T * B, *v.shape[2:]) for k, v in obs.items()}
    x = torch.cat((features(p, spec, flat), prev_actions.reshape(T * B, -1)), -1)
    r = spec["rnn"]
    if r.get("pre"):
        x = _dense(p, "rnn._pre_mlp", x, r["pre"], act)
    out, _ = lstm(p, x.reshape(T, B, -1), h0, c0, lengths)
    y = out.reshape(T * B, -1)
    if r.get("post"):
        y = _dense(p, "rnn._post_mlp", y, r["post"], act)
    values = PO._mlp(p, "critic", y, PO.net_cfg(spec, "critic"), act)
    h = PO._mlp(p, "actor.actor_backbone", y, PO.net_cfg(spec, "actor"), act, last=False)
    logits = [F.linear(h, p[f"actor.actor_heads.{i}.weight"], p[f"actor.actor_heads.{i}.bias"]).reshape(T, B, -1)
              for i in range(len(spec["actions_dim"]))]
    return logits, values.reshape(T, B, 1)


def masked_losses(logits, values, batch, spec, hp):
    mask = batch["mask"]
    lps, ents, off = [], [], 0
    for lg, a in zip(logits, spec["actions_dim"]):
        logp = lg - lg.logsumexp(-1, keepdim=True)
        lps.append((logp * batch["actions"][..., off:off + a]).sum(-1))
        ents.append(-(torch.clamp(logp, min=torch.finfo(logp.dtype).min) * logp.exp()).sum(-1))
        off += a
    lp, ent = torch.stack(lps, -1).sum(-1)[mask], torch.stack(ents, -1).sum(-1)[mask]
    adv = batch["advantages"][..., 0][mask]
    if hp["normalize_advantages"] and adv.numel() > 1:
        adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    ratio = (lp - batch["logprobs"][..., 0][mask]).exp()
    pg = -torch.min(adv * ratio, adv * torch.clamp(ratio, 1 - hp["clip_coef"], 1 + hp["clip_coef"])).mean()
    v, old, ret = values[..., 0][mask], batch["values"][..., 0][mask], batch["returns"][..., 0][mask]
    if hp["clip_vloss"]:
        vc = old + torch.clamp(v - old, -hp["clip_coef"], hp["clip_coef"])
        vl = 0.5 * torch.max((v - ret) ** 2, (vc - ret) ** 2).mean()
    else:
        vl = ((v - ret) ** 2).mean()
    return pg, vl, (-ent).mean()


def train(p: Dict[str, torch.Tensor], opt: "AdamState", spec, data: Dict[str, torch.Tensor],
          index_batches: Sequence[Sequence[int]], hp) -> List[Dict[str, float]]:
    """`train()` over the given lists of sequence indices.  data: [T, S, ...] (rgb raw 0..255 as float).  Mutates p."""
    logs = []
    for idx in index_batches:
        idx = torch.as_tensor(idx)
        batch = {k: v[:, idx] for k, v in data.items()}
        obs = {}
        if spec["cnn_channels"]:
            obs["rgb"] = batch["rgb"] / 255 - 0.5
        if spec["mlp_dim"]:
            obs["state"] = batch["state"]
        lengths = batch["mask"].sum(0)
        q = {k: v.detach().requires_grad_(True) for k, v in p.items()}
        logits, values = forward(q, spec, obs, batch["prev_actions"], batch["prev_hx"][0], batch["prev_cx"][0], lengths)
        pg, v, e = masked_losses(logits, values, batch, spec, hp)
        loss = pg + hp["vf_coef"] * v + hp["ent_coef"] * e
        grads = dict(zip(q.keys(), torch.autograd.grad(loss, list(q.values()))))
        if hp["max_grad_norm"] > 0:
            total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
            coef = torch.clamp(hp["max_grad_norm"] / (total + 1e-6), max=1.0)
            grads = {k: g * coef for k, g in grads.items()}
        opt.step(p, grads)
        logs.append({"Loss/policy_loss": float(pg.detach()), "Loss/value_loss": float(v.detach()),
                     "Loss/entropy_loss": float(e.detach())})
    return logs


def make_rollout(spec, T: int, lengths: Sequence[int], seed: int) -> Dict[str, torch.Tensor]:
    """Synthetic padded rollout [T, S, ...] as the reference's main builds it (pad_sequence with 0 after each
    sequence's length, ppo_recurrent.py:438-444)."""
    g = torch.Generator().manual_seed(seed)
    S, H, A = len(lengths), spec["rnn"]["hidden"], sum(spec["actions_dim"])
    mask = torch.arange(T).unsqueeze(1) < torch.as_tensor(lengths).unsqueeze(0)
    d = {}
    if spec["cnn_channels"]:
        d["rgb"] = torch.randint(0, 256, (T, S, spec["cnn_channels"], spec["screen"], spec["screen"]), generator=g).float()
    if spec["mlp_dim"]:
        d["state"] = torch.randn(T, S, spec["mlp_dim"], generator=g)
    onehot = lambda: torch.cat([F.one_hot(torch.randint(0, a, (T, S), generator=g), a).float()  # noqa: E731
                                for a in spec["actions_dim"]], -1)
    d["actions"], d["prev_actions"] = onehot(), onehot()
    d["prev_actions"][0, : S // 2] = 0                      # sequences that start an episode see no previous action
    d["logprobs"] = -torch.rand(T, S, 1, generator=g) * 2
    d["values"] = torch.randn(T, S, 1, generator=g)
    d["returns"] = d["values"] + torch.randn(T, S, 1, generator=g) * 0.5
    d["advantages"] = torch.randn(T, S, 1, generator=g)
    d["prev_hx"] = torch.randn(T, S, H, generator=g) * 0.3
    d["prev_cx"] = torch.randn(T, S, H, generator=g) * 0.3
    for k, v in d.items():
        v[~mask] = 0
    d["mask"] = mask
    return d


def init_params(spec, seed: int) -> Dict[str, torch.Tensor]:
    """Deterministic initial parameters for the fixtures (CPU torch.Generator draws, identical on every host), so the
    fixtures store a seed instead of the tensors: weights and biases U(-1/sqrt(fan_in), 1/sqrt(fan_in)), LayerNorm
    weights 1 + N(0, 0.1), LayerNorm biases N(0, 0.1) (away from 1 / 0 so their gradients are exercised)."""
    g = torch.Generator().manual_seed(seed)
    out, shapes = {}, param_shapes(spec)
    ln = {k for k, s in shapes.items() if k.endswith(".weight") and len(s) == 1}
    ln |= {k[:-6] + "bias" for k in ln}
    fan = 1
    for k, s in shapes.items():
        if k in ln:
            base = 1.0 if k.endswith(".weight") else 0.0
            out[k] = base + 0.1 * torch.randn(*s, generator=g)
            continue
        if k.endswith(".weight") or k.startswith("rnn._lstm.weight"):
            fan = 1
            for d in s[1:]:
                fan *= d
        out[k] = (torch.rand(*s, generator=g) * 2 - 1) / fan ** 0.5
    return out


def pack_after(init: Dict[str, torch.Tensor], after: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """What a fixture stores of the parameters after train(): the update `after - init` in fp16.  An Adam update of a
    few steps is at most a few times lr, so the fp16 rounding of it (2^-11 relative) is ~1e-6 absolute, far inside the
    parameter tolerance (2e-5 + 1e-4 relative)."""
    return {k: (after[k] - init[k]).half() for k in init}


def unpack_after(init: Dict[str, torch.Tensor], delta: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    return {k: init[k] + delta[k].float() for k in init}


def player_obs(raw: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The observation dict the reference's rollout loop hands the player (ppo_recurrent/utils.py:27-39): images as
    float x/255 - 0.5, vectors as they are."""
    return {k: (v.float() / 255 - 0.5 if k == "rgb" else v) for k, v in raw.items()}
