"""Kernel schedule of the PPO update (SURVEY §8 a19): per minibatch one row gather, the NatureCNN / MLP forward, the
fused PPO objective, a hand-derived backward and a fused clip+Adam — ~70 launches on one stream, no autograd.

Reference being replaced: `train` sheeprl/algos/ppo/ppo.py:30-102, `PPOAgent.forward` ppo/agent.py:208-239, NatureCNN
models/models.py:288-328, losses ppo/loss.py.  `ops` is `sheeprl_b200.lib.CudaOps` in production (tests on a GPU-less
host pass the torch test double `oracle/ops_emul.py::EmulOps`).

Layout decisions:
  * ONE flat parameter group (the reference has a single optimiser over the whole agent): one norm pass, one Adam
    launch, one all-reduce per minibatch;
  * activations are channel-last; conv weights live in the group as [Cout, k, k, Cin] and the fc weight as
    [F, Ho, Wo, C] (the layouts the patch-matrix products want), so nothing is re-packed per step — only
    `state_dict()` / `load_state_dict()` permute to the reference's [Cout, Cin, k, k] / [F, C*Ho*Wo];
  * all action heads are one stacked Linear; the encoders write straight into their column range of the feature
    buffer (no torch.cat), and the feature gradient is accumulated in place by the actor and critic backward.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional, Sequence

import torch

from sheeprl_b200.dense import Act, LayerNormAct, Linear, Stack
from sheeprl_b200.lib import sync_deterministic
from sheeprl_b200.params import FlatGroup

CONVS = ((8, 4, 32), (4, 2, 64), (3, 1, 64))        # NatureCNN (kernel, stride, channels) models.py:301-309
LN_EPS = 1e-5                                        # nn.LayerNorm default (ppo/agent.py:63-64 passes only the shape)
DIST_MODE = {"discrete": 0, "normal": 1, "tanh_normal": 2}


def net_cfg(spec: dict, which: str):
    """(dense_units, mlp_layers, layer_norm) of the "encoder" / "actor" / "critic" MLP: spec["nets"][which] = (dense,
    layers) and spec["layer_norm"] (bool or per-net dict) override the shared spec["dense"] / spec["layers"]."""
    dense, layers = (spec.get("nets") or {}).get(which, (spec["dense"], spec["layers"]))
    ln = spec.get("layer_norm", False)
    ln = bool(ln.get(which, False)) if isinstance(ln, dict) else bool(ln)
    return int(dense), int(layers), ln


class PPOEngine:
    def __init__(self, spec: dict, hp: dict, opt: dict, device, ops, seed: int = 0):
        """spec: cnn_channels (0 = none), screen, mlp_dim (0 = none), dense, layers, cnn_features, mlp_features,
        actions_dim, is_continuous, act ('tanh' | 'relu') [, dist ('normal' | 'tanh_normal'), layer_norm (bool or
        {"encoder"/"actor"/"critic": bool}), nets ({"encoder"/"actor"/"critic": (dense, layers)})].  cnn_channels /
        mlp_dim are the sums over the image / vector keys (the encoders concatenate them, ppo/agent.py:34-36,67-69).  hp: clip_coef, vf_coef, ent_coef, clip_vloss,
        normalize_advantages, max_grad_norm.  opt: lr, eps, betas."""
        self.spec, self.hp, self.opt = dict(spec), dict(hp), dict(opt)
        self.device, self.ops = torch.device(device), ops
        self.allreduce = None
        s = self.spec
        self.act = s.get("act", "tanh")
        self.head_dims = list(s["actions_dim"])
        self.head_width = 2 * sum(self.head_dims) if s["is_continuous"] else sum(self.head_dims)
        self.dist = (s.get("dist") or "normal") if s["is_continuous"] else "discrete"
        if self.dist not in DIST_MODE or (s["is_continuous"] and self.dist == "discrete"):
            raise ValueError(f"distribution must be one of {sorted(DIST_MODE)}, got {self.dist!r}")
        self.dist_mode = DIST_MODE[self.dist]
        self.F = s["cnn_features"] if s["cnn_channels"] else 0
        self.Mf = s["mlp_features"] if s["mlp_dim"] else 0
        self.feat_dim = self.F + self.Mf
        self.geo = []                                    # per conv: (H, W, Cin, k, stride, Ho, Wo, Cout)
        if s["cnn_channels"]:
            h, c = s["screen"], s["cnn_channels"]
            for k, st, co in CONVS:
                ho = (h - k) // st + 1
                self.geo.append((h, h, c, k, st, ho, ho, co))
                h, c = ho, co
        self.group = FlatGroup(self._internal_shapes(), device)
        self._build_layers()
        self._bufs: Dict[int, dict] = {}
        self.normsq = torch.zeros(1, dtype=torch.float64, device=self.device)
        self.norm_out = torch.zeros(1, dtype=torch.float32, device=self.device)
        self.losses = torch.zeros(3, dtype=torch.float32, device=self.device)

    # ------------------------------------------------------------------ parameters
    @property
    def actor_in(self) -> int:
        """width of the actor's and critic's input: the features"""
        return self.feat_dim

    def _internal_shapes(self):
        s, out = self.spec, OrderedDict()
        pre = "feature_extractor.cnn_encoder.model"
        for i, (H, W, C, k, st, Ho, Wo, Co) in enumerate(self.geo):
            out[f"{pre}._model.{2 * i}.weight"] = (Co, k, k, C)
            out[f"{pre}._model.{2 * i}.bias"] = (Co,)
        if self.geo:
            _, _, _, _, _, Ho, Wo, Co = self.geo[-1]
            out[f"{pre}.fc.weight"] = (s["cnn_features"], Ho * Wo * Co)
            out[f"{pre}.fc.bias"] = (s["cnn_features"],)
        def stack(prefix, d, which, last):
            dense, layers, ln = net_cfg(s, which)
            st = 3 if ln else 2
            for i in range(layers):
                out[f"{prefix}._model.{st * i}.weight"] = (dense, d)
                out[f"{prefix}._model.{st * i}.bias"] = (dense,)
                if ln:
                    out[f"{prefix}._model.{st * i + 1}.weight"] = (dense,)
                    out[f"{prefix}._model.{st * i + 1}.bias"] = (dense,)
                d = dense
            if last is not None:
                out[f"{prefix}._model.{st * layers}.weight"] = (last, d)
                out[f"{prefix}._model.{st * layers}.bias"] = (last,)

        if s["mlp_dim"]:
            stack("feature_extractor.mlp_encoder.model", s["mlp_dim"], "encoder", s["mlp_features"])
        stack("critic", self.actor_in, "critic", 1)
        stack("actor.actor_backbone", self.actor_in, "actor", None)
        # every head reads `actor.dense_units` inputs, also with an empty backbone (ppo/agent.py:180-183)
        out["actor.heads.weight"] = (self.head_width, net_cfg(s, "actor")[0])
        out["actor.heads.bias"] = (self.head_width,)
        return out

    def _build_layers(self):
        pre = "feature_extractor.cnn_encoder.model"
        self.convs = [Linear.of(self.group, f"{pre}._model.{2 * i}.weight") for i in range(len(self.geo))]
        self.fc = Linear.of(self.group, f"{pre}.fc.weight") if self.geo else None
        self.menc = self._stack("feature_extractor.mlp_encoder.model", "encoder") if self.spec["mlp_dim"] else None
        self.critic = self._stack("critic", "critic")
        self.actor = self._stack("actor.actor_backbone", "actor", last_key="actor.heads.weight")
        if len(self.actor.layers) == 1 and net_cfg(self.spec, "actor")[0] != self.actor_in:
            raise ValueError(f"actor.mlp_layers == 0 needs actor.dense_units == the actor's input width {self.actor_in} "
                             "(the heads read dense_units inputs)")

    def _stack(self, prefix: str, which: str, last_key: Optional[str] = None) -> Stack:
        """An `MLP` of the reference (models/models.py:17-126): `layers` hidden blocks Linear [-> LayerNorm] -> act, then
        an output Linear without activation (for the actor backbone: the stacked action heads)."""
        _, layers, ln = net_cfg(self.spec, which)
        st = 3 if ln else 2
        out = [(Linear.of(self.group, f"{prefix}._model.{st * i}.weight"),
                LayerNormAct(self.group, f"{prefix}._model.{st * i + 1}", LN_EPS, self.act) if ln else Act(self.act))
               for i in range(layers)]
        return Stack(self.ops, out + [(Linear.of(self.group, last_key or f"{prefix}._model.{st * layers}.weight"), Act("none"))])

    def reference_shapes(self) -> "OrderedDict[str, tuple]":
        out = OrderedDict()
        for k, shp in self.group.shapes.items():
            if len(shp) == 4:
                out[k] = (shp[0], shp[3], shp[1], shp[2])
            elif k == "actor.heads.weight":
                heads = [self.head_width] if self.spec["is_continuous"] else self.head_dims
                for i, a in enumerate(heads):
                    out[f"actor.actor_heads.{i}.weight"] = (a, shp[1])
            elif k == "actor.heads.bias":
                heads = [self.head_width] if self.spec["is_continuous"] else self.head_dims
                for i, a in enumerate(heads):
                    out[f"actor.actor_heads.{i}.bias"] = (a,)
            else:
                out[k] = shp
        return out

    def load_reference_state(self, state: Dict[str, torch.Tensor]):
        """reference PPOAgent.state_dict() keys/shapes ('_forward_module.' infixes of Fabric wrappers are ignored)"""
        self.group.load(self.internal_state(state))

    def internal_state(self, state: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """tensors in the reference's keys / shapes -> the flat group's names / layouts (the inverse of
        export_reference_state; also used for optimizer state, which has the parameters' layout)"""
        st = {k.replace("_forward_module.", ""): v for k, v in state.items()}
        want = self.reference_shapes()
        missing, extra = set(want) - set(st), set(st) - set(want)
        if missing or extra:
            raise KeyError(f"state dict mismatch: missing={sorted(missing)} unexpected={sorted(extra)}")
        internal = {}
        heads = [self.head_width] if self.spec["is_continuous"] else self.head_dims
        for k, shp in self.group.shapes.items():
            if len(shp) == 4:
                internal[k] = st[k].permute(0, 2, 3, 1).contiguous()
            elif k.endswith("fc.weight") and self.geo:
                _, _, _, _, _, Ho, Wo, Co = self.geo[-1]
                internal[k] = st[k].reshape(shp[0], Co, Ho, Wo).permute(0, 2, 3, 1).reshape(shp)
            elif k == "actor.heads.weight":
                internal[k] = torch.cat([st[f"actor.actor_heads.{i}.weight"] for i in range(len(heads))], 0)
            elif k == "actor.heads.bias":
                internal[k] = torch.cat([st[f"actor.actor_heads.{i}.bias"] for i in range(len(heads))], 0)
            else:
                internal[k] = st[k]
        return internal

    def export_reference_state(self, views=None) -> "OrderedDict[str, torch.Tensor]":
        views = self.group.views if views is None else views
        out = OrderedDict()
        heads = [self.head_width] if self.spec["is_continuous"] else self.head_dims
        for k, shp in self.group.shapes.items():
            v = views[k].detach()
            if len(shp) == 4:
                out[k] = v.permute(0, 3, 1, 2).contiguous()
            elif k.endswith("fc.weight") and self.geo:
                _, _, _, _, _, Ho, Wo, Co = self.geo[-1]
                out[k] = v.reshape(shp[0], Ho, Wo, Co).permute(0, 3, 1, 2).reshape(shp).contiguous()
            elif k in ("actor.heads.weight", "actor.heads.bias"):
                off, kind = 0, k.rsplit(".", 1)[1]
                for i, a in enumerate(heads):
                    out[f"actor.actor_heads.{i}.{kind}"] = v[off:off + a].clone()
                    off += a
            else:
                out[k] = v.clone()
        return out

    # ------------------------------------------------------------------ buffers for a minibatch of B rows
    def _buffers(self, B: int) -> dict:
        if B in self._bufs:
            return self._bufs[B]
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        s = self.spec
        b = {"idx": torch.zeros(B, dtype=torch.int64, device=self.device)}
        if self.geo:
            H, W, C = self.geo[0][:3]
            b["x0"] = f(B, H, W, C)
            b["col"] = [f(1, B * Ho * Wo, k * k * Ci) for (_, _, Ci, k, _, Ho, Wo, _) in self.geo]
            b["y"] = [f(1, B * Ho * Wo, Co) for (_, _, _, _, _, Ho, Wo, Co) in self.geo]
            b["dy"] = [f(1, B * Ho * Wo, Co) for (_, _, _, _, _, Ho, Wo, Co) in self.geo]
            b["dcol"] = [None] + [f(1, B * Ho * Wo, k * k * Ci) for (_, _, Ci, k, _, Ho, Wo, _) in self.geo[1:]]
        b["feat"], b["dfeat"] = f(1, B, self.feat_dim), f(1, B, self.feat_dim)
        for name, st in (("menc", self.menc), ("critic", self.critic), ("actor", self.actor)):
            if st is not None:
                b[name] = st.acts(B)
        b["values"], b["dvalues"] = f(1, B, 1), f(1, B, 1)
        b["head"], b["dhead"] = f(1, B, self.head_width), f(1, B, self.head_width)
        self._bufs[B] = b
        return b

    def forward(self, b: dict, rgb, x_state, rgb_normalized: bool = False, actor: bool = True, critic: bool = True):
        """PPOAgent.forward up to the head / value outputs (ppo/agent.py:208-212) into the buffer set `b`.
        rgb: [B,C,H,W] uint8 / float raw 0..255 (normalised here, ppo/utils.py:69-72) or, with rgb_normalized, float
        already normalised (what the reference's rollout loop passes to the player); x_state: [1,B,mlp_dim]."""
        o = self.ops
        feat = b["feat"]
        B = feat.shape[1]
        if self.geo:
            if rgb_normalized:
                H, W, C = self.geo[0][:3]
                o.transpose_batched(rgb.float().contiguous().view(B, C, H * W), b["x0"].view(B, H * W, C))
            else:
                o.obs_prep(rgb, b["x0"])                    # /255 - 0.5, NCHW -> channel-last
            x = b["x0"]
            for i, (H, W, C, k, st, Ho, Wo, Co) in enumerate(self.geo):
                o.im2col(x, b["col"][i][0], k, st)
                self.convs[i].forward(o, b["col"][i], b["y"][i], "relu")
                x = b["y"][i][0].view(B, Ho, Wo, Co)
            self.fc.forward(o, b["y"][-1].view(1, B, -1), feat[:, :, :self.F], "relu")
        if self.menc is not None:
            self.menc.forward(x_state, b["menc"], feat[:, :, self.F:])
        if critic:
            self.critic.forward(feat, b["critic"], b["values"])
        if actor:
            self.actor.forward(feat, b["actor"], b["head"])

    # ------------------------------------------------------------------ one minibatch
    def minibatch_step(self, data: Dict[str, torch.Tensor], idx: torch.Tensor):
        """data: flat [N, ...] device tensors (rgb uint8 or float32 raw 0..255; everything else float32);
        idx: int64 device tensor of the minibatch rows."""
        o, s, hp = self.ops, self.spec, self.hp
        B = idx.numel()
        b = self._buffers(B)

        def rows(key):
            v = data[key]
            out = torch.empty((B, *v.shape[1:]), dtype=v.dtype, device=v.device)
            o.replay_gather(v.reshape(v.shape[0], -1), idx, out, 1, B, 1)
            return out

        # ---- forward
        x_state = rows("state").unsqueeze(0) if s["mlp_dim"] else None
        self.forward(b, rows("rgb") if self.geo else None, x_state)
        # ---- objective + gradients w.r.t. head outputs and values
        o.ppo_loss(b["head"][0], rows("actions"), rows("logprobs").reshape(-1), rows("advantages").reshape(-1),
                   b["values"].reshape(-1), rows("values").reshape(-1), rows("returns").reshape(-1), b["dhead"][0],
                   b["dvalues"].reshape(-1), self.losses, self.head_dims, self.dist_mode, hp["clip_vloss"],
                   hp["normalize_advantages"], hp["clip_coef"], hp["vf_coef"], hp["ent_coef"])
        self._backward(b, x_state)
        self._optimizer_step()

    def _backward(self, b: dict, x_state):
        """every weight gradient from b["dhead"] / b["dvalues"] (the objective's output) down to the encoders; each
        product reduces over all rows of `b`"""
        # actor, critic -> feature gradient (cnn columns masked by the fc ReLU)
        for j, (name, dout) in enumerate((("actor", b["dhead"]), ("critic", b["dvalues"]))):
            getattr(self, name).backward(dout, b["feat"], b[name], self.feature_grads(b), accumulate=j > 0)
        self._encoder_bwd(b, x_state)

    def feature_grads(self, b: dict, width: Optional[int] = None):
        """`Linear.input_grad` products of the feature gradient b["dfeat"] from a layer whose first `width` (default:
        all) inputs are the features: image columns times the fc ReLU's derivative, vector columns as they are"""
        F_, feat, dfeat = self.F, b["feat"], b["dfeat"]
        return ([(dfeat[:, :, :F_], slice(None, F_), "drelu", feat[:, :, :F_])] if F_ else []) + \
               ([(dfeat[:, :, F_:], slice(F_, width), "none", None)] if self.Mf else [])

    def _encoder_bwd(self, b: dict, x_state):
        """weight gradients of the vector and image encoders from b["dfeat"] (its image columns already masked by the
        fc ReLU)"""
        o, F_ = self.ops, self.F
        B = b["dfeat"].shape[1]
        if self.menc is not None:
            self.menc.backward(b["dfeat"][:, :, F_:], x_state, b["menc"])
        if self.geo:
            flat = b["y"][-1].view(1, B, -1)
            self.fc.weight_grad(o, b["dfeat"][:, :, :F_], flat)
            self.fc.input_grad(o, b["dfeat"][:, :, :F_], [(b["dy"][-1].view(1, B, -1), None, "drelu", flat)])
            for i in range(len(self.geo) - 1, -1, -1):
                H, W, C, k, st, Ho, Wo, Co = self.geo[i]
                self.convs[i].weight_grad(o, b["dy"][i], b["col"][i])
                if i > 0:
                    self.convs[i].input_grad(o, b["dy"][i], [(b["dcol"][i], None, "none", None)])
                    o.col2im(b["dcol"][i][0], b["y"][i - 1][0].view(B, H, W, C), b["dy"][i - 1][0].view(B, H, W, C), k, st)

    def _optimizer_step(self):
        o, hp = self.ops, self.hp
        # ---- all-reduce, clip, Adam (ppo.py:92-96)
        g = self.group
        if self.allreduce is not None:
            self.allreduce(g.grad, "agent")
        if hp["max_grad_norm"] > 0:
            o.sumsq(g.grad, self.normsq)
        o.increment(g.step_t)
        g.step += 1
        handle = getattr(g, "optimizer", None)              # B200Adam: the reference's PolynomialLR edits its param_groups
        self._apply_update(handle.lr if handle is not None else self.opt["lr"])

    def _apply_update(self, lr: float):
        """the fused clip + optimizer update of the flat group (gradient norm already in self.normsq)"""
        g = self.group
        self.ops.adam_step(g.flat, g.grad, g.exp_avg, g.exp_avg_sq, self.normsq, float(self.hp["max_grad_norm"]), lr,
                           self.opt["betas"][0], self.opt["betas"][1], self.opt["eps"], g.step_t, self.norm_out,
                           **g.adam_kwargs(self.opt.get("weight_decay", 0.0)))

    def train(self, data: Dict[str, torch.Tensor], index_batches: Sequence[Sequence[int]], on_minibatch=None):
        sync_deterministic(self.ops)
        for ib in index_batches:
            idx = torch.as_tensor(ib, dtype=torch.int64).to(self.device, non_blocking=True)
            self.minibatch_step(data, idx)
            if on_minibatch is not None:
                on_minibatch(self.losses.clone())
