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
from typing import Dict, List, Optional, Sequence

import torch

from sheeprl_b200.params import FlatGroup

CONVS = ((8, 4, 32), (4, 2, 64), (3, 1, 64))        # NatureCNN (kernel, stride, channels) models.py:301-309
LN_EPS = 1e-5                                        # nn.LayerNorm default (ppo/agent.py:63-64 passes only the shape)
ACT_CODE = {"none": 0, "tanh": 2, "relu": 3}         # b200rl_ln_act_* activation codes
DIST_MODE = {"discrete": 0, "normal": 1, "tanh_normal": 2}


def net_cfg(spec: dict, which: str):
    """(dense_units, mlp_layers, layer_norm) of the "encoder" / "actor" / "critic" MLP: spec["nets"][which] = (dense,
    layers) and spec["layer_norm"] (bool or per-net dict) override the shared spec["dense"] / spec["layers"]."""
    dense, layers = (spec.get("nets") or {}).get(which, (spec["dense"], spec["layers"]))
    ln = spec.get("layer_norm", False)
    ln = bool(ln.get(which, False)) if isinstance(ln, dict) else bool(ln)
    return int(dense), int(layers), ln


class _Lin:
    """One Linear layer bound to flat-group views: W [1,out,in], b [1,out] and their gradients."""

    def __init__(self, eng, wkey: str, act: str):
        v, g = eng.group.views, eng.group.gviews
        bkey = wkey[:-6] + "bias"
        self.W, self.b = v[wkey].unsqueeze(0), v[bkey].unsqueeze(0)
        self.gW, self.gb = g[wkey].unsqueeze(0), g[bkey].unsqueeze(0)
        self.act = act
        self.ln = None                                   # (gamma, beta, dgamma, dbeta) when a LayerNorm follows


class _Stack:
    """An `MLP` of the reference (models/models.py:17-126): `layers` hidden blocks Linear [-> LayerNorm] -> act, then an
    output Linear without activation (absent for the actor backbone, whose output layer is the stacked action heads)."""

    def __init__(self, eng, prefix: str, which: str, tag: str, last_key: Optional[str] = None):
        dense, layers, ln = net_cfg(eng.spec, which)
        st = 3 if ln else 2
        v, g = eng.group.views, eng.group.gviews
        self.tag, self.has_ln, self.dense = tag, ln, dense
        self.lins: List[_Lin] = []
        for i in range(layers):
            lin = _Lin(eng, f"{prefix}._model.{st * i}.weight", eng.act)
            if ln:
                wk, bk = f"{prefix}._model.{st * i + 1}.weight", f"{prefix}._model.{st * i + 1}.bias"
                lin.ln = (v[wk], v[bk], g[wk], g[bk])
            self.lins.append(lin)
        self.lins.append(_Lin(eng, last_key or f"{prefix}._model.{st * layers}.weight", "none"))

    @property
    def n_hidden(self):
        return len(self.lins) - 1


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
        stack("critic", self.feat_dim, "critic", 1)
        stack("actor.actor_backbone", self.feat_dim, "actor", None)
        # every head reads `actor.dense_units` inputs, also with an empty backbone (ppo/agent.py:180-183)
        out["actor.heads.weight"] = (self.head_width, net_cfg(s, "actor")[0])
        out["actor.heads.bias"] = (self.head_width,)
        return out

    def _build_layers(self):
        s = self.spec
        pre = "feature_extractor.cnn_encoder.model"
        self.convs = [_Lin(self, f"{pre}._model.{2 * i}.weight", "relu") for i in range(len(self.geo))]
        for c in self.convs:                              # [1, Cout, k*k*Cin]
            c.W, c.gW = c.W.flatten(2), c.gW.flatten(2)
        self.fc = _Lin(self, f"{pre}.fc.weight", "relu") if self.geo else None
        self.menc = _Stack(self, "feature_extractor.mlp_encoder.model", "encoder", "m") if s["mlp_dim"] else None
        self.critic = _Stack(self, "critic", "critic", "c")
        self.actor = _Stack(self, "actor.actor_backbone", "actor", "a", last_key="actor.heads.weight")
        if self.actor.n_hidden == 0 and self.actor.dense != self.feat_dim:
            raise ValueError("actor.mlp_layers == 0 needs actor.dense_units == feature dim (the heads read dense_units inputs)")

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
        self.group.load(internal)

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
        for st in (self.menc, self.critic, self.actor):
            if st is None:
                continue
            n, D = st.n_hidden, st.dense
            b[st.tag + "h"], b["d" + st.tag + "h"] = [f(1, B, D) for _ in range(n)], [f(1, B, D) for _ in range(n)]
            b[st.tag + "pre"] = [f(1, B, D) for _ in range(n)] if st.has_ln else None     # pre-LayerNorm activations
        b["values"], b["dvalues"] = f(1, B, 1), f(1, B, 1)
        b["head"], b["dhead"] = f(1, B, self.head_width), f(1, B, self.head_width)
        self._bufs[B] = b
        return b

    # ------------------------------------------------------------------ layer helpers
    def _fwd(self, lin: _Lin, x, y):
        self.ops.bgemm(x, lin.W.transpose(1, 2), y, bias=lin.b, epi=lin.act)

    def _bwd(self, lin: _Lin, dpre, x, dx=None, dx_epi="none", dx_aux=None, accumulate_dx=False, Wcols=None):
        """weight/bias gradient of `lin` from the pre-activation gradient `dpre`; optionally the input gradient
        (times the derivative `dx_epi` of the producer's activation, whose output is `dx_aux`)."""
        o = self.ops
        o.bgemm(dpre.transpose(1, 2), x, lin.gW, rsum=lin.gb)
        if dx is not None:
            W = lin.W if Wcols is None else lin.W[:, :, Wcols[0]:Wcols[1]]
            o.bgemm(dpre, W, dx, aux=dx_aux, epi=dx_epi, accumulate=accumulate_dx)

    def _mlp_fwd(self, st: _Stack, b: dict, x, out):
        hidden, pre = b[st.tag + "h"], b[st.tag + "pre"]
        for i, lin in enumerate(st.lins):
            y = hidden[i] if i < st.n_hidden else out
            if lin.ln is not None:                          # Linear -> LayerNorm -> act (utils/model.py:76-87)
                self.ops.bgemm(x, lin.W.transpose(1, 2), pre[i], bias=lin.b)
                self.ops.ln_act_fwd(pre[i][0], lin.ln[0], lin.ln[1], LN_EPS, ACT_CODE[lin.act], y[0])
            else:
                self._fwd(lin, x, y)
            x = y

    def _mlp_bwd(self, st: _Stack, b: dict, dout):
        """backward through the stack down to its first layer; weight / LayerNorm gradients of layers >= 1 are written,
        the return value is the gradient w.r.t. layer 0's Linear output (the caller owns layer 0's products)."""
        hidden, dhidden, pre = b[st.tag + "h"], b["d" + st.tag + "h"], b[st.tag + "pre"]
        dpre = dout
        for i in range(st.n_hidden, 0, -1):
            below = st.lins[i - 1]
            if below.ln is not None:
                self._bwd(st.lins[i], dpre, hidden[i - 1], dx=dhidden[i - 1])
                gam, bet, dgam, dbet = below.ln
                self.ops.ln_act_bwd(pre[i - 1][0], gam, bet, LN_EPS, ACT_CODE[below.act], dhidden[i - 1][0], dhidden[i - 1][0],
                                    dgam, dbet)
            else:
                self._bwd(st.lins[i], dpre, hidden[i - 1], dx=dhidden[i - 1], dx_epi="d" + below.act, dx_aux=hidden[i - 1])
            dpre = dhidden[i - 1]
        return dpre

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
                self._fwd(self.convs[i], b["col"][i], b["y"][i])
                x = b["y"][i][0].view(B, Ho, Wo, Co)
            self._fwd(self.fc, b["y"][-1].view(1, B, -1), feat[:, :, :self.F])
        if self.menc is not None:
            self._mlp_fwd(self.menc, b, x_state, feat[:, :, self.F:])
        if critic:
            self._mlp_fwd(self.critic, b, feat, b["values"])
        if actor:
            self._mlp_fwd(self.actor, b, feat, b["head"])

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
        feat = b["feat"]
        x_state = rows("state").unsqueeze(0) if s["mlp_dim"] else None
        self.forward(b, rows("rgb") if self.geo else None, x_state)
        # ---- objective + gradients w.r.t. head outputs and values
        o.ppo_loss(b["head"][0], rows("actions"), rows("logprobs").reshape(-1), rows("advantages").reshape(-1),
                   b["values"].reshape(-1), rows("values").reshape(-1), rows("returns").reshape(-1), b["dhead"][0],
                   b["dvalues"].reshape(-1), self.losses, self.head_dims, self.dist_mode, hp["clip_vloss"],
                   hp["normalize_advantages"], hp["clip_coef"], hp["vf_coef"], hp["ent_coef"])
        # ---- backward: actor, critic -> feature gradient (cnn columns masked by the fc ReLU)
        F_ = self.F
        for j, (st, dout) in enumerate(((self.actor, b["dhead"]), (self.critic, b["dvalues"]))):
            dpre0, l0 = self._mlp_bwd(st, b, dout), st.lins[0]
            o.bgemm(dpre0.transpose(1, 2), feat, l0.gW, rsum=l0.gb)
            if F_:
                o.bgemm(dpre0, l0.W[:, :, :F_], b["dfeat"][:, :, :F_], aux=feat[:, :, :F_], epi="drelu", accumulate=j > 0)
            if self.Mf:
                o.bgemm(dpre0, l0.W[:, :, F_:], b["dfeat"][:, :, F_:], accumulate=j > 0)
        self._encoder_bwd(b, x_state)
        self._optimizer_step()

    def _encoder_bwd(self, b: dict, x_state):
        """weight gradients of the vector and image encoders from b["dfeat"] (its image columns already masked by the
        fc ReLU)"""
        o, F_ = self.ops, self.F
        B = b["dfeat"].shape[1]
        if self.menc is not None:
            dpre0, l0 = self._mlp_bwd(self.menc, b, b["dfeat"][:, :, F_:]), self.menc.lins[0]
            o.bgemm(dpre0.transpose(1, 2), x_state, l0.gW, rsum=l0.gb)
        if self.geo:
            n = len(self.geo)
            flat = b["y"][-1].view(1, B, -1)
            self._bwd(self.fc, b["dfeat"][:, :, :F_], flat, dx=b["dy"][-1].view(1, B, -1), dx_epi="drelu", dx_aux=flat)
            for i in range(n - 1, -1, -1):
                H, W, C, k, st, Ho, Wo, Co = self.geo[i]
                if i > 0:
                    self._bwd(self.convs[i], b["dy"][i], b["col"][i], dx=b["dcol"][i])
                    o.col2im(b["dcol"][i][0], b["y"][i - 1][0].view(B, H, W, C), b["dy"][i - 1][0].view(B, H, W, C), k, st)
                else:
                    self._bwd(self.convs[0], b["dy"][0], b["col"][0])

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
        lr = handle.lr if handle is not None else self.opt["lr"]
        o.adam_step(g.flat, g.grad, g.exp_avg, g.exp_avg_sq, self.normsq, float(hp["max_grad_norm"]), lr,
                    self.opt["betas"][0], self.opt["betas"][1], self.opt["eps"], g.step_t, self.norm_out)

    def train(self, data: Dict[str, torch.Tensor], index_batches: Sequence[Sequence[int]], on_minibatch=None):
        for ib in index_batches:
            idx = torch.as_tensor(ib, dtype=torch.int64).to(self.device, non_blocking=True)
            self.minibatch_step(data, idx)
            if on_minibatch is not None:
                on_minibatch(self.losses.clone())
