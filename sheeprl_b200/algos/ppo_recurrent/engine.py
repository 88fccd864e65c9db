"""Kernel schedule of the recurrent PPO update: PPO with a single-layer LSTM between the encoders and the actor / critic.

Reference being replaced: `train` sheeprl/algos/ppo_recurrent/ppo_recurrent.py:31-116, `RecurrentPPOAgent.forward` /
`RecurrentModel.forward` ppo_recurrent/agent.py:67-80, 233-262 (pack_padded_sequence -> nn.LSTM -> pad_packed_sequence)
and the masked losses of ppo/loss.py.  `ops` is `sheeprl_b200.lib.CudaOps` in production (tests on a GPU-less host pass
the torch test double `oracle/ops_emul_recurrent.py::RecurrentEmulOps`).

The engine is a `PPOEngine` (same flat parameter group, encoders, LayerNorm MLP stacks, stacked action heads and fused
clip+Adam) whose actor and critic read the LSTM output instead of the features.  Per minibatch of B sequences of T
steps (N = T*B time-major rows):

  gather rows -> encoders -> [features | prev_actions] -> optional pre-MLP -> xw = x W_ih^T + b_ih + b_hh (one product)
  -> lstm_seq_fwd (one launch for all T steps) -> optional post-MLP -> critic, actor -> ppo_loss_masked
  -> backward in reverse: heads, post-MLP, lstm_seq_bwd (one launch), dW_ih / dW_hh / biases / input gradient as four
     products over all N rows, pre-MLP, encoders -> clip+Adam.

So the LSTM costs a fixed handful of launches whatever T is.  The hidden state row t of sequence b lives in
`hbuf[t + 1, b]` and `hbuf[0]` holds the sequence's initial state, so the h_{t-1} operand of dW_hh is `hbuf[:-1]`.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional, Sequence

import torch

from sheeprl_b200.algos.ppo.engine import ACT_CODE, PPOEngine, _Lin, _Stack

RNN_LN_EPS = 1e-3                                     # RecurrentModel's pre/post MLP LayerNorm (agent.py:31-35, 52-56)


class _Dense:
    """One hidden block Linear -> [LayerNorm(eps 1e-3)] -> act of the pre- / post-RNN MLP (models.py MLP with one
    hidden size and no output layer): keys `{prefix}._model.0.*` and, with LayerNorm, `{prefix}._model.1.*`."""

    def __init__(self, eng, prefix: str, ln: bool, act: str):
        v, g = eng.group.views, eng.group.gviews
        self.W, self.b = v[f"{prefix}._model.0.weight"].unsqueeze(0), v[f"{prefix}._model.0.bias"].unsqueeze(0)
        self.gW, self.gb = g[f"{prefix}._model.0.weight"].unsqueeze(0), g[f"{prefix}._model.0.bias"].unsqueeze(0)
        self.ln = (v[f"{prefix}._model.1.weight"], v[f"{prefix}._model.1.bias"], g[f"{prefix}._model.1.weight"],
                   g[f"{prefix}._model.1.bias"]) if ln else None
        self.act = act
        self.dense = self.W.shape[1]


class RecurrentPPOEngine(PPOEngine):
    def __init__(self, spec: dict, hp: dict, opt: dict, device, ops, seed: int = 0):
        """spec: the PPOEngine spec plus rnn = dict(hidden=H, pre=None | (dense_units, layer_norm),
        post=None | (dense_units, layer_norm)).  Discrete actions only."""
        if spec["is_continuous"]:
            raise NotImplementedError("recurrent PPO supports discrete actions only (the reference's continuous path "
                                      "fails in RecurrentPPOAgent._get_actions)")
        rnn = spec["rnn"]
        self.H = int(rnn["hidden"])
        self.pre_cfg = tuple(rnn["pre"]) if rnn.get("pre") else None
        self.post_cfg = tuple(rnn["post"]) if rnn.get("post") else None
        if self.post_cfg and int(self.post_cfg[0]) != self.H:
            raise ValueError(f"rnn.post_rnn_mlp.dense_units ({self.post_cfg[0]}) must equal rnn.lstm.hidden_size "
                             f"({self.H}): RecurrentModel.forward reshapes the post-MLP output to the LSTM output shape")
        super().__init__(spec, hp, opt, device, ops, seed)
        self._rbufs: Dict[tuple, dict] = {}

    # ------------------------------------------------------------------ parameters
    @property
    def n_actions(self) -> int:
        return sum(self.head_dims)

    @property
    def lstm_in(self) -> int:
        return int(self.pre_cfg[0]) if self.pre_cfg else self.feat_dim + self.n_actions

    def _internal_shapes(self):
        out = OrderedDict()
        base = super()._internal_shapes()             # encoders, critic / actor on feat_dim inputs, stacked heads
        for k, v in base.items():
            if k.startswith("feature_extractor."):
                out[k] = v
        H, G = self.H, 4 * self.H
        d_in = self.feat_dim + self.n_actions
        if self.pre_cfg:
            dense, ln = int(self.pre_cfg[0]), bool(self.pre_cfg[1])
            out["rnn._pre_mlp._model.0.weight"], out["rnn._pre_mlp._model.0.bias"] = (dense, d_in), (dense,)
            if ln:
                out["rnn._pre_mlp._model.1.weight"], out["rnn._pre_mlp._model.1.bias"] = (dense,), (dense,)
        out["rnn._lstm.weight_ih_l0"], out["rnn._lstm.weight_hh_l0"] = (G, self.lstm_in), (G, H)
        out["rnn._lstm.bias_ih_l0"], out["rnn._lstm.bias_hh_l0"] = (G,), (G,)
        if self.post_cfg:
            ln = bool(self.post_cfg[1])
            out["rnn._post_mlp._model.0.weight"], out["rnn._post_mlp._model.0.bias"] = (H, H), (H,)
            if ln:
                out["rnn._post_mlp._model.1.weight"], out["rnn._post_mlp._model.1.bias"] = (H,), (H,)
        for k, v in base.items():                      # critic / actor read the H-wide RNN output
            if k.startswith(("critic.", "actor.")):
                out[k] = (v[0], H) if k.endswith("._model.0.weight") else v
        return out

    def _build_layers(self):
        s = self.spec
        pre = "feature_extractor.cnn_encoder.model"
        self.convs = [_Lin(self, f"{pre}._model.{2 * i}.weight", "relu") for i in range(len(self.geo))]
        for c in self.convs:
            c.W, c.gW = c.W.flatten(2), c.gW.flatten(2)
        self.fc = _Lin(self, f"{pre}.fc.weight", "relu") if self.geo else None
        self.menc = _Stack(self, "feature_extractor.mlp_encoder.model", "encoder", "m") if s["mlp_dim"] else None
        self.critic = _Stack(self, "critic", "critic", "c")
        self.actor = _Stack(self, "actor.actor_backbone", "actor", "a", last_key="actor.heads.weight")
        if self.actor.n_hidden == 0 and self.actor.dense != self.H:
            raise ValueError("actor.mlp_layers == 0 needs actor.dense_units == rnn.lstm.hidden_size")
        v, g = self.group.views, self.group.gviews
        self.pre_mlp = _Dense(self, "rnn._pre_mlp", bool(self.pre_cfg[1]), self.act) if self.pre_cfg else None
        self.post_mlp = _Dense(self, "rnn._post_mlp", bool(self.post_cfg[1]), self.act) if self.post_cfg else None
        self.W_ih, self.gW_ih = v["rnn._lstm.weight_ih_l0"].unsqueeze(0), g["rnn._lstm.weight_ih_l0"].unsqueeze(0)
        self.W_hh, self.gW_hh = v["rnn._lstm.weight_hh_l0"], g["rnn._lstm.weight_hh_l0"].unsqueeze(0)
        self.b_ih, self.b_hh = v["rnn._lstm.bias_ih_l0"], v["rnn._lstm.bias_hh_l0"]
        self.gb_ih, self.gb_hh = g["rnn._lstm.bias_ih_l0"], g["rnn._lstm.bias_hh_l0"]
        self.bsum = torch.zeros(4 * self.H, dtype=torch.float32, device=self.device)

    # ------------------------------------------------------------------ buffers for B sequences of T steps
    def seq_buffers(self, T: int, B: int) -> dict:
        key = (T, B)
        if key in self._rbufs:
            return self._rbufs[key]
        N, H, G = T * B, self.H, 4 * self.H
        b = dict(PPOEngine._buffers(self, N))           # encoder / critic / actor buffers of N rows
        self._bufs.pop(N, None)
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        b["xin"] = f(1, N, self.feat_dim + self.n_actions)
        b["feat"] = b["xin"][:, :, :self.feat_dim]      # the encoders write their columns in place
        for name, mlp in (("pre", self.pre_mlp), ("post", self.post_mlp)):
            if mlp is not None:
                b[name + "_y"], b["d" + name + "_y"] = f(1, N, mlp.dense), f(1, N, mlp.dense)
                b[name + "_pre"] = f(1, N, mlp.dense) if mlp.ln is not None else None
        b["xw"], b["hbuf"], b["c0"] = f(T, B, G), f(T + 1, B, H), f(B, H)
        b["gates"], b["cs"], b["dout"], b["dgates"] = f(T, B, G), f(T, B, H), f(T, B, H), f(T, B, G)
        b["lengths"] = torch.ones(B, dtype=torch.int32, device=self.device)
        b["T"], b["B"] = T, B
        self._rbufs[key] = b
        return b

    # ------------------------------------------------------------------ forward
    def _dense_fwd(self, m: _Dense, b: dict, name: str, x):
        y = b[name + "_y"]
        if m.ln is not None:
            self.ops.bgemm(x, m.W.transpose(1, 2), b[name + "_pre"], bias=m.b)
            self.ops.ln_act_fwd(b[name + "_pre"][0], m.ln[0], m.ln[1], RNN_LN_EPS, ACT_CODE[m.act], y[0])
        else:
            self.ops.bgemm(x, m.W.transpose(1, 2), y, bias=m.b, epi=m.act)
        return y

    def seq_forward(self, b: dict, rgb, x_state, prev_actions, rgb_normalized: bool = False, keep: bool = True,
                    hT=None, cT=None, actor: bool = True, critic: bool = True):
        """RecurrentPPOAgent.forward up to the head / value outputs for the sequences of buffer set `b`, whose
        b["hbuf"][0], b["c0"] and b["lengths"] the caller has filled.  prev_actions: [N, sum(actions_dim)] rows."""
        o = self.ops
        T, B = b["T"], b["B"]
        N = T * B
        self.forward(b, rgb, x_state, rgb_normalized=rgb_normalized, actor=False, critic=False)   # encoders -> feat
        o.copy(prev_actions.reshape(N, -1), b["xin"][0][:, self.feat_dim:])
        x = b["xin"]
        if self.pre_mlp is not None:
            x = self._dense_fwd(self.pre_mlp, b, "pre", x)
        o.copy(self.b_ih, self.bsum)
        o.axpy(self.b_hh, self.bsum)
        o.bgemm(x, self.W_ih.transpose(1, 2), b["xw"].view(1, N, -1), bias=self.bsum.unsqueeze(0))
        o.lstm_seq_fwd(b["xw"], self.W_hh, b["hbuf"][0], b["c0"], b["lengths"], b["hbuf"][1:],
                       b["gates"] if keep else None, b["cs"] if keep else None, hT, cT)
        y = b["hbuf"][1:].view(1, N, self.H)
        if self.post_mlp is not None:
            y = self._dense_fwd(self.post_mlp, b, "post", y)
        if critic:
            self._mlp_fwd(self.critic, b, y, b["values"])
        if actor:
            self._mlp_fwd(self.actor, b, y, b["head"])
        return y

    # ------------------------------------------------------------------ one minibatch
    def prepare(self, data: Dict[str, torch.Tensor]) -> dict:
        """[T, S, ...] rollout tensors -> time-major row storage [T*S, ...] plus the per-sequence lengths.  The mask
        must be a prefix of each column (what the reference's pad_sequence produces); anything else is refused."""
        mask = data["mask"]
        mask = mask.reshape(mask.shape[0], mask.shape[1]).to(torch.bool)
        T, S = mask.shape
        lengths = mask.sum(0)
        prefix = torch.arange(T, device=mask.device).unsqueeze(1) < lengths.unsqueeze(0)
        if not bool(torch.equal(mask, prefix)) or bool((lengths < 1).any()):
            raise ValueError("mask must be a non-empty prefix of every sequence column (padding only at the end)")
        d = {"T": T, "S": S, "lengths": lengths.to(torch.int32).contiguous(),
             "mask": mask.float().reshape(T * S, 1).contiguous()}
        for k in ("actions", "logprobs", "values", "returns", "advantages", "prev_actions"):
            d[k] = data[k].float().reshape(T * S, -1).contiguous()
        for k in ("prev_hx", "prev_cx"):
            d[k] = data[k][0].float().reshape(S, -1).contiguous()
        for k in ("rgb", "state"):
            if data.get(k) is not None:
                v = data[k]
                d[k] = v.reshape(T * S, *v.shape[2:]).contiguous()
        return d

    def minibatch_step(self, d: dict, seqs: torch.Tensor):
        """d: `prepare()`d rollout; seqs: int64 device tensor of the minibatch's sequence (column) indices."""
        o, s, hp = self.ops, self.spec, self.hp
        T, S, B = d["T"], d["S"], seqs.numel()
        N = T * B
        b = self.seq_buffers(T, B)
        rows_idx = (torch.arange(T, device=seqs.device).unsqueeze(0) * S + seqs.unsqueeze(1)).reshape(-1)

        def rows(key):
            v = d[key]
            out = torch.empty((N, *v.shape[1:]), dtype=v.dtype, device=v.device)
            o.replay_gather(v.reshape(v.shape[0], -1), rows_idx, out, 1, B, T)
            return out

        o.replay_gather(d["prev_hx"], seqs, b["hbuf"][0], 1, B, 1)
        o.replay_gather(d["prev_cx"], seqs, b["c0"], 1, B, 1)
        o.replay_gather(d["lengths"].view(S, 1), seqs, b["lengths"], 1, B, 1)
        x_state = rows("state").unsqueeze(0) if s["mlp_dim"] else None
        y = self.seq_forward(b, rows("rgb") if self.geo else None, x_state, rows("prev_actions"))
        o.ppo_loss_masked(b["head"][0], rows("actions"), rows("logprobs").reshape(-1), rows("advantages").reshape(-1),
                          b["values"].reshape(-1), rows("values").reshape(-1), rows("returns").reshape(-1),
                          rows("mask").reshape(-1), b["dhead"][0], b["dvalues"].reshape(-1), self.losses,
                          self.head_dims, 0, hp["clip_vloss"], hp["normalize_advantages"], hp["clip_coef"],
                          hp["vf_coef"], hp["ent_coef"])
        # ---- backward: actor, critic -> gradient w.r.t. the RNN output (post-MLP output)
        post = self.post_mlp
        dy = b["dpost_y"] if post is not None else b["dout"].view(1, N, self.H)
        epi = "d" + post.act if (post is not None and post.ln is None) else "none"
        aux = b["post_y"] if epi != "none" else None
        for j, (st, dout) in enumerate(((self.actor, b["dhead"]), (self.critic, b["dvalues"]))):
            dpre0, l0 = self._mlp_bwd(st, b, dout), st.lins[0]
            o.bgemm(dpre0.transpose(1, 2), y, l0.gW, rsum=l0.gb)
            o.bgemm(dpre0, l0.W, dy, aux=aux, epi=epi, accumulate=j > 0)
        h_out = b["hbuf"][1:].view(1, N, self.H)
        if post is not None:
            self._dense_bwd(post, b, "post", h_out)
            o.bgemm(b["dpost_y"], post.W, b["dout"].view(1, N, self.H))
        # ---- LSTM: one backward-through-time launch, then the dense products over all N rows
        o.lstm_seq_bwd(b["dout"], self.W_hh, b["gates"], b["cs"], b["c0"], b["lengths"], b["dgates"])
        dg = b["dgates"].view(1, N, 4 * self.H)
        x = b["pre_y"] if self.pre_mlp is not None else b["xin"]
        o.bgemm(dg.transpose(1, 2), x, self.gW_ih, rsum=self.gb_ih.unsqueeze(0))
        o.copy(self.gb_ih, self.gb_hh)
        o.bgemm(dg.transpose(1, 2), b["hbuf"][:-1].view(1, N, self.H), self.gW_hh)
        if self.pre_mlp is not None:
            pm = self.pre_mlp
            pepi = "d" + pm.act if pm.ln is None else "none"
            o.bgemm(dg, self.W_ih, b["dpre_y"], aux=b["pre_y"] if pm.ln is None else None, epi=pepi)
            self._dense_bwd(pm, b, "pre", b["xin"])
            dfirst, Wfirst = b["dpre_y"], pm.W
        else:
            dfirst, Wfirst = dg, self.W_ih
        # ---- feature gradient (image columns masked by the fc ReLU), encoders, clip + Adam
        F_, feat = self.F, b["feat"]
        if F_:
            o.bgemm(dfirst, Wfirst[:, :, :F_], b["dfeat"][:, :, :F_], aux=feat[:, :, :F_], epi="drelu")
        if self.Mf:
            o.bgemm(dfirst, Wfirst[:, :, F_:self.feat_dim], b["dfeat"][:, :, F_:])
        self._encoder_bwd(b, x_state)
        self._optimizer_step()

    def _dense_bwd(self, m: _Dense, b: dict, name: str, x):
        """b["d<name>_y"] holds the gradient w.r.t. the block's output (already times act' when there is no
        LayerNorm); turn it into the Linear output gradient in place and write the weight / LayerNorm gradients."""
        d = b["d" + name + "_y"]
        if m.ln is not None:
            gam, bet, dgam, dbet = m.ln
            self.ops.ln_act_bwd(b[name + "_pre"][0], gam, bet, RNN_LN_EPS, ACT_CODE[m.act], d[0], d[0], dgam, dbet)
        self.ops.bgemm(d.transpose(1, 2), x, m.gW, rsum=m.gb)

    def train(self, data: Dict[str, torch.Tensor], index_batches: Sequence[Sequence[int]], on_minibatch=None,
              prepared: Optional[dict] = None):
        d = prepared if prepared is not None else self.prepare(data)
        for ib in index_batches:
            seqs = torch.as_tensor(ib, dtype=torch.int64).to(self.device, non_blocking=True)
            self.minibatch_step(d, seqs)
            if on_minibatch is not None:
                on_minibatch(self.losses.clone())
