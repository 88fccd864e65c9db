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

from sheeprl_b200.algos.ppo.engine import PPOEngine
from sheeprl_b200.dense import Act, LayerNormAct, Linear, Stack

RNN_LN_EPS = 1e-3                                     # RecurrentModel's pre/post MLP LayerNorm (agent.py:31-35, 52-56)


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

    @property
    def actor_in(self) -> int:
        """the critic and actor read the H-wide RNN output"""
        return self.H

    def _internal_shapes(self):
        out = OrderedDict()
        base = super()._internal_shapes()             # encoders, critic / actor on H inputs, stacked heads
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
        for k, v in base.items():
            if k.startswith(("critic.", "actor.")):
                out[k] = v
        return out

    def _build_layers(self):
        super()._build_layers()
        v, g = self.group.views, self.group.gviews
        self.pre_mlp = self._rnn_mlp("rnn._pre_mlp", self.pre_cfg)
        self.post_mlp = self._rnn_mlp("rnn._post_mlp", self.post_cfg)
        self.bsum = torch.zeros(4 * self.H, dtype=torch.float32, device=self.device)    # b_ih + b_hh
        self.W_ih = Linear(v["rnn._lstm.weight_ih_l0"].unsqueeze(0), self.bsum.unsqueeze(0),
                           g["rnn._lstm.weight_ih_l0"].unsqueeze(0), g["rnn._lstm.bias_ih_l0"].unsqueeze(0))
        self.W_hh, self.gW_hh = v["rnn._lstm.weight_hh_l0"], g["rnn._lstm.weight_hh_l0"].unsqueeze(0)
        self.b_ih, self.b_hh = v["rnn._lstm.bias_ih_l0"], v["rnn._lstm.bias_hh_l0"]
        self.gb_ih, self.gb_hh = g["rnn._lstm.bias_ih_l0"], g["rnn._lstm.bias_hh_l0"]

    def _rnn_mlp(self, prefix: str, cfg) -> Optional[Stack]:
        """the pre- / post-RNN MLP (models.py MLP with one hidden size and no output layer): Linear `{prefix}._model.0`
        -> [LayerNorm(eps 1e-3) `{prefix}._model.1`] -> act"""
        if not cfg:
            return None
        block = LayerNormAct(self.group, f"{prefix}._model.1", RNN_LN_EPS, self.act) if cfg[1] else Act(self.act)
        return Stack(self.ops, [(Linear.of(self.group, f"{prefix}._model.0.weight"), block)])

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
                dense = mlp.layers[0][0].W.shape[1]
                b[name + "_y"], b["d" + name + "_y"], b[name] = f(1, N, dense), f(1, N, dense), mlp.acts(N)
        b["xw"], b["hbuf"], b["c0"] = f(T, B, G), f(T + 1, B, H), f(B, H)
        b["gates"], b["cs"], b["dout"], b["dgates"] = f(T, B, G), f(T, B, H), f(T, B, H), f(T, B, G)
        b["lengths"] = torch.ones(B, dtype=torch.int32, device=self.device)
        b["T"], b["B"] = T, B
        self._rbufs[key] = b
        return b

    # ------------------------------------------------------------------ forward
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
            self.pre_mlp.forward(x, b["pre"], b["pre_y"])
            x = b["pre_y"]
        o.copy(self.b_ih, self.bsum)
        o.axpy(self.b_hh, self.bsum)
        self.W_ih.forward(o, x, b["xw"].view(1, N, -1))
        o.lstm_seq_fwd(b["xw"], self.W_hh, b["hbuf"][0], b["c0"], b["lengths"], b["hbuf"][1:],
                       b["gates"] if keep else None, b["cs"] if keep else None, hT, cT)
        y = b["hbuf"][1:].view(1, N, self.H)
        if self.post_mlp is not None:
            self.post_mlp.forward(y, b["post"], b["post_y"])
            y = b["post_y"]
        if critic:
            self.critic.forward(y, b["critic"], b["values"])
        if actor:
            self.actor.forward(y, b["actor"], b["head"])
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
        post, pre = self.post_mlp, self.pre_mlp
        h_out = b["hbuf"][1:].view(1, N, self.H)
        dy = [(b["dpost_y"], None, *post.layers[0][1].dx_epi(b["post_y"])) if post is not None else
              (b["dout"].view(1, N, self.H), None, "none", None)]
        for j, (name, dout) in enumerate((("actor", b["dhead"]), ("critic", b["dvalues"]))):
            getattr(self, name).backward(dout, y, b[name], dy, accumulate=j > 0)
        if post is not None:
            post.backward(b["dpost_y"], h_out, b["post"], [(b["dout"].view(1, N, self.H), None, "none", None)])
        # ---- LSTM: one backward-through-time launch, then the dense products over all N rows
        o.lstm_seq_bwd(b["dout"], self.W_hh, b["gates"], b["cs"], b["c0"], b["lengths"], b["dgates"])
        dg = b["dgates"].view(1, N, 4 * self.H)
        self.W_ih.weight_grad(o, dg, b["pre_y"] if pre is not None else b["xin"])
        o.copy(self.gb_ih, self.gb_hh)
        o.bgemm(dg.transpose(1, 2), b["hbuf"][:-1].view(1, N, self.H), self.gW_hh)
        # ---- feature gradient (image columns masked by the fc ReLU), encoders, clip + Adam
        feats = self.feature_grads(b, self.feat_dim)
        if pre is not None:
            self.W_ih.input_grad(o, dg, [(b["dpre_y"], None, *pre.layers[0][1].dx_epi(b["pre_y"]))])
            pre.backward(b["dpre_y"], b["xin"], b["pre"], feats)
        else:
            self.W_ih.input_grad(o, dg, feats)
        self._encoder_bwd(b, x_state)
        self._optimizer_step()

    def train(self, data: Dict[str, torch.Tensor], index_batches: Sequence[Sequence[int]], on_minibatch=None,
              prepared: Optional[dict] = None):
        d = prepared if prepared is not None else self.prepare(data)
        for ib in index_batches:
            seqs = torch.as_tensor(ib, dtype=torch.int64).to(self.device, non_blocking=True)
            self.minibatch_step(d, seqs)
            if on_minibatch is not None:
                on_minibatch(self.losses.clone())
