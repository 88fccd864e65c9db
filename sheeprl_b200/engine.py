"""Dreamer-V3 update step as an explicit kernel schedule (no autograd, no torch math).

`DV3Engine.train_step` is the B200 implementation of the reference's
`sheeprl/algos/dreamer_v3/dreamer_v3.py:48-357` (`train`).  Every arithmetic operation is a call into
the C-ABI CUDA library (`include/b200rl.h`, loaded by `sheeprl_b200.lib.CudaOps`): forward, the
hand-derived backward (SURVEY.md Appendix E is the gradient-flow map it follows), global-norm clip,
Adam.  PyTorch is used only to own device memory and the CUDA stream.  Because nothing on this path
allocates, synchronises or branches on device data, the whole step is CUDA-graph capturable:
`sheeprl_b200.graph.StepGraph` captures it on the third call of the public `train()` and replays it afterwards.

Layouts (all fp32, row-major):
  * replay rows are flattened time-major: row n = t*B + b  (matches `posteriors.reshape(1,-1,Z)` in
    dreamer_v3.py:203-204), N = T*B;
  * images are channel-last `[N,H,W,C]` inside the engine (LayerNorm over C is contiguous and the
    implicit-GEMM K slices are contiguous); the CHW flatten order the reference's weights expect
    (`nn.Flatten(-3,-1)`, agent.py:90 / `Unflatten(1,(-1,4,4))`, agent.py:201) is restored by a
    batched transpose at the encoder output / decoder input;
  * latent states `[z (S*D) | h (R)]` live directly in `traj[0]` so imagination starts in place;
  * conv weights keep the reference layout: Conv2d `[Cout,Cin,4,4]`, ConvTranspose2d `[Cin,Cout,4,4]`
    — both are `[C_small_image, C_big_image, ky, kx]` for the three stride-2 kernels.
"""
from __future__ import annotations

import math
from typing import Dict, Mapping, Optional, Sequence

import torch

from sheeprl_b200.params import FlatGroup
from sheeprl_b200.lib import sync_deterministic

ACT_NONE, ACT_SILU = 0, 1
TWOHOT_LOW, TWOHOT_HIGH = -20.0, 20.0


def decoder_channels(cfg, in_channels: int, cnn_dims: Optional[Mapping[str, int]] = None) -> int:
    """Channels of the CNN decoder's output: the sum over cfg.algo.cnn_keys.decoder (CNNDecoder, agent.py:1067-1081).
    cnn_dims: {image key: channels}; not needed when the decoder's keys are the encoder's, in the same order."""
    a = cfg.algo
    dec = list(a.cnn_keys.decoder or [])
    if dec == list(a.cnn_keys.encoder or []):
        return in_channels
    missing = [k for k in dec if k not in (cnn_dims or {})]
    if missing:
        raise ValueError(f"the channel count of the decoded image key(s) {missing} is not known (pass cnn_dims)")
    return sum(int(cnn_dims[k]) for k in dec)


def check_decoder_keys(cfg) -> None:
    """The decoders reconstruct a subset of the encoded keys (the reference's main, dreamer_v3.py:413-427; its train()
    fails with a KeyError on a decoder key that is not encoded)"""
    a = cfg.algo
    for kind in ("cnn_keys", "mlp_keys"):
        enc, dec = list(a[kind].encoder or []), list(a[kind].decoder or [])
        for k in dec:
            if k not in enc:
                raise ValueError(f"{kind}.decoder: key '{k}' is not in {kind}.encoder {enc}: the decoder can only "
                                 f"reconstruct encoded keys")
        if len(set(dec)) != len(dec):
            raise ValueError(f"{kind}.decoder names a key twice: {dec}")
    if not a.cnn_keys.decoder and not a.mlp_keys.decoder:
        raise ValueError("There must be at least one decoder: cnn_keys.decoder and mlp_keys.decoder are both empty")


def dv3_param_shapes(cfg, actions_dim: Sequence[int], in_channels: int, is_continuous: bool = False,
                     mlp_dims: Optional[Mapping[str, int]] = None, cnn_dims: Optional[Mapping[str, int]] = None):
    """Shapes keyed by the reference's state-dict names (SURVEY.md §8b; built in agent.py:935-1180).
    mlp_dims: {vector observation key: dimension} for the keys of cfg.algo.mlp_keys (MLPEncoder / MLPDecoder,
    agent.py:100-152, 229-278); the CNN encoder exists only when cfg.algo.cnn_keys.encoder is not empty, the CNN / MLP
    decoder only when cfg.algo.cnn_keys.decoder / mlp_keys.decoder is not empty.  cnn_dims: {image key: channels}, for
    a CNN decoder over other keys than the encoder's (`decoder_channels`)."""
    a, w = cfg.algo, cfg.algo.world_model
    S, D = w.stochastic_size, w.discrete_size
    Z, R = S * D, w.recurrent_model.recurrent_state_size
    L = Z + R
    du, nh = a.dense_units, a.mlp_layers
    mult = w.encoder.cnn_channels_multiplier
    stages = int(round(math.log2(cfg.env.screen_size) - 2))
    A = int(sum(actions_dim))
    wm, actor, critic = {}, {}, {}

    def mlp(d, prefix, i, hidden, n_hidden, o):
        for k in range(n_hidden):
            d[f"{prefix}{3 * k}.weight"] = (hidden, i if k == 0 else hidden)
            d[f"{prefix}{3 * k + 1}.weight"] = (hidden,)
            d[f"{prefix}{3 * k + 1}.bias"] = (hidden,)
        if o is not None:
            d[f"{prefix}{3 * n_hidden}.weight"] = (o, hidden)
            d[f"{prefix}{3 * n_hidden}.bias"] = (o,)

    has_cnn = len(a.cnn_keys.encoder) > 0
    vkeys, vdims = list(a.mlp_keys.encoder), dict(mlp_dims or {})
    chans = [in_channels] + [mult * 2 ** i for i in range(stages)]
    for i in range(stages if has_cnn else 0):
        p = f"encoder.cnn_encoder.model.0._model.{3 * i}"
        wm[p + ".weight"] = (chans[i + 1], chans[i], 4, 4)
        wm[f"encoder.cnn_encoder.model.0._model.{3 * i + 1}.weight"] = (chans[i + 1],)
        wm[f"encoder.cnn_encoder.model.0._model.{3 * i + 1}.bias"] = (chans[i + 1],)
    E = chans[-1] * 16 if has_cnn else 0                     # CNN features; the vector features follow them
    Ev = w.encoder.dense_units if vkeys else 0
    if vkeys:
        mlp(wm, "encoder.mlp_encoder.model._model.", sum(vdims[k] for k in vkeys), w.encoder.dense_units,
            w.encoder.mlp_layers, None)
    dx = w.recurrent_model.dense_units
    wm["rssm.initial_recurrent_state"] = (R,)
    wm["rssm.recurrent_model.mlp._model.0.weight"] = (dx, Z + A)
    wm["rssm.recurrent_model.mlp._model.1.weight"] = (dx,)
    wm["rssm.recurrent_model.mlp._model.1.bias"] = (dx,)
    wm["rssm.recurrent_model.rnn.linear.weight"] = (3 * R, R + dx)
    wm["rssm.recurrent_model.rnn.layer_norm.weight"] = (3 * R,)
    wm["rssm.recurrent_model.rnn.layer_norm.bias"] = (3 * R,)
    # decoupled RSSM: the posterior is a function of the embedding alone (agent.py:1017-1019)
    mlp(wm, "rssm.representation_model._model.", (0 if w.decoupled_rssm else R) + E + Ev,
        w.representation_model.hidden_size, 1, Z)
    mlp(wm, "rssm.transition_model._model.", R, w.transition_model.hidden_size, 1, Z)
    has_cnn_dec = len(a.cnn_keys.decoder or []) > 0
    if has_cnn_dec:
        wm["observation_model.cnn_decoder.model.0.weight"] = (E, L)
        wm["observation_model.cnn_decoder.model.0.bias"] = (E,)
    dch = [chans[-1]] + [mult * 2 ** i for i in reversed(range(stages - 1))] + [
        decoder_channels(cfg, in_channels, cnn_dims) if has_cnn_dec else in_channels]
    for i in range(stages if has_cnn_dec else 0):
        p = f"observation_model.cnn_decoder.model.2._model.{3 * i}"
        wm[p + ".weight"] = (dch[i], dch[i + 1], 4, 4)
        if i == stages - 1:
            wm[p + ".bias"] = (dch[i + 1],)
        else:
            wm[f"observation_model.cnn_decoder.model.2._model.{3 * i + 1}.weight"] = (dch[i + 1],)
            wm[f"observation_model.cnn_decoder.model.2._model.{3 * i + 1}.bias"] = (dch[i + 1],)
    if a.mlp_keys.decoder:
        om = w.observation_model
        mlp(wm, "observation_model.mlp_decoder.model._model.", L, om.dense_units, om.mlp_layers, None)
        for i, k in enumerate(a.mlp_keys.decoder):
            wm[f"observation_model.mlp_decoder.heads.{i}.weight"] = (vdims[k], om.dense_units)
            wm[f"observation_model.mlp_decoder.heads.{i}.bias"] = (vdims[k],)
    mlp(wm, "reward_model._model.", L, du, nh, w.reward_model.bins)
    mlp(wm, "continue_model._model.", L, du, nh, 1)
    mlp(actor, "model._model.", L, du, nh, None)
    if is_continuous:      # one head: [mean | std] of every action dimension (agent.py:772)
        actor["mlp_heads.0.weight"] = (2 * A, du)
        actor["mlp_heads.0.bias"] = (2 * A,)
    else:
        for i, ad in enumerate(actions_dim):
            actor[f"mlp_heads.{i}.weight"] = (ad, du)
            actor[f"mlp_heads.{i}.bias"] = (ad,)
    mlp(critic, "_model.", L, du, nh, a.critic.bins)
    return wm, actor, critic, dict(chans=chans, dch=dch, E=E, Ev=Ev, stages=stages)


def _check_supported_modules(cfg) -> None:
    """The kernels implement the reference's default module choices (configs/algo/dreamer_v3.yaml): SiLU everywhere,
    LayerNorm after every hidden layer / conv stage, heads as wide and deep as `algo.dense_units` / `algo.mlp_layers`.
    Anything else must fail loudly instead of silently training a different network."""
    a, w = cfg.algo, cfg.algo.world_model
    blocks = {"algo": a, "encoder": w.encoder, "observation_model": w.observation_model, "reward_model": w.reward_model,
              "discount_model": w.discount_model, "transition_model": w.transition_model,
              "representation_model": w.representation_model, "recurrent_model": w.recurrent_model, "actor": a.actor,
              "critic": a.critic}
    for name, blk in blocks.items():
        for key in ("dense_act", "cnn_act"):
            v = blk.get(key, None)
            if v is not None and not str(v).endswith("SiLU"):
                raise NotImplementedError(f"{name}.{key} = {v}: only torch.nn.SiLU is built")
        for key in ("layer_norm", "mlp_layer_norm", "cnn_layer_norm"):
            v = blk.get(key, None)
            if v is not None and "LayerNorm" not in str(v.get("cls", "LayerNorm")):
                raise NotImplementedError(f"{name}.{key}.cls = {v.get('cls')}: only the LayerNorm variants are built")
    for name in ("reward_model", "discount_model"):
        blk = blocks[name]
        if int(blk.get("dense_units", a.dense_units)) != int(a.dense_units) or int(blk.get("mlp_layers", a.mlp_layers)) != int(a.mlp_layers):
            raise NotImplementedError(f"world_model.{name}: dense_units / mlp_layers must equal algo.dense_units / algo.mlp_layers")
    if int(w.observation_model.get("cnn_channels_multiplier", w.encoder.cnn_channels_multiplier)) != int(w.encoder.cnn_channels_multiplier):
        raise NotImplementedError("observation_model.cnn_channels_multiplier must equal encoder.cnn_channels_multiplier")
    for name in ("actor", "critic"):
        blk = blocks[name]
        if int(blk.get("dense_units", a.dense_units)) != int(a.dense_units) or int(blk.get("mlp_layers", a.mlp_layers)) != int(a.mlp_layers):
            raise NotImplementedError(f"algo.{name}: dense_units / mlp_layers must equal algo.dense_units / algo.mlp_layers")


FUSED_DENSE_MAX_ROWS = 4096


def dense_ln_act(ops, x, W, gamma, beta, eps, act, out, pre=None, scratch=None):
    """out = act(LayerNorm(x W^T)) (the miniblock of sheeprl/utils/model.py:34-88, bias-free Linear).  Small row counts
    (imagination steps, heads on one batch) take the two-launch fused path of csrc/gemm_tc.cu; `pre` keeps x W^T for a
    backward and may be None there.  The unfused path needs somewhere to put x W^T: `pre`, else `scratch`."""
    if x.shape[0] <= FUSED_DENSE_MAX_ROWS and ops.gemm_ln_supported(x, W):
        ops.gemm_ln_act(x, W, gamma, beta, eps, act, out, pre)
        return
    tmp = pre if pre is not None else scratch
    ops.gemm(x, W, tmp, False, True)
    ops.ln_act_fwd(tmp, gamma, beta, eps, act, out)


class _MLP:
    """n_hidden x [Linear(no bias) -> LN -> SiLU] (+ output Linear with bias): forward with saved
    pre-activations, hand-written backward.  (reference: sheeprl/models/models.py:16-119)"""

    def __init__(self, eng, group: FlatGroup, prefix: str, in_dim: int, hidden: int, n_hidden: int,
                 out_dim: Optional[int], rows: int, eps: float, tag: str, train: bool):
        self.eng, self.g, self.prefix = eng, group, prefix
        self.in_dim, self.hidden, self.n_hidden, self.out_dim, self.eps = in_dim, hidden, n_hidden, out_dim, eps
        self.rows = rows
        new = eng._buf
        self.pre = [new(f"{tag}.pre{i}", rows, hidden) for i in range(n_hidden)]
        self.act = [new(f"{tag}.act{i}", rows, hidden) for i in range(n_hidden)]
        self.out = new(f"{tag}.out", rows, out_dim) if out_dim is not None else None
        if train:
            self.dact = new(f"{tag}.dact", rows, hidden)
            self.dpre = new(f"{tag}.dpre", rows, hidden)

    def W(self, i):
        return self.g.views[f"{self.prefix}{3 * i}.weight"]

    def forward(self, x: torch.Tensor, group: Optional[FlatGroup] = None, M: Optional[int] = None):
        """x [M,in_dim] view; returns output logits (or last activation)."""
        ops = self.eng.ops
        g = group or self.g
        M = x.shape[0] if M is None else M
        cur = x
        for i in range(self.n_hidden):
            dense_ln_act(ops, cur, g.views[f"{self.prefix}{3 * i}.weight"], g.views[f"{self.prefix}{3 * i + 1}.weight"],
                         g.views[f"{self.prefix}{3 * i + 1}.bias"], self.eps, ACT_SILU, self.act[i][:M], self.pre[i][:M])
            cur = self.act[i][:M]
        if self.out_dim is None:
            return cur
        j = 3 * self.n_hidden
        ops.gemm(cur, g.views[f"{self.prefix}{j}.weight"], self.out[:M], False, True,
                 bias=g.views[f"{self.prefix}{j}.bias"])
        return self.out[:M]

    def backward(self, x: torch.Tensor, dout: torch.Tensor, dx: Optional[torch.Tensor], accumulate_dx: bool,
                 M: Optional[int] = None, data_only: bool = False, group: Optional[FlatGroup] = None):
        """dout: grad wrt output logits (or wrt last activation when out_dim is None).  Parameter grads
        are written (not accumulated) into the group's grad views; dx (+)= grad wrt x."""
        ops, g = self.eng.ops, group or self.g
        M = x.shape[0] if M is None else M
        if self.out_dim is not None:
            j = 3 * self.n_hidden
            last = self.act[-1][:M]
            if not data_only:
                ops.gemm(dout, last, g.gviews[f"{self.prefix}{j}.weight"], True, False)
                ops.col_sum(dout, g.gviews[f"{self.prefix}{j}.bias"])
            ops.gemm(dout, g.views[f"{self.prefix}{j}.weight"], self.dact[:M], False, False)
            d = self.dact[:M]
        else:
            d = dout
        for i in reversed(range(self.n_hidden)):
            ops.ln_act_bwd(self.pre[i][:M], g.views[f"{self.prefix}{3 * i + 1}.weight"],
                           g.views[f"{self.prefix}{3 * i + 1}.bias"], self.eps, ACT_SILU, d, self.dpre[:M],
                           None if data_only else g.gviews[f"{self.prefix}{3 * i + 1}.weight"],
                           None if data_only else g.gviews[f"{self.prefix}{3 * i + 1}.bias"])
            inp = x if i == 0 else self.act[i - 1][:M]
            if not data_only:
                ops.gemm(self.dpre[:M], inp, g.gviews[f"{self.prefix}{3 * i}.weight"], True, False)
            if i > 0:
                ops.gemm(self.dpre[:M], g.views[f"{self.prefix}{3 * i}.weight"], self.dact[:M], False, False)
                d = self.dact[:M]
            elif dx is not None:
                ops.gemm(self.dpre[:M], g.views[f"{self.prefix}0.weight"], dx, False, False, accumulate=accumulate_dx)


class DV3Engine:
    def __init__(self, cfg, actions_dim: Sequence[int], in_channels: int = 3, device="cuda", ops=None,
                 is_continuous: bool = False, groups=None, mlp_dims: Optional[Mapping[str, int]] = None,
                 cnn_dims: Optional[Mapping[str, int]] = None):
        """groups: optional (wm, actor, critic, target) FlatGroups to adopt instead of allocating new ones — the acting
        engine of PlayerDV3 shares the trainer's parameters this way (the reference ties `.data`, agent.py:1229-1235).
        mlp_dims: {key: dimension} of the vector observations named in cfg.algo.mlp_keys (default: cfg.env.mlp_dims).
        cnn_dims: {key: channels} of the image keys; needed only when cnn_keys.decoder differs from cnn_keys.encoder
        (default: cfg.env.cnn_channels)."""
        a, w = cfg.algo, cfg.algo.world_model
        self.is_continuous = bool(is_continuous)
        if self.is_continuous and str(cfg.distribution.get("type", "auto")).lower() not in ("auto", "scaled_normal"):
            raise NotImplementedError(
                "continuous actions: distribution.type must be auto / scaled_normal — the reference's own train() fails "
                "with tanh_normal (entropy fallback shape, dreamer_v3.py:294-297) and normal (negative scale)")
        self.decoupled = bool(w.decoupled_rssm)           # DecoupledRSSM (agent.py:501-593): z_t does not depend on h_t
        _check_supported_modules(cfg)
        if not a.cnn_keys.encoder and not a.mlp_keys.encoder:
            raise ValueError("There must be at least one encoder, both cnn and mlp encoders are None")     # models.py:420-421
        check_decoder_keys(cfg)
        actor_cls = str(a.actor.get("cls", "Actor"))
        # MinedojoActor (agent.py:848-932): the Actor's parameters; imagination takes the mode of each head and the
        # player applies the observation's action masks (PlayerDV3.get_actions)
        self.minedojo = actor_cls.endswith("MinedojoActor")
        if self.minedojo and (is_continuous or len(actions_dim) != 3 or int(actions_dim[0]) != 19):
            raise NotImplementedError(
                f"algo.actor.cls = {actor_cls}: the MineDojo actor is built for the MineDojo action space only (discrete, "
                f"three heads, 19 functional actions first), got actions_dim={tuple(actions_dim)}"
                f"{' continuous' if is_continuous else ''}")
        self.cnn_keys = list(a.cnn_keys.encoder)          # several image keys: concatenated on the channel axis (agent.py:96)
        self.has_cnn = len(self.cnn_keys) > 0
        self.vec_keys = list(a.mlp_keys.encoder)
        vd = dict(mlp_dims if mlp_dims is not None else (cfg.env.get("mlp_dims", None) or {}))
        self.vec_dims = [int(vd[k]) for k in self.vec_keys]
        self.Dv = sum(self.vec_dims)
        # decoders: a subset of the encoded keys, in their own order (heads and the CNN output split follow it)
        self.dec_cnn_keys = list(a.cnn_keys.decoder or [])
        self.has_cnn_dec = len(self.dec_cnn_keys) > 0
        self.cnn_dec_same = self.dec_cnn_keys == self.cnn_keys         # target = the encoder's input x0
        self.dec_vec_keys = list(a.mlp_keys.decoder or [])
        self.dec_vec_dims = [int(vd[k]) for k in self.dec_vec_keys]
        self.has_vec_dec = len(self.dec_vec_keys) > 0
        self.vec_dec_same = self.dec_vec_keys == self.vec_keys          # target = the encoder's input vx
        self.Dvd = sum(self.dec_vec_dims)
        self.cnn_dims = dict(cnn_dims if cnn_dims is not None else (cfg.env.get("cnn_channels", None) or {}))
        if ops is None:
            from sheeprl_b200.lib import CudaOps  # raises loudly if the extension / a GPU is missing

            ops = CudaOps(device)
        if self.minedojo and not (hasattr(ops, "minedojo_sample") and ops.minedojo_sample_supported(actions_dim)):
            raise NotImplementedError(f"the MineDojo actor's masked sample has no kernel for actions_dim={tuple(actions_dim)} "
                                      f"on the {type(ops).__name__} backend")
        self.ops = ops
        self.cfg = cfg
        self.device = torch.device(device)
        self.actions_dim = tuple(int(x) for x in actions_dim)
        self.Cin = in_channels
        self.T, self.B = a.per_rank_sequence_length, a.per_rank_batch_size
        self.N = self.T * self.B
        self.H = a.horizon
        self.S, self.D = w.stochastic_size, w.discrete_size
        self.Z, self.R = self.S * self.D, w.recurrent_model.recurrent_state_size
        self.L = self.Z + self.R
        self.Rh = 0 if self.decoupled else self.R          # h columns in front of the representation model's input
        self.A = int(sum(self.actions_dim))
        self.du, self.nh = a.dense_units, a.mlp_layers
        self.Dx = w.recurrent_model.dense_units
        self.Dt, self.Dr = w.transition_model.hidden_size, w.representation_model.hidden_size
        self.eps = float(a.mlp_layer_norm.kw.eps)
        self.ceps = float(a.cnn_layer_norm.kw.eps)
        self.unimix = float(a.unimix)
        self.img = cfg.env.screen_size
        self.key = a.cnn_keys.encoder[0] if self.has_cnn else None
        self.bins_r, self.bins_c = w.reward_model.bins, a.critic.bins
        self.Cdec = decoder_channels(cfg, in_channels, self.cnn_dims) if self.has_cnn_dec else 0
        wm_s, ac_s, cr_s, meta = dv3_param_shapes(cfg, self.actions_dim, in_channels, self.is_continuous,
                                                  dict(zip(self.vec_keys, self.vec_dims)), self.cnn_dims)
        self.Ev = meta["Ev"]                                      # width of the vector-encoder features (0: none)
        self.AW = 2 * self.A if self.is_continuous else self.A          # width of the actor head output
        self.chans, self.dch, self.E, self.stages = meta["chans"], meta["dch"], meta["E"], meta["stages"]
        if groups is not None:
            self.wm, self.actor, self.critic, self.target = groups
        else:
            self.wm = FlatGroup(wm_s, device)
            self.actor = FlatGroup(ac_s, device)
            self.critic = FlatGroup(cr_s, device)
            self.target = FlatGroup(cr_s, device, with_optimizer=False)
        self.moments_state = torch.zeros(2, dtype=torch.float32, device=device)  # (low, high)
        self.world_size = 1
        self.allreduce = None          # set by the data-parallel wrapper: fn(flat_grad_tensor)
        self.allgather = None          # fn(tensor) -> gathered tensor (Moments)
        self.allreduce_async = None    # fn(slice of a flat gradient): reduce on a side stream (parallel.py)
        self.allreduce_join = None
        self._bufs: Dict[str, torch.Tensor] = {}
        self._alloc()

    # ------------------------------------------------------------------ buffers
    def _buf(self, name: str, *shape, dtype=torch.float32) -> torch.Tensor:
        assert name not in self._bufs, name
        t = torch.zeros(*shape, dtype=dtype, device=self.device)
        self._bufs[name] = t
        return t

    def _buf_ld4(self, name: str, rows: int, cols: int) -> torch.Tensor:
        """[rows, cols] view of a buffer whose row stride is rounded up to 4 floats: gradients of the 255-bin two-hot
        logits are GEMM operands (dX = dlogits W, dW = dlogits^T act) and TMA needs 16-byte row strides — with
        ld = 255 those products fell back to the SIMT GEMM (0.4 ms / step in the ncu launch list)"""
        return self._buf(name, rows, (cols + 3) // 4 * 4)[:, :cols]

    def _alloc(self):
        N, T, B, H, Z, R, L, A, E = self.N, self.T, self.B, self.H, self.Z, self.R, self.L, self.A, self.E
        b = self._buf
        img = self.img
        n_st = self.stages if self.has_cnn else 0                # CNN encoder / decoder buffers exist only with an image key
        self.x0 = b("x0", N, img, img, self.Cin) if self.has_cnn else None
        self.enc_y, self.enc_a = [], []
        s = img
        for i in range(n_st):
            s //= 2
            self.enc_y.append(b(f"enc_y{i}", N, s, s, self.chans[i + 1]))
            self.enc_a.append(b(f"enc_a{i}", N, s, s, self.chans[i + 1]))
        self.emb = b("emb", N, E) if self.has_cnn else None
        self.pe = b("pe", N, self.Dr)
        we, wo = self.cfg.algo.world_model.encoder, self.cfg.algo.world_model.observation_model
        if self.vec_keys:
            # vector observations: vx = symlog(concat(obs_k)) is the MLP encoder's input, and the MLP decoder's target
            # when that decodes the same keys in the same order
            self.vx = b("vx", N, self.Dv)
            self.venc = _MLP(self, self.wm, "encoder.mlp_encoder.model._model.", self.Dv, we.dense_units, we.mlp_layers, None,
                             N, float(we.mlp_layer_norm.kw.eps), "venc", True)
            self.d_emb_vec = b("d_emb_vec", N, self.Ev)
        if self.has_vec_dec:
            self.vdec = _MLP(self, self.wm, "observation_model.mlp_decoder.model._model.", L, wo.dense_units, wo.mlp_layers,
                             None, N, float(wo.mlp_layer_norm.kw.eps), "vdec", True)
            self.vrecon, self.vec_rows = b("vrecon", N, self.Dvd), b("vec_rows", N)
            self.d_vdec_hidden = b("d_vdec_hidden", N, wo.dense_units)
            # symlog(concat(obs_k)) over the decoder's keys in decoder order
            self.vtgt = self.vx if self.vec_dec_same else b("vtgt", N, self.Dvd)
        self.traj = b("traj", H + 1, N, L)
        self.latent = self.traj[0]
        # scan saves
        self.z_in, self.h_in, self.a_in = b("z_in", N, Z), b("h_in", N, R), b("a_in", N, A)
        self.x_pre, self.x_act = b("x_pre", N, self.Dx), b("x_act", N, self.Dx)
        self.g_pre, self.g_ln = b("g_pre", N, 3 * R), b("g_ln", N, 3 * R)
        self.tr_pre, self.tr_act = b("tr_pre", N, self.Dt), b("tr_act", N, self.Dt)
        self.rp_pre, self.rp_act = b("rp_pre", N, self.Dr), b("rp_act", N, self.Dr)
        self.post_raw, self.prior_raw = b("post_raw", N, Z), b("prior_raw", N, Z)
        self.post_mix, self.prior_mix = b("post_mix", N, Z), b("prior_mix", N, Z)
        self.h0, self.z0 = b("h0", 1, R), b("z0", 1, Z)
        self.init_tr_pre, self.init_tr_act = b("init_tr_pre", 1, self.Dt), b("init_tr_act", 1, self.Dt)
        self.init_raw = b("init_raw", 1, Z)
        self.zero_h, self.zero_z = b("zero_h", B, R), b("zero_z", B, Z)
        self.shift_actions = b("shift_actions", N, A)
        # scan grads
        self.d_latent = b("d_latent", N, L)
        self.d_post_mix, self.d_prior_mix = b("d_post_mix", N, Z), b("d_prior_mix", N, Z)
        self.d_post_raw, self.d_prior_raw = b("d_post_raw", N, Z), b("d_prior_raw", N, Z)
        self.d_rp_act, self.d_rp_pre = b("d_rp_act", N, self.Dr), b("d_rp_pre", N, self.Dr)
        self.d_tr_act, self.d_tr_pre = b("d_tr_act", N, self.Dt), b("d_tr_pre", N, self.Dt)
        self.d_g_ln, self.d_g_pre = b("d_g_ln", N, 3 * R), b("d_g_pre", N, 3 * R)
        self.d_x_act, self.d_x_pre = b("d_x_act", N, self.Dx), b("d_x_pre", N, self.Dx)
        self.dz_carry, self.dh_carry = b("dz_carry", B, Z), b("dh_carry", B, R)
        self.dz_tot, self.dh_tot = b("dz_tot", B, Z), b("dh_tot", B, R)
        self.dh_in, self.dz_in = b("dh_in", B, R), b("dz_in", B, Z)
        self.d_h0 = b("d_h0", R)
        self.kl_rows = b("kl_rows", N, 4)
        self.dec_y, self.dec_a, self.d_dec_a, self.d_enc_a = [], [], [], []
        if self.has_cnn:
            self.d_emb = b("d_emb", N, E)
        if self.has_cnn_dec:
            # decoder
            self.dec_lin = b("dec_lin", N, E)
            C0 = self.dch[0]
            self.dec_in = b("dec_in", N, 4, 4, C0)
            s = 4
            for i in range(self.stages - 1):
                s *= 2
                self.dec_y.append(b(f"dec_y{i}", N, s, s, self.dch[i + 1]))
                self.dec_a.append(b(f"dec_a{i}", N, s, s, self.dch[i + 1]))
            self.recon = b("recon", N, img, img, self.Cdec)
            self.d_dec_in = b("d_dec_in", N, 4, 4, C0)
            self.d_dec_lin = b("d_dec_lin", N, E)
            self.d_dec_a = [b(f"d_dec_a{i}", *self.dec_a[i].shape) for i in range(self.stages - 1)]
            # the decoder's target: the encoder's input, else the normalised pixels of the decoder's keys
            self.x_dec = self.x0 if self.cnn_dec_same else b("x_dec", N, img, img, self.Cdec)
        if self.has_cnn:
            self.d_enc_a = [b(f"d_enc_a{i}", *self.enc_a[i].shape) for i in range(self.stages)]
        # losses
        self.obs_rows, self.rew_rows, self.cont_rows = b("obs_rows", N), b("rew_rows", N), b("cont_rows", N)
        self.metrics = b("metrics", 16)
        self.normsq = {k: self._buf(f"normsq_{k}", (), dtype=torch.float64) for k in ("wm", "actor", "critic")}
        self.norms = b("norms", 3)
        # heads on the replay batch (world-model phase)
        self.reward_wm = _MLP(self, self.wm, "reward_model._model.", L, self.du, self.nh, self.bins_r, N, self.eps,
                              "rew", True)
        self.cont_wm = _MLP(self, self.wm, "continue_model._model.", L, self.du, self.nh, 1, N, self.eps, "cont", True)
        self.d_rew_logits, self.d_cont_logit = self._buf_ld4("d_rew_logits", N, self.bins_r), b("d_cont_logit", N, 1)
        # behaviour phase
        M1 = (H + 1) * N
        self.actions = b("img_actions", H + 1, N, A)
        self.actor_mlp = _MLP(self, self.actor, "model._model.", L, self.du, self.nh, None, M1, self.eps, "actor", True)
        self.actor_raw = b("actor_raw", M1, self.AW)
        self.d_actor_raw = b("d_actor_raw", H * N, self.AW)
        self.d_actor_hidden = b("d_actor_hidden", H * N, self.du)
        self.critic_mlp = _MLP(self, self.critic, "_model.", L, self.du, self.nh, self.bins_c, M1, self.eps,
                               "critic", True)
        self.target_mlp = _MLP(self, self.target, "_model.", L, self.du, self.nh, self.bins_c, H * N, self.eps,
                               "target", False)
        self.rew_img = _MLP(self, self.wm, "reward_model._model.", L, self.du, self.nh, self.bins_r, M1, self.eps,
                            "rew_img", self.is_continuous)     # continuous actions back-propagate through this head
        self.cont_img = _MLP(self, self.wm, "continue_model._model.", L, self.du, self.nh, 1, M1, self.eps,
                             "cont_img", False)
        self.values, self.rew_pred = b("values", H + 1, N), b("rew_pred", H + 1, N)
        self.target_values = b("target_values", H * N)
        self.true_cont = b("true_cont", N)
        self.lam, self.discount = b("lam", H, N), b("discount", H + 1, N)
        self.moments_out = b("moments_out", 2)
        self.policy_rows = b("policy_rows", H * N)
        self.value_rows = b("value_rows", H * N)
        self.d_critic_logits = self._buf_ld4("d_critic_logits", H * N, self.bins_c)
        # imagination step scratch (N rows)
        self.i_x_pre = b("i_x_pre", N, self.Dx)
        # imagination keeps the GRU input [h | x] contiguous so that its Linear is ONE product (weights are [h, x] ordered)
        self.i_hx = b("i_hx", N, self.R + self.Dx)
        self.i_x_act = self.i_hx[:, self.R:]
        self.i_g_pre, self.i_g_ln = b("i_g_pre", N, 3 * R), b("i_g_ln", N, 3 * R)
        self.i_tr_pre, self.i_tr_act = b("i_tr_pre", N, self.Dt), b("i_tr_act", N, self.Dt)
        self.i_raw = b("i_raw", N, Z)
        if self.is_continuous:
            # the policy gradient flows back through the rollout (dreamer_v3.py:283-284): every step's activations
            # are kept, plus the gradient buffers of the data-only BPTT
            self.c_x_pre, self.c_hx = b("c_x_pre", H, N, self.Dx), b("c_hx", H, N, self.R + self.Dx)
            self.c_g_pre, self.c_g_ln = b("c_g_pre", H, N, 3 * R), b("c_g_ln", H, N, 3 * R)
            self.c_tr_pre, self.c_tr_act = b("c_tr_pre", H, N, self.Dt), b("c_tr_act", H, N, self.Dt)
            self.c_raw = b("c_raw", H, N, Z)
            self.act_ent = b("act_ent", M1)
            self.d_values, self.d_rew = b("d_values", H + 1, N), b("d_rew", H + 1, N)
            self.d_v_logits = self._buf_ld4("d_v_logits", M1, self.bins_c)
            self.d_r_logits = self._buf_ld4("d_r_logits", M1, self.bins_r)
            self.d_traj = b("d_traj", H + 1, N, L)
            self.cd_raw = b("cd_raw", N, Z)
            self.cd_tr_act, self.cd_tr_pre = b("cd_tr_act", N, self.Dt), b("cd_tr_pre", N, self.Dt)
            self.cd_g_ln, self.cd_g_pre = b("cd_g_ln", N, 3 * R), b("cd_g_pre", N, 3 * R)
            self.cd_x_act, self.cd_x_pre = b("cd_x_act", N, self.Dx), b("cd_x_pre", N, self.Dx)
            self.cd_dz, self.cd_dh = b("cd_dz", N, Z), b("cd_dh", N, R)
            self.cd_dz_carry, self.cd_dh_carry = b("cd_dz_carry", N, Z), b("cd_dh_carry", N, R)
            self.cd_a = b("cd_a", N, A)
        # default noise buffers (production: filled by the Philox kernel each step)
        self.noise_post = b("noise_post", T, B, Z)
        self.noise_img_state = b("noise_img_state", H, N, Z)
        self.noise_img_action = b("noise_img_action", H + 1, N, A)
        self.rng_seed = int(self.cfg.get("seed", 0) or 0)      # build_agent folds the rank in (agent.py)
        self.rng_t = torch.zeros(1, dtype=torch.int32, device=self.device)   # device-side step counter for Philox
        self.cuda_graph = bool(self.cfg.algo.get("cuda_graph", True))  # B200 knob: replay the update as one CUDA graph
        # the reference applies cfg.float32_matmul_precision with torch.set_float32_matmul_precision (cli.py:186;
        # configs/config.yaml:18 defaults to "high" = TF32 products).  Here the key is honoured when PRESENT; without it the
        # products stay fp32-accurate (3xTF32), which is what the 1e-4 parity contract is stated for.
        prec = self.cfg.get("float32_matmul_precision", None)
        if prec is not None and hasattr(self.ops, "set_matmul_precision"):
            self.ops.set_matmul_precision(str(prec))
        self._graph = None
        # persistent fused RSSM scan (csrc/rssm_scan.cu) when the ops backend has it and the model is inside the kernels'
        # envelope; the backward kernel needs more shared memory than the forward, so it can be refused alone
        # (decoupled RSSM: the GRU-only scan kernels of the same file, with their own envelope)
        if self.decoupled:
            has_scan, dims = hasattr(self.ops, "gru_scan_fwd"), self._gru_scan_dims()
            self.fused_scan = has_scan and self.ops.gru_scan_supported(dims, backward=False)
            self.fused_scan_bwd = has_scan and self.ops.gru_scan_supported(dims, backward=True)
        else:
            has_scan, dims = hasattr(self.ops, "rssm_scan_fwd"), self._scan_dims()
            self.fused_scan = has_scan and self.ops.rssm_scan_supported(dims, backward=False)
            self.fused_scan_bwd = has_scan and self.ops.rssm_scan_supported(dims, backward=True)
        self._scan_ws = None
        self._scan_q = None

    # ------------------------------------------------------------------ CUDA-graph replay of the step
    def optimizer_groups(self):
        return [self.wm, self.actor, self.critic]

    def use_cuda_graph(self) -> bool:
        return self.cuda_graph and self.device.type == "cuda" and type(self.ops).__name__ == "CudaOps"

    def graph_key(self) -> tuple:
        """what a captured step bakes in besides the batch shapes: the learning rates and weight decays (kernel arguments
        by value), the matmul precision and the deterministic mode (which kernels run)"""
        prec = self.ops.matmul_precision() if hasattr(self.ops, "matmul_precision") else "highest"
        return tuple((float(g.optimizer.lr), g.adam_kwargs().get("weight_decay", 0.0))
                     if getattr(g, "optimizer", None) is not None else -1.0 for g in self.optimizer_groups()) + (
                         prec, "deterministic" if torch.are_deterministic_algorithms_enabled() else "default")

    def step_graph(self):
        if self._graph is None:
            from sheeprl_b200.graph import StepGraph

            groups = self.optimizer_groups()

            def bump():
                for g in groups:
                    g.step += 1

            self._graph = StepGraph(self.device, warmup=2, on_replay=bump,
                                    host_state=(lambda: [g.step for g in groups],
                                                lambda s: [setattr(g, "step", v) for g, v in zip(groups, s)]))
        return self._graph

    def rng_state(self) -> Dict[str, torch.Tensor]:
        """Philox position of the sampling noise (saved with the optimizer state so a resumed run continues the stream)"""
        return {"rng_t": self.rng_t.detach().clone().cpu(), "rng_seed": torch.tensor(self.rng_seed)}

    def load_rng_state(self, st) -> None:
        self.rng_t.copy_(st["rng_t"].to(self.rng_t.device))
        self.rng_seed = int(st["rng_seed"])

    def bytes_allocated(self) -> int:
        tot = sum(t.numel() * t.element_size() for t in self._bufs.values())
        for g in (self.wm, self.actor, self.critic):
            tot += 4 * g.numel * 4
        return tot + self.target.numel * 4

    # ------------------------------------------------------------------ parameter name helpers
    def _w(self, name):
        return self.wm.views[name]

    def _gw(self, name):
        return self.wm.gviews[name]

    # ------------------------------------------------------------------ the step
    def train_step(self, data: Dict[str, torch.Tensor], noise: Optional[Dict[str, torch.Tensor]] = None):
        """data: the reference's batch dict ([T,B,...]; image key uint8 or float 0..255).
        noise: optional injected Exp(1) noise {"post":[T,B,S,D], "img_state":[H,N,S,D],
        "img_action":[list per head of [H+1,N,A_h]]} (parity mode); None -> on-device Philox."""
        sync_deterministic(self.ops)
        self._draw_noise(noise)
        self._world_model_phase(data)
        # ---- behaviour learning with the updated world model
        self._imagine()
        self._behaviour_losses()
        return self.metrics

    def _draw_noise(self, noise: Optional[Dict[str, torch.Tensor]]):
        ops = self.ops
        T, B, N, H, Z = self.T, self.B, self.N, self.H, self.Z
        if noise is None:
            ops.increment(self.rng_t)
            ops.fill_exponential(self.noise_post.view(-1), self.rng_seed, 0, self.rng_t)
            ops.fill_exponential(self.noise_img_state.view(-1), self.rng_seed, 1, self.rng_t)
            if not self.minedojo:          # the MineDojo actor imagines the mode of each head: no action noise
                fill = ops.fill_normal if self.is_continuous else ops.fill_exponential
                fill(self.noise_img_action.view(-1), self.rng_seed, 2, self.rng_t)
        else:
            self.noise_post.copy_(noise["post"].reshape(T, B, Z))
            self.noise_img_state.copy_(noise["img_state"].reshape(H, N, Z))
            if not self.minedojo:
                self.noise_img_action.copy_(torch.cat([x for x in noise["img_action"]], -1))

    def _world_model_phase(self, data: Dict[str, torch.Tensor], heads_detached: bool = False):
        """Dynamic learning (dreamer_v3.py:98-200): forward, losses, backward, clip + Adam of the world model.
        heads_detached: the reward / continue losses do not reach the latent state (Plan2Explore feeds those heads
        `latent_states.detach()`, p2e_dv3_exploration.py:157,160)."""
        ops = self.ops
        B, N, R, A = self.B, self.N, self.R, self.A
        w = self.cfg.algo.world_model
        # ---- inputs (dreamer_v3.py:98-104): normalise pixels, force is_first[0]=1, shift actions
        if self.has_cnn:
            ops.obs_prep(self.image_batch(data, N), self.x0)
        off = 0
        for k, d in zip(self.vec_keys, self.vec_dims):       # symlog squashing (MLPEncoder.forward, agent.py:150)
            ops.symlog(data[k].reshape(N, d), self.vx[:, off:off + d])
            off += d
        if self.has_cnn_dec and not self.cnn_dec_same:
            ops.obs_prep(self.image_batch(data, N, self.dec_cnn_keys), self.x_dec)
        if self.has_vec_dec and not self.vec_dec_same:
            off = 0
            for k, d in zip(self.dec_vec_keys, self.dec_vec_dims):
                ops.symlog(data[k].reshape(N, d), self.vtgt[:, off:off + d])
                off += d
        data["is_first"][0].fill_(1.0)                      # same in-place mutation as the reference (:100)
        first = data["is_first"].reshape(N)
        ops.zero(self.shift_actions[:B])
        ops.copy(data["actions"].reshape(N, A)[: N - B], self.shift_actions[B:])
        rewards = data["rewards"].reshape(N)
        ops.affine(data["terminated"].reshape(N), self.true_cont, -1.0, 1.0)   # 1 - terminated

        self._encoder_forward()
        # embed part of the representation model's first layer, for all T at once (no recurrence in it)
        # (decoupled RSSM: that share is the whole first product)
        self._project_embedding(self.rp_pre if self.decoupled else self.pe)
        self._scan_forward(first)
        self._decoder_forward()
        rew_logits = self.reward_wm.forward(self.latent)
        cont_logit = self.cont_wm.forward(self.latent)

        # ---- losses + seed gradients (loss.py:9-88); mean over T*B
        inv = 1.0 / N
        if self.has_cnn_dec:
            # MSEDistribution per decoded key (loss.py:61): the per-key sums add up to one sum over the channels
            P = self.img * self.img * self.Cdec
            ops.mse_loss_grad(self.recon.view(N, P), self.x_dec.view(N, P), inv, self.obs_rows, self.recon.view(N, P))
        if self.has_vec_dec:
            # SymlogDistribution (utils/distribution.py:177-192): squared error against symlog(obs), summed over keys and
            # dims (its `tol` = 1e-8 cut on the squared distance is not reproduced: |effect| < 1e-8 per element)
            rows = self.vec_rows if self.has_cnn_dec else self.obs_rows
            ops.mse_loss_grad(self.vrecon, self.vtgt, inv, rows, self.vrecon)
            if self.has_cnn_dec:
                ops.axpy(self.vec_rows, self.obs_rows)
        ops.twohot_loss_grad(rew_logits, rewards, None, inv, TWOHOT_LOW, TWOHOT_HIGH, self.rew_rows, self.d_rew_logits)
        ops.bce_loss_grad(cont_logit, self.true_cont, float(w.continue_scale_factor), inv, self.cont_rows,
                          self.d_cont_logit)
        ops.kl_loss_grad(self.post_mix, self.prior_mix, self.S, self.D, float(w.kl_dynamic),
                         float(w.kl_representation), float(w.kl_free_nats), float(w.kl_regularizer), inv,
                         self.d_post_mix, self.d_prior_mix, self.kl_rows)
        # metrics 0..7: wm_loss, obs, reward, state, continue, kl, post_ent, prior_ent
        ops.sum_rows(self.obs_rows.view(N, 1), self.metrics[1:2], inv)
        ops.sum_rows(self.rew_rows.view(N, 1), self.metrics[2:3], inv)
        ops.sum_rows(self.cont_rows.view(N, 1), self.metrics[4:5], inv)
        ops.sum_rows(self.kl_rows[:, 1:2], self.metrics[3:4], inv)
        ops.sum_rows(self.kl_rows[:, 0:1], self.metrics[5:6], inv)
        ops.sum_rows(self.kl_rows[:, 2:4], self.metrics[6:8], inv)
        ops.zero(self.metrics[0:1])
        ops.axpy(self.metrics[1:2], self.metrics[0:1])
        ops.axpy(self.metrics[2:3], self.metrics[0:1])
        ops.axpy(self.metrics[3:4], self.metrics[0:1], float(w.kl_regularizer))
        ops.axpy(self.metrics[4:5], self.metrics[0:1])

        # ---- world-model backward
        ops.zero(self.wm.grad)
        self._decoder_backward()                                       # writes d_latent
        self.reward_wm.backward(self.latent, self.d_rew_logits, None if heads_detached else self.d_latent, True)
        self.cont_wm.backward(self.latent, self.d_cont_logit, None if heads_detached else self.d_latent, True)
        # data parallel: the flat gradient is laid out encoder | rssm | decoder, reward, continue, and the backward
        # finishes those three ranges in REVERSE order, so each is all-reduced on a side stream as soon as it is final
        # (the reference's DDP buckets, fabric.backward dreamer_v3.py:191, overlap the same way)
        b_enc, b_tail = self._wm_buckets()
        # default: overlap unless the persistent scan kernels run — they hold 128 of the 132 SMs with all of their shared
        # memory, NCCL's CTAs then only fit on the other 20 and the reductions get slower than one call in front of the
        # optimizer (measured at 2 GPUs: 16.96 vs 16.73 ms / step); per-step scans (XL) leave room and overlap pays
        overlap = self.allreduce_async is not None and bool(self.cfg.algo.get("overlap_allreduce", not self.fused_scan))
        if overlap:
            self.allreduce_async(self.wm.grad[b_tail:])
        self._scan_backward(first)
        if overlap:
            self.allreduce_async(self.wm.grad[b_enc:b_tail])
        self._encoder_backward()
        if overlap:
            self.allreduce_async(self.wm.grad[:b_enc])
            self.allreduce_join()
        self._optimizer_step("wm", self.wm, float(w.clip_gradients or 0.0), w.optimizer, 0, reduced=overlap)

    # ------------------------------------------------------------------ encoder / decoder
    def _enc_names(self, i):
        p = "encoder.cnn_encoder.model.0._model."
        return f"{p}{3 * i}.weight", f"{p}{3 * i + 1}.weight", f"{p}{3 * i + 1}.bias"

    def _dec_names(self, i):
        p = "observation_model.cnn_decoder.model.2._model."
        return f"{p}{3 * i}.weight", f"{p}{3 * i + 1}.weight", f"{p}{3 * i + 1}.bias"

    def image_batch(self, obs: Dict[str, torch.Tensor], rows: int, keys: Optional[Sequence[str]] = None) -> torch.Tensor:
        """[rows, C, H, W] pixels (uint8 or float) of the image key(s) (default: the encoder's); more than one key is
        concatenated on the channel axis, as CNNEncoder.forward does on every call (agent.py:96) — a device copy, no
        arithmetic.  `keys`: the CNN decoder's keys, whose concatenation is its target."""
        keys = self.cnn_keys if keys is None else keys
        C = self.Cin if keys is self.cnn_keys else self.Cdec
        imgs = [obs[k].reshape(rows, -1, self.img, self.img) for k in keys]
        if len(imgs) == 1:
            return imgs[0]
        if any(t.dtype != imgs[0].dtype for t in imgs):
            imgs = [t.float() for t in imgs]
        out = torch.cat(imgs, 1)
        assert out.shape[1] == C, f"image keys {keys} carry {out.shape[1]} channels, the network was built for {C}"
        return out

    def _project_embedding(self, out: torch.Tensor):
        """out = embed W_r1[:, Rh:]^T with embed = [cnn features | vector features] (MultiEncoder, models.py:466-475); the
        two feature blocks stay in their own buffers and meet in this product"""
        ops, R, E = self.ops, self.Rh, self.E
        Wr1 = self._w("rssm.representation_model._model.0.weight")
        if self.has_cnn:
            ops.gemm(self.emb, Wr1[:, R:R + E], out, False, True)
        if self.vec_keys:
            ops.gemm(self.venc.act[-1], Wr1[:, R + E:], out, False, True, accumulate=self.has_cnn)

    def _encoder_forward(self):
        ops = self.ops
        if self.vec_keys:
            self.venc.forward(self.vx)
        if not self.has_cnn:
            return
        cur = self.x0
        for i in range(self.stages):
            wn, gn, bn = self._enc_names(i)
            ops.conv_down(cur, self._w(wn), self.enc_y[i])
            C = self.chans[i + 1]
            ops.ln_act_fwd(self.enc_y[i].view(-1, C), self._w(gn), self._w(bn), self.ceps, ACT_SILU,
                           self.enc_a[i].view(-1, C))
            cur = self.enc_a[i]
        C = self.chans[-1]
        ops.transpose_batched(cur.view(self.N, 16, C), self.emb.view(self.N, C, 16))

    def _encoder_backward(self):
        """d_emb [N,E] (CHW order) -> conv weight / LN grads; d_emb_vec -> vector-encoder grads."""
        ops = self.ops
        if self.vec_keys:
            self.venc.backward(self.vx, self.d_emb_vec, None, False)
        if not self.has_cnn:
            return
        C = self.chans[-1]
        ops.transpose_batched(self.d_emb.view(self.N, C, 16), self.d_enc_a[-1].view(self.N, 16, C))
        for i in reversed(range(self.stages)):
            wn, gn, bn = self._enc_names(i)
            C = self.chans[i + 1]
            d = self.d_enc_a[i].view(-1, C)
            ops.ln_act_bwd(self.enc_y[i].view(-1, C), self._w(gn), self._w(bn), self.ceps, ACT_SILU, d, d,
                           self._gw(gn), self._gw(bn))
            inp = self.x0 if i == 0 else self.enc_a[i - 1]
            ops.conv_wgrad(self.d_enc_a[i], inp, self._gw(wn))
            if i > 0:
                ops.conv_up(self.d_enc_a[i], self._w(wn), self.d_enc_a[i - 1])

    def _vec_heads(self):
        """[(head weight name, column offset, width)] of the MLP decoder's per-key output layers"""
        out, off = [], 0
        for i, d in enumerate(self.dec_vec_dims):
            out.append((f"observation_model.mlp_decoder.heads.{i}", off, d))
            off += d
        return out

    def _decoder_forward(self):
        ops = self.ops
        if self.has_vec_dec:
            hid = self.vdec.forward(self.latent)
            for name, off, d in self._vec_heads():
                ops.gemm(hid, self._w(name + ".weight"), self.vrecon[:, off:off + d], False, True, bias=self._w(name + ".bias"))
        if not self.has_cnn_dec:
            return
        p = "observation_model.cnn_decoder.model."
        ops.gemm(self.latent, self._w(p + "0.weight"), self.dec_lin, False, True, bias=self._w(p + "0.bias"))
        C0 = self.dch[0]
        ops.transpose_batched(self.dec_lin.view(self.N, C0, 16), self.dec_in.view(self.N, 16, C0))
        cur = self.dec_in
        for i in range(self.stages - 1):
            wn, gn, bn = self._dec_names(i)
            C = self.dch[i + 1]
            ops.conv_up(cur, self._w(wn), self.dec_y[i])
            ops.ln_act_fwd(self.dec_y[i].view(-1, C), self._w(gn), self._w(bn), self.ceps, ACT_SILU,
                           self.dec_a[i].view(-1, C))
            cur = self.dec_a[i]
        wn = self._dec_names(self.stages - 1)[0]
        ops.conv_up(cur, self._w(wn), self.recon, bias=self._w(wn.replace(".weight", ".bias")))

    def _decoder_backward(self):
        """self.recon / self.vrecon hold d(loss)/d(reconstruction) (written in place by mse_loss_grad). Writes d_latent:
        the first decoder writes it, the second accumulates."""
        ops = self.ops
        if self.has_cnn_dec:
            self._cnn_decoder_backward()
        if self.has_vec_dec:
            hid = self.vdec.act[-1]
            ops.zero(self.d_vdec_hidden)
            for name, off, d in self._vec_heads():
                dv = self.vrecon[:, off:off + d]
                ops.gemm(dv, hid, self._gw(name + ".weight"), True, False)
                ops.col_sum(dv, self._gw(name + ".bias"))
                ops.gemm(dv, self._w(name + ".weight"), self.d_vdec_hidden, False, False, accumulate=True)
            self.vdec.backward(self.latent, self.d_vdec_hidden, self.d_latent, self.has_cnn_dec)

    def _cnn_decoder_backward(self):
        ops = self.ops
        st = self.stages
        wn = self._dec_names(st - 1)[0]
        d_big = self.recon
        ops.col_sum(d_big.view(-1, self.Cdec), self._gw(wn.replace(".weight", ".bias")))
        for i in reversed(range(st)):
            wn, gn, bn = self._dec_names(i)
            inp = self.dec_in if i == 0 else self.dec_a[i - 1]
            d_inp = self.d_dec_in if i == 0 else self.d_dec_a[i - 1]
            ops.conv_wgrad(inp, d_big, self._gw(wn))
            ops.conv_down(d_big, self._w(wn), d_inp)
            if i > 0:
                gn_p, bn_p = self._dec_names(i - 1)[1:]
                C = self.dch[i]
                d = d_inp.view(-1, C)
                ops.ln_act_bwd(self.dec_y[i - 1].view(-1, C), self._w(gn_p), self._w(bn_p), self.ceps, ACT_SILU, d, d,
                               self._gw(gn_p), self._gw(bn_p))
            d_big = d_inp
        C0 = self.dch[0]
        ops.transpose_batched(self.d_dec_in.view(self.N, 16, C0), self.d_dec_lin.view(self.N, C0, 16))
        p = "observation_model.cnn_decoder.model."
        ops.gemm(self.d_dec_lin, self.latent, self._gw(p + "0.weight"), True, False)
        ops.col_sum(self.d_dec_lin, self._gw(p + "0.bias"))
        ops.gemm(self.d_dec_lin, self._w(p + "0.weight"), self.d_latent, False, False)

    # ------------------------------------------------------------------ RSSM pieces
    def _recurrent_forward(self, z, act, h_prev, x_pre, x_act, g_pre, g_ln, h_out, win_t=None, hx=None, h_next=None,
                           keep: bool = True):
        """RecurrentModel + LayerNormGRUCell on M rows (agent.py:328-341, models.py:396-403).  `win_t`: transposed
        first-layer weight; given only when z is an exact one-hot sample (imagination), the product becomes a gather.
        `keep`: pre-activations are needed by a backward (x_pre / g_pre / g_ln are written); `h_next`: optional second
        destination of the new h.  Returns True when `h_next` was written."""
        self._recurrent_input(z, act, x_pre, x_act, win_t, keep)
        return self._gru_forward(h_prev, x_act, g_pre, g_ln, h_out, hx, h_next, keep)

    def _recurrent_input(self, z, act, x_pre, x_act, win_t=None, keep: bool = True):
        """x = SiLU(LN(W_in [z, a])) (RecurrentModel.mlp, agent.py:328-341)"""
        ops, Z = self.ops, self.Z
        p = "rssm.recurrent_model."
        Win = self._w(p + "mlp._model.0.weight")
        fused_x = win_t is not None and ops.onehot_linear_ln_supported(win_t, x_act, x_pre if keep else None)
        if fused_x:
            ops.onehot_linear_ln(z, act, win_t, self._w(p + "mlp._model.1.weight"), self._w(p + "mlp._model.1.bias"),
                                 self.eps, x_act, self.S, self.D, pre=x_pre if keep else None)
        elif win_t is not None:
            ops.onehot_linear(z, act, win_t, x_pre, self.S, self.D)
        else:
            ops.gemm(z, Win[:, :Z], x_pre, False, True)
            ops.gemm(act, Win[:, Z:], x_pre, False, True, accumulate=True)
        if not fused_x:
            ops.ln_act_fwd(x_pre, self._w(p + "mlp._model.1.weight"), self._w(p + "mlp._model.1.bias"), self.eps,
                           ACT_SILU, x_act)

    def _gru_forward(self, h_prev, x_act, g_pre, g_ln, h_out, hx=None, h_next=None, keep: bool = True):
        """LayerNormGRUCell (models.py:396-403).  `x_act` None: g_pre already holds x's share of the product (decoupled
        RSSM: x is known for every step up front), h's share is added to it."""
        ops, R = self.ops, self.R
        p = "rssm.recurrent_model."
        Wg = self._w(p + "rnn.linear.weight")
        if hx is not None and hx.shape[0] <= FUSED_DENSE_MAX_ROWS and ops.gemm_ln_supported(hx, Wg, 1):
            # product + split-K sum + LayerNorm + gate in two launches; the new h also lands in `h_next` (the next
            # step's [h | x] input)
            ops.gemm_ln_gru(hx, Wg, self._w(p + "rnn.layer_norm.weight"), self._w(p + "rnn.layer_norm.bias"), self.eps,
                            h_prev, h_out, h_next, g_pre if keep else None, g_ln if keep else None)
            return True
        if hx is not None:                                   # [h | x] contiguous (x_act is its right half)
            ops.gemm(hx, Wg, g_pre, False, True)
        else:
            ops.gemm(h_prev, Wg[:, :R], g_pre, False, True, accumulate=x_act is None)
            if x_act is not None:
                ops.gemm(x_act, Wg[:, R:], g_pre, False, True, accumulate=True)
        ops.ln_act_fwd(g_pre, self._w(p + "rnn.layer_norm.weight"), self._w(p + "rnn.layer_norm.bias"), self.eps,
                       ACT_NONE, g_ln)
        ops.gru_gate_fwd(g_ln, h_prev, h_out)
        return False

    def _recurrent_backward(self, g_ln, h_prev, g_pre, x_pre, dh, d_g_ln, d_g_pre, d_x_act, d_x_pre, dh_prev, dz,
                            da=None):
        """Data-gradient backward of `_recurrent_forward` (its parameter gradients are batched products of the caller):
        dh, the gradient of the new h -> dh_prev (gradient of h_prev) and dz (of z); `da`: also the gradient of the
        action columns."""
        ops, Z, R = self.ops, self.Z, self.R
        p = "rssm.recurrent_model."
        Win, Wg = self._w(p + "mlp._model.0.weight"), self._w(p + "rnn.linear.weight")
        self._gru_backward(g_ln, h_prev, g_pre, dh, d_g_ln, d_g_pre, dh_prev)
        ops.gemm(d_g_pre, Wg[:, R:], d_x_act, False, False)
        ops.ln_act_bwd(x_pre, self._w(p + "mlp._model.1.weight"), self._w(p + "mlp._model.1.bias"), self.eps, ACT_SILU,
                       d_x_act, d_x_pre, None, None)
        ops.gemm(d_x_pre, Win[:, :Z], dz, False, False)
        if da is not None:
            ops.gemm(d_x_pre, Win[:, Z:], da, False, False)

    def _gru_backward(self, g_ln, h_prev, g_pre, dh, d_g_ln, d_g_pre, dh_prev):
        """Data-gradient backward of `_gru_forward` with respect to h_prev: dh -> d_g_ln, d_g_pre, dh_prev"""
        ops = self.ops
        p = "rssm.recurrent_model.rnn."
        ops.gru_gate_bwd(g_ln, h_prev, dh, d_g_ln, dh_prev)
        ops.ln_act_bwd(g_pre, self._w(p + "layer_norm.weight"), self._w(p + "layer_norm.bias"), self.eps, ACT_NONE,
                       d_g_ln, d_g_pre, None, None)
        ops.gemm(d_g_pre, self._w(p + "linear.weight")[:, :self.R], dh_prev, False, False, accumulate=True)

    def _transition_forward(self, h, tr_pre, tr_act, raw, keep: bool = True):
        ops = self.ops
        p = "rssm.transition_model._model."
        dense_ln_act(ops, h, self._w(p + "0.weight"), self._w(p + "1.weight"), self._w(p + "1.bias"), self.eps, ACT_SILU,
                     tr_act, tr_pre if keep else None, scratch=tr_pre)
        ops.gemm(tr_act, self._w(p + "3.weight"), raw, False, True, bias=self._w(p + "3.bias"))

    def _transition_backward(self, raw, tr_pre, dz, dmix, d_raw, d_tr_act, d_tr_pre, dh, ln_grads: bool = False):
        """Backward of `_transition_forward` and the categorical sample of its logits `raw`: the straight-through `dz`
        and / or the unimix log-probabilities' `dmix` -> d_raw -> dh += gradient of h.  `ln_grads`: also write the
        LayerNorm parameter gradients (the products' weight gradients are the caller's)."""
        ops = self.ops
        p = "rssm.transition_model._model."
        ops.cat_sample_bwd(raw, dz, dmix, self.unimix, self.S, self.D, d_raw)
        ops.gemm(d_raw, self._w(p + "3.weight"), d_tr_act, False, False)
        ops.ln_act_bwd(tr_pre, self._w(p + "1.weight"), self._w(p + "1.bias"), self.eps, ACT_SILU, d_tr_act, d_tr_pre,
                       self._gw(p + "1.weight") if ln_grads else None, self._gw(p + "1.bias") if ln_grads else None)
        ops.gemm(d_tr_pre, self._w(p + "0.weight"), dh, False, False, accumulate=True)

    def _posterior_forward(self, h, rp_pre, rp_act, raw, noise, z_out, mix_out=None):
        """Representation model on [h | embed] and its sample z_out (agent.py:451-465).  `rp_pre` holds the embedding's
        share of the first product on entry (`_project_embedding`); h's share is added to it (decoupled RSSM,
        agent.py:582-593: there is none and `h` is None)."""
        ops, R = self.ops, self.R
        pr = "rssm.representation_model._model."
        if h is not None:
            ops.gemm(h, self._w(pr + "0.weight")[:, :R], rp_pre, False, True, accumulate=True)
        ops.ln_act_fwd(rp_pre, self._w(pr + "1.weight"), self._w(pr + "1.bias"), self.eps, ACT_SILU, rp_act)
        ops.gemm(rp_act, self._w(pr + "3.weight"), raw, False, True, bias=self._w(pr + "3.bias"))
        ops.cat_sample(raw, noise, self.unimix, self.S, self.D, z_out, mix_out)

    def _scan_forward(self, first: torch.Tensor):
        """64-step RSSM scan (dreamer_v3.py:131-145, agent.py:396-435): the posterior recurrence, then the prior of
        every step off the recurrence."""
        ops, B, Z, R = self.ops, self.B, self.Z, self.R
        # learned initial state, identical for every row and step (agent.py:391-394)
        ops.tanh_fwd(self._w("rssm.initial_recurrent_state").view(1, R), self.h0)
        self._transition_forward(self.h0, self.init_tr_pre, self.init_tr_act, self.init_raw)
        ops.cat_sample(self.init_raw, None, self.unimix, self.S, self.D, self.z0)
        if self.decoupled:
            self._scan_forward_decoupled(first)
        elif self.fused_scan:
            self._scan_forward_fused(first)
        for t in (() if self.fused_scan or self.decoupled else range(self.T)):
            s = slice(t * B, (t + 1) * B)
            f = first[s]
            if t == 0:
                zp, hp = self.zero_z, self.zero_h
            else:
                sp = slice((t - 1) * B, t * B)
                zp, hp = self.latent[sp, :Z], self.latent[sp, Z:]
            ops.mask_rows(self.shift_actions[s], f, self.a_in[s])
            ops.mask_mix(hp, self.h0, f, self.h_in[s])
            ops.mask_mix(zp, self.z0, f, self.z_in[s])
            h = self.latent[s, Z:]
            self._recurrent_forward(self.z_in[s], self.a_in[s], self.h_in[s], self.x_pre[s], self.x_act[s],
                                    self.g_pre[s], self.g_ln[s], h)
            ops.copy(self.pe[s], self.rp_pre[s])
            self._posterior_forward(h, self.rp_pre[s], self.rp_act[s], self.post_raw[s], self.noise_post[t],
                                    self.latent[s, :Z], self.post_mix[s])
        self._prior_forward()

    def _scan_forward_decoupled(self, first: torch.Tensor):
        """DecoupledRSSM (dreamer_v3.py:115-129, agent.py:571-593): the posterior is a function of the embedding alone, so
        z of every step, x = SiLU(LN(W_in [z_{t-1}, a_{t-1}])) and x's share of the GRU product are batched over all
        T*B rows; only h_in W_g[:, :R]^T, the GRU LayerNorm and the gate stay on the recurrence."""
        ops, B, N, Z, R = self.ops, self.B, self.N, self.Z, self.R
        self._posterior_forward(None, self.rp_pre, self.rp_act, self.post_raw, self.noise_post.view(N, Z),
                                self.latent[:, :Z], self.post_mix)
        ops.mask_mix(self.zero_z, self.z0, first[:B], self.z_in[:B])
        if N > B:
            ops.mask_mix(self.latent[:N - B, :Z], self.z0, first[B:], self.z_in[B:])
        ops.mask_rows(self.shift_actions, first, self.a_in)
        self._recurrent_input(self.z_in, self.a_in, self.x_pre, self.x_act)
        ops.gemm(self.x_act, self._w("rssm.recurrent_model.rnn.linear.weight")[:, R:], self.g_pre, False, True)
        if self.fused_scan:
            if self._scan_ws is None:
                self._scan_ws = ops.gru_scan_workspace(self.T, B, R)
            ops.gru_scan_fwd(self._gru_scan_dims(), self.eps, self._gru_scan_tensors(first), self._scan_ws)
            return
        for t in range(self.T):
            s = slice(t * B, (t + 1) * B)
            hp = self.zero_h if t == 0 else self.latent[(t - 1) * B:t * B, Z:]
            ops.mask_mix(hp, self.h0, first[s], self.h_in[s])
            self._gru_forward(self.h_in[s], None, self.g_pre[s], self.g_ln[s], self.latent[s, Z:])

    def _gru_scan_dims(self):
        return dict(T=self.T, B=self.B, R=self.R, ld_wg=self.R + self.Dx, ld_lat=self.L, lat_off=self.Z)

    def _gru_scan_tensors(self, first: torch.Tensor):
        p = "rssm.recurrent_model.rnn."
        return dict(W_g=self._w(p + "linear.weight"), lng_g=self._w(p + "layer_norm.weight"),
                    lng_b=self._w(p + "layer_norm.bias"), h0=self.h0, first=first, g_pre=self.g_pre, g_ln=self.g_ln,
                    h_in=self.h_in, latent=self.latent)

    def _prior_forward(self):
        """The prior of every step (transition model on h_t, agent.py:433) is off the recurrence: with the h sequence
        finished it is two batched tensor-core products over all T*B rows instead of 2 x T skinny ones in the scan."""
        Z = self.Z
        self._transition_forward(self.latent[:, Z:], self.tr_pre, self.tr_act, self.prior_raw)
        # only the prior's unimix log-probs are needed (the prior sample is discarded, dreamer_v3.py:135)
        self.ops.cat_sample(self.prior_raw, None, self.unimix, self.S, self.D, None, self.prior_mix)

    def _scan_forward_fused(self, first: torch.Tensor):
        """The posterior recurrence of the scan as ONE persistent cooperative kernel (csrc/rssm_scan.cu).  Produces
        exactly the saved activations of the per-step path."""
        if self._scan_ws is None:
            self._scan_ws = self.ops.rssm_scan_workspace(self.T, self.B, self.S, self.D, self.Dx, self.R, self.Dr)
        self.ops.rssm_scan_fwd(self._scan_dims(), self.eps, self.unimix, self._scan_tensors(first), self._scan_ws)

    def _scan_dims(self):
        return dict(T=self.T, B=self.B, S=self.S, D=self.D, R=self.R, A=self.A, Dx=self.Dx, Dt=self.Dt, Dr=self.Dr,
                    ld_lat=self.L, ld_wr1=self.Rh + self.E + self.Ev)

    def _scan_tensors(self, first: torch.Tensor):
        p = "rssm.recurrent_model."
        pt, pr = "rssm.transition_model._model.", "rssm.representation_model._model."
        w = self._w
        return dict(
            W_in=w(p + "mlp._model.0.weight"), lnx_g=w(p + "mlp._model.1.weight"), lnx_b=w(p + "mlp._model.1.bias"),
            W_g=w(p + "rnn.linear.weight"), lng_g=w(p + "rnn.layer_norm.weight"), lng_b=w(p + "rnn.layer_norm.bias"),
            W_t1=w(pt + "0.weight"), lnt_g=w(pt + "1.weight"), lnt_b=w(pt + "1.bias"), W_t2=w(pt + "3.weight"),
            b_t2=w(pt + "3.bias"), W_r1=w(pr + "0.weight"), lnr_g=w(pr + "1.weight"), lnr_b=w(pr + "1.bias"),
            W_r2=w(pr + "3.weight"), b_r2=w(pr + "3.bias"), h0=self.h0, z0=self.z0, pe=self.pe,
            actions=self.shift_actions, first=first, noise=self.noise_post, latent=self.latent, z_in=self.z_in,
            h_in=self.h_in, a_in=self.a_in, x_pre=self.x_pre, x_act=self.x_act, g_pre=self.g_pre, g_ln=self.g_ln,
            tr_pre=self.tr_pre, tr_act=self.tr_act, rp_pre=self.rp_pre, rp_act=self.rp_act, post_raw=self.post_raw,
            prior_raw=self.prior_raw, post_mix=self.post_mix, prior_mix=self.prior_mix)

    def _prior_backward(self):
        """Backward of the batched prior: its gradient comes from the KL term only (d_prior_mix), so it does not depend on
        the BPTT; its contribution to dh is added to d_latent before the backward scan starts.  Also writes the
        transition model's LayerNorm parameter gradients."""
        self._transition_backward(self.prior_raw, self.tr_pre, None, self.d_prior_mix, self.d_prior_raw, self.d_tr_act,
                                  self.d_tr_pre, self.d_latent[:, self.Z:], ln_grads=True)

    def _scan_backward_fused(self, first: torch.Tensor):
        """BPTT of the posterior recurrence as ONE persistent cooperative kernel, after the three `pre-activation x
        weight` products that let the kernel apply every LayerNorm-backward correction on the consumer side
        (csrc/rssm_scan.cu).  It fills d_post_raw and the activation gradients d_rp_act / d_g_ln / d_x_act; the deferred
        section turns those into the pre-activation gradients for all T*B rows at once."""
        ops, Z, R = self.ops, self.Z, self.R
        if self._scan_q is None:
            new = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=self.device)  # noqa: E731
            self._scan_q = (new(self.N, R), new(self.N, R + self.Dx), new(self.N, Z))
        q_r, q_g, q_x = self._scan_q
        grads = dict(d_latent=self.d_latent, d_post_mix=self.d_post_mix, d_prior_mix=self.d_prior_mix,
                     d_post_raw=self.d_post_raw, d_prior_raw=self.d_prior_raw, d_rp_act=self.d_rp_act,
                     d_rp_pre=self.d_rp_pre, d_tr_act=self.d_tr_act, d_tr_pre=self.d_tr_pre, d_g_ln=self.d_g_ln,
                     d_g_pre=self.d_g_pre, d_x_act=self.d_x_act, d_x_pre=self.d_x_pre, d_h0=self.d_h0,
                     q_r=q_r, q_g=q_g, q_x=q_x)
        p, pr = "rssm.recurrent_model.", "rssm.representation_model._model."
        ops.gemm(self.rp_pre, self._w(pr + "0.weight")[:, :R], q_r, False, False)
        ops.gemm(self.g_pre, self._w(p + "rnn.linear.weight"), q_g, False, False)
        ops.gemm(self.x_pre, self._w(p + "mlp._model.0.weight")[:, :Z], q_x, False, False)
        ops.rssm_scan_bwd(self._scan_dims(), self.eps, self.unimix, self._scan_tensors(first), grads, self._scan_ws)

    def _scan_backward(self, first: torch.Tensor):
        """BPTT over the scan (SURVEY.md App. E): the batched prior backward, then the posterior recurrence.  Per step
        only the data-gradient GEMMs run; the weight gradients are single big GEMMs over all T*B rows afterwards."""
        ops, B, Z, R = self.ops, self.B, self.Z, self.R
        pt, pr = "rssm.transition_model._model.", "rssm.representation_model._model."
        Wr1 = self._w(pr + "0.weight")
        ops.zero(self.dz_carry)
        ops.zero(self.dh_carry)
        ops.zero(self.d_h0)
        self._prior_backward()
        fused = self.fused_scan and self.fused_scan_bwd
        if self.decoupled:
            self._scan_backward_decoupled(first, fused)
        elif fused:
            self._scan_backward_fused(first)
        for t in (() if fused or self.decoupled else reversed(range(self.T))):
            s = slice(t * B, (t + 1) * B)
            f = first[s]
            ops.copy(self.d_latent[s, :Z], self.dz_tot)
            ops.axpy(self.dz_carry, self.dz_tot)
            ops.copy(self.d_latent[s, Z:], self.dh_tot)
            ops.axpy(self.dh_carry, self.dh_tot)
            # posterior: straight-through sample + KL -> raw logits -> representation model
            ops.cat_sample_bwd(self.post_raw[s], self.dz_tot, self.d_post_mix[s], self.unimix, self.S, self.D,
                               self.d_post_raw[s])
            ops.gemm(self.d_post_raw[s], self._w(pr + "3.weight"), self.d_rp_act[s], False, False)
            ops.ln_act_bwd(self.rp_pre[s], self._w(pr + "1.weight"), self._w(pr + "1.bias"), self.eps, ACT_SILU,
                           self.d_rp_act[s], self.d_rp_pre[s], None, None)
            ops.gemm(self.d_rp_pre[s], Wr1[:, :R], self.dh_tot, False, False, accumulate=True)
            self._recurrent_backward(self.g_ln[s], self.h_in[s], self.g_pre[s], self.x_pre[s], self.dh_tot,
                                     self.d_g_ln[s], self.d_g_pre[s], self.d_x_act[s], self.d_x_pre[s], self.dh_in,
                                     self.dz_in)
            ops.mask_bwd(self.dz_in, f, self.dz_carry, None)
            ops.mask_bwd(self.dh_in, f, self.dh_carry, self.d_h0)
        # ---- deferred parameter gradients over all N rows
        self._representation_param_grads()
        gW, h_all = self._gw, self.latent[:, Z:]
        # transition model
        ops.gemm(self.d_prior_raw, self.tr_act, gW(pt + "3.weight"), True, False)
        ops.col_sum(self.d_prior_raw, gW(pt + "3.bias"))
        ops.gemm(self.d_tr_pre, h_all, gW(pt + "0.weight"), True, False)
        if not self.decoupled:          # (decoupled: done in front of the posterior's backward, which consumes d_x_pre)
            self._recurrent_param_grads()
        # learned initial recurrent state: h0 = tanh(param)
        if self.cfg.algo.world_model.get("learnable_initial_recurrent_state", True):
            ops.tanh_bwd(self.h0.view(R), self.d_h0, gW("rssm.initial_recurrent_state"))
        # else: a buffer in the reference (agent.py:382-389) — its gradient stays at the zero `wm.grad` was reset to, the
        # norm ignores it and Adam's zero moments leave the value untouched

    def _representation_param_grads(self):
        """Parameter gradients of the representation model over all N rows, and the gradient of the embedding"""
        ops, R, E, Z, gW = self.ops, self.Rh, self.E, self.Z, self._gw
        pr = "rssm.representation_model._model."
        Wr1 = self._w(pr + "0.weight")
        ops.gemm(self.d_post_raw, self.rp_act, gW(pr + "3.weight"), True, False)
        ops.col_sum(self.d_post_raw, gW(pr + "3.bias"))
        # LayerNorm parameter gradients over all rows; the same pass (re)writes the pre-activation gradients the weight
        # products below consume (the fused backward kernel saves only the activation gradients)
        ops.ln_act_bwd(self.rp_pre, self._w(pr + "1.weight"), self._w(pr + "1.bias"), self.eps, ACT_SILU,
                       self.d_rp_act, self.d_rp_pre, gW(pr + "1.weight"), gW(pr + "1.bias"))
        gWr1 = gW(pr + "0.weight")
        if R:
            ops.gemm(self.d_rp_pre, self.latent[:, Z:], gWr1[:, :R], True, False)
        if self.has_cnn:
            ops.gemm(self.d_rp_pre, self.emb, gWr1[:, R:R + E], True, False)
            ops.gemm(self.d_rp_pre, Wr1[:, R:R + E], self.d_emb, False, False)
        if self.vec_keys:
            ops.gemm(self.d_rp_pre, self.venc.act[-1], gWr1[:, R + E:], True, False)
            ops.gemm(self.d_rp_pre, Wr1[:, R + E:], self.d_emb_vec, False, False)

    def _recurrent_param_grads(self, x_data_grad: bool = False):
        """Parameter gradients of the recurrent model over all N rows.  `x_data_grad`: d_x_act is not there yet and is
        one batched product of d_g_pre (decoupled RSSM: x is off the recurrence)."""
        ops, Z, R, gW = self.ops, self.Z, self.R, self._gw
        p = "rssm.recurrent_model."
        ops.ln_act_bwd(self.g_pre, self._w(p + "rnn.layer_norm.weight"), self._w(p + "rnn.layer_norm.bias"),
                       self.eps, ACT_NONE, self.d_g_ln, self.d_g_pre, gW(p + "rnn.layer_norm.weight"),
                       gW(p + "rnn.layer_norm.bias"))
        gWg = gW(p + "rnn.linear.weight")
        ops.gemm(self.d_g_pre, self.h_in, gWg[:, :R], True, False)
        ops.gemm(self.d_g_pre, self.x_act, gWg[:, R:], True, False)
        if x_data_grad:
            ops.gemm(self.d_g_pre, self._w(p + "rnn.linear.weight")[:, R:], self.d_x_act, False, False)
        ops.ln_act_bwd(self.x_pre, self._w(p + "mlp._model.1.weight"), self._w(p + "mlp._model.1.bias"), self.eps,
                       ACT_SILU, self.d_x_act, self.d_x_pre, gW(p + "mlp._model.1.weight"),
                       gW(p + "mlp._model.1.bias"))
        gWin = gW(p + "mlp._model.0.weight")
        ops.gemm(self.d_x_pre, self.z_in, gWin[:, :Z], True, False)
        ops.gemm(self.d_x_pre, self.a_in, gWin[:, Z:], True, False)

    def _scan_backward_decoupled(self, first: torch.Tensor, fused: bool):
        """BPTT of the decoupled scan: the GRU recurrence alone walks back through time (one persistent kernel inside
        its envelope, else per step); x, z_{t-1} and the posterior are batched over all T*B rows behind it."""
        ops, B, N, Z, R = self.ops, self.B, self.N, self.Z, self.R
        p, pr = "rssm.recurrent_model.", "rssm.representation_model._model."
        if fused:
            if self._scan_q is None:
                self._scan_q = torch.zeros(N, R, dtype=torch.float32, device=self.device)
            # g_pre W_g[:, :R]: lets the kernel apply the LayerNorm-backward correction on the consumer side
            ops.gemm(self.g_pre, self._w(p + "rnn.linear.weight")[:, :R], self._scan_q, False, False)
            ops.gru_scan_bwd(self._gru_scan_dims(), self.eps, self._gru_scan_tensors(first),
                             dict(d_latent=self.d_latent, d_g_ln=self.d_g_ln, d_h0=self.d_h0, q_g=self._scan_q),
                             self._scan_ws)
        for t in (() if fused else reversed(range(self.T))):
            s = slice(t * B, (t + 1) * B)
            ops.copy(self.d_latent[s, Z:], self.dh_tot)
            ops.axpy(self.dh_carry, self.dh_tot)
            self._gru_backward(self.g_ln[s], self.h_in[s], self.g_pre[s], self.dh_tot, self.d_g_ln[s], self.d_g_pre[s],
                               self.dh_in)
            ops.mask_bwd(self.dh_in, first[s], self.dh_carry, self.d_h0)
        self._recurrent_param_grads(x_data_grad=True)
        # z_{t-1} feeds x_t: (1 - f_t) d_x_pre[t] W_in[:, :Z] joins the gradient of z_{t-1} (the f_t share goes to z0, a
        # mode: no gradient); d_x_act has been consumed and stages the masked rows
        if N > B:
            ops.mask_rows(self.d_x_pre, first, self.d_x_act)
            ops.gemm(self.d_x_act[B:], self._w(p + "mlp._model.0.weight")[:, :Z], self.d_latent[:N - B, :Z], False, False,
                     accumulate=True)
        ops.cat_sample_bwd(self.post_raw, self.d_latent[:, :Z], self.d_post_mix, self.unimix, self.S, self.D,
                           self.d_post_raw)
        ops.gemm(self.d_post_raw, self._w(pr + "3.weight"), self.d_rp_act, False, False)

    # ------------------------------------------------------------------ optimiser
    def _wm_buckets(self):
        """(first float of the rssm range, first float of the decoder / heads range) of the world model's flat buffer"""
        off = self.wm.offsets
        b_enc = off["rssm.initial_recurrent_state"]
        tail = [v for k, v in off.items() if not (k.startswith("encoder.") or k.startswith("rssm."))]
        return b_enc, min(tail)

    def _optimizer_step(self, name: str, g: FlatGroup, max_norm: float, ocfg, slot: int, reduced: bool = False):
        ops = self.ops
        if self.allreduce is not None and not reduced:
            self.allreduce(g.grad, name)
        ops.sumsq(g.grad, self.normsq[name])
        g.step += 1
        ops.increment(g.step_t)
        b1, b2 = ocfg.betas
        opt = getattr(g, "optimizer", None)                  # the handle build by main / make_optimizers (schedulers edit it)
        lr = opt.lr if opt is not None else float(ocfg.lr)
        ops.adam_step(g.flat, g.grad, g.exp_avg, g.exp_avg_sq, self.normsq[name], max_norm, lr,
                      float(b1), float(b2), float(ocfg.eps), g.step_t, self.norms[slot: slot + 1],
                      **g.adam_kwargs(ocfg.get("weight_decay", 0.0)))

    # ------------------------------------------------------------------ behaviour learning
    def _actor_heads(self, hidden: torch.Tensor, raw_out: torch.Tensor, actor: Optional[FlatGroup] = None):
        actor = actor or self.actor
        if self.is_continuous:
            self.ops.gemm(hidden, actor.views["mlp_heads.0.weight"], raw_out, False, True,
                          bias=actor.views["mlp_heads.0.bias"])
            return
        off = 0
        for i, ad in enumerate(self.actions_dim):
            self.ops.gemm(hidden, actor.views[f"mlp_heads.{i}.weight"], raw_out[:, off:off + ad], False, True,
                          bias=actor.views[f"mlp_heads.{i}.bias"])
            off += ad

    def _imagine(self, actor: Optional[FlatGroup] = None, actor_mlp: Optional["_MLP"] = None):
        """H-step rollout from every posterior state (dreamer_v3.py:203-241), forward only: with discrete
        actions the policy gradient does not flow through the rollout (SURVEY.md App. E).  `actor` / `actor_mlp`:
        another policy over the same world model (Plan2Explore's exploration actor); default the task actor."""
        ops, N, Z, R, H = self.ops, self.N, self.Z, self.R, self.H
        actor = actor or self.actor
        am = actor_mlp or self.actor_mlp
        # imagined z is an exact one-hot sample: its Linear is a gather over the transposed weight (refreshed here,
        # after the world-model update)
        Win = self._w("rssm.recurrent_model.mlp._model.0.weight")
        gather = ops.onehot_linear_supported(self.S, self.D, self.A, Win.shape[0])
        if gather:
            if getattr(self, "_win_t", None) is None:
                self._win_t = torch.empty(Win.shape[1], Win.shape[0], dtype=torch.float32, device=self.device)
            ops.transpose2d(Win, self._win_t)
        h_staged = False
        for i in range(H + 1):
            rows = slice(i * N, (i + 1) * N)
            if i > 0:
                prev, cur = self.traj[i - 1], self.traj[i]
                if self.is_continuous:       # keep every step's activations for the backward through the rollout
                    j = i - 1
                    x_pre, hx, g_pre, g_ln = self.c_x_pre[j], self.c_hx[j], self.c_g_pre[j], self.c_g_ln[j]
                    tr_pre, tr_act, raw = self.c_tr_pre[j], self.c_tr_act[j], self.c_raw[j]
                else:
                    x_pre, hx, g_pre, g_ln = self.i_x_pre, self.i_hx, self.i_g_pre, self.i_g_ln
                    tr_pre, tr_act, raw = self.i_tr_pre, self.i_tr_act, self.i_raw
                if not h_staged:
                    ops.copy(prev[:, Z:], hx[:, :R])
                keep = self.is_continuous
                h_next = None
                if i < H:
                    h_next = (self.c_hx[i] if self.is_continuous else hx)[:, :R]
                h_staged = self._recurrent_forward(prev[:, :Z], self.actions[i - 1], prev[:, Z:], x_pre, hx[:, R:], g_pre,
                                                   g_ln, cur[:, Z:], win_t=self._win_t if gather else None, hx=hx,
                                                   h_next=h_next, keep=keep) and h_next is not None
                self._transition_forward(cur[:, Z:], tr_pre, tr_act, raw, keep=keep)
                ops.cat_sample(raw, self.noise_img_state[i - 1], self.unimix, self.S, self.D, cur[:, :Z])
            # actor on traj[i]; activations are kept for the policy-gradient backward (the reference's second
            # actor evaluation at dreamer_v3.py:273 recomputes exactly these numbers)
            x = self.traj[i]
            cur_in = x
            for l in range(am.n_hidden):
                dense_ln_act(ops, cur_in, am.W(l), actor.views[f"model._model.{3 * l + 1}.weight"],
                             actor.views[f"model._model.{3 * l + 1}.bias"], self.eps, ACT_SILU, am.act[l][rows],
                             am.pre[l][rows])
                cur_in = am.act[l][rows]
            if not self.is_continuous:
                off, done = 0, True
                for k, ad in enumerate(self.actions_dim):
                    Wh = actor.views[f"mlp_heads.{k}.weight"]
                    done = done and ops.head_sample_supported(cur_in, Wh)
                if done:
                    for k, ad in enumerate(self.actions_dim):
                        ops.head_sample(cur_in, actor.views[f"mlp_heads.{k}.weight"], actor.views[f"mlp_heads.{k}.bias"],
                                        self._img_action_noise(i, off, ad), self.unimix,
                                        self.actor_raw[rows, off:off + ad], self.actions[i, :, off:off + ad])
                        off += ad
                    continue
            self._actor_heads(cur_in, self.actor_raw[rows], actor)
            if self.is_continuous:
                ac = self.cfg.algo.actor
                ops.cont_action_fwd(self.actor_raw[rows], self.noise_img_action[i], self.actions[i], self.act_ent[rows],
                                    float(ac.min_std), float(ac.max_std), float(ac.init_std), float(ac.action_clip))
                continue
            off = 0
            for k, ad in enumerate(self.actions_dim):
                ops.cat_sample(self.actor_raw[rows, off:off + ad], self._img_action_noise(i, off, ad),
                               self.unimix, 1, ad, self.actions[i, :, off:off + ad])
                off += ad


    def _img_action_noise(self, i: int, off: int, ad: int) -> Optional[torch.Tensor]:
        """Exp(1) noise of one action head at imagination step i; None (the mode) for the MineDojo actor, whose
        forward defaults to greedy=True when train() calls it (dreamer_v3.py:219,240; agent.py:882)"""
        return None if self.minedojo else self.noise_img_action[i, :, off:off + ad]

    def _continuous_policy_gradient(self, c_logit, critics):
        """Continuous actions: objective = advantage (dreamer_v3.py:283-284), so d(policy_loss) flows from the
        lambda-values and the baseline through the critic / reward heads into the imagined states, back through the
        15 dynamics steps (straight-through prior samples, transition MLP, GRU, Linear([z, a])) into each step's
        action and from there into the actor head.  World-model / critic weights are constants here (the reference
        discards their gradients from this loss): every product is a data-gradient product.
        critics: one (mlp, v_logits, values, lam, moments_out, share, r_logits, rows) per critic whose advantage enters
        the objective with weight `share` (Dreamer-V3: the task critic alone, share 1; Plan2Explore: every exploration
        critic).  r_logits: the reward head's logits when that critic's reward is the task reward, None when it is a
        constant of the loss (the intrinsic reward).  rows[m] = discount * (advantage + entropy bonus / share); the
        bonus is counted in the first critic's rows only, its gradient once in the rollout backward."""
        ops, N, H, Z, R, L = self.ops, self.N, self.H, self.Z, self.R, self.L
        a = self.cfg.algo
        ac = a.actor
        M1, M0 = (H + 1) * N, H * N
        traj2, d_traj2 = self.traj.view(M1, L), self.d_traj.view(M1, L)
        for j, (mlp, v_logits, values, lam, moments, share, r_logits, rows) in enumerate(critics):
            ops.lambda_returns_bwd(c_logit.view(H + 1, N), self.discount, moments, lam, values, self.act_ent,
                                   float(a.gamma), float(a.lmbda), float(ac.ent_coef) / share if j == 0 else 0.0,
                                   share / M0, self.d_values, self.d_rew, rows.view(H, N))
            ops.twohot_mean_bwd(v_logits, self.d_values.view(-1), TWOHOT_LOW, TWOHOT_HIGH, self.d_v_logits)
            if r_logits is not None:
                ops.twohot_mean_bwd(r_logits, self.d_rew.view(-1), TWOHOT_LOW, TWOHOT_HIGH, self.d_r_logits)
            mlp.backward(traj2, self.d_v_logits, d_traj2, j > 0, data_only=True)
            if r_logits is not None:
                self.rew_img.backward(traj2, self.d_r_logits, d_traj2, True, data_only=True)
        args = (float(ac.min_std), float(ac.max_std), float(ac.init_std), float(ac.action_clip))
        ops.zero(self.cd_dz_carry)
        ops.zero(self.cd_dh_carry)
        for i in range(H, 0, -1):
            j = i - 1
            # total gradient of state i = heads (critic / reward on traj[i]) + what step i+1 sent back
            ops.copy(self.d_traj[i][:, :Z], self.cd_dz)
            ops.axpy(self.cd_dz_carry, self.cd_dz)
            ops.copy(self.d_traj[i][:, Z:], self.cd_dh)
            ops.axpy(self.cd_dh_carry, self.cd_dh)
            # z_i = straight-through sample of prior(h_i) -> transition MLP -> h_i
            self._transition_backward(self.c_raw[j], self.c_tr_pre[j], self.cd_dz, None, self.cd_raw, self.cd_tr_act,
                                      self.cd_tr_pre, self.cd_dh)
            # h_i = GRU(h_{i-1}, x_i), x_i = SiLU(LN(W_in [z_{i-1}, a_{i-1}]))
            self._recurrent_backward(self.c_g_ln[j], self.c_hx[j][:, :R], self.c_g_pre[j], self.c_x_pre[j], self.cd_dh,
                                     self.cd_g_ln, self.cd_g_pre, self.cd_x_act, self.cd_x_pre, self.cd_dh_carry,
                                     self.cd_dz_carry, da=self.cd_a)
            # a_{i-1}: through the clipped rsample into the actor head; entropy bonus of step i-1
            rows = slice(j * N, (j + 1) * N)
            ops.cont_action_bwd(self.actor_raw[rows], self.noise_img_action[j], self.cd_a, self.discount[j],
                                self.d_actor_raw[rows], *args, -float(ac.ent_coef) / M0)

    def _behaviour_losses(self):
        ops, N, H, L = self.ops, self.N, self.H, self.L
        a = self.cfg.algo
        M1, M0 = (H + 1) * N, H * N
        traj2 = self.traj.view(M1, L)
        # ---- values / rewards / continues on the trajectories (dreamer_v3.py:244-248)
        v_logits = self.critic_mlp.forward(traj2)
        ops.twohot_mean(v_logits, TWOHOT_LOW, TWOHOT_HIGH, self.values.view(-1))
        r_logits = self.rew_img.forward(traj2)
        ops.twohot_mean(r_logits, TWOHOT_LOW, TWOHOT_HIGH, self.rew_pred.view(-1))
        c_logit = self.cont_img.forward(traj2)
        ops.lambda_returns(self.rew_pred, self.values, c_logit.view(H + 1, N), self.true_cont, float(a.gamma),
                           float(a.lmbda), self.lam, self.discount)
        # ---- Moments (dreamer_v3/utils.py:56-63)
        mo = a.actor.moments
        lam_all = self.lam if self.allgather is None else self.allgather(self.lam)
        ops.moments_update(lam_all.view(-1), self.moments_state, float(mo.decay), float(mo.max),
                           float(mo.percentile.low), float(mo.percentile.high), self.moments_out)
        # ---- actor (dreamer_v3.py:272-304)
        if self.is_continuous:
            self._continuous_policy_gradient(c_logit, [(self.critic_mlp, v_logits, self.values, self.lam, self.moments_out,
                                                        1.0, r_logits, self.policy_rows)])   # fills d_actor_raw, policy_rows
        else:
            ops.actor_loss_grad(self.actor_raw[:M0], self.actions.view(M1, self.A)[:M0], self.lam.view(-1),
                                self.values.view(-1)[:M0], self.discount.view(-1)[:M0], self.moments_out,
                                self.actions_dim, self.unimix, float(a.actor.ent_coef), 1.0 / M0, self.policy_rows,
                                self.d_actor_raw)
        ops.sum_rows(self.policy_rows.view(M0, 1), self.metrics[8:9], -1.0 / M0)
        self._actor_update(self.actor, self.actor_mlp, "actor", 1)
        # ---- critic (dreamer_v3.py:307-327): qv logits are the first H*N rows of v_logits (same weights,
        # same inputs as the reference's second critic evaluation)
        self._critic_update(self.critic, self.critic_mlp, self.target_mlp, v_logits, self.lam, self.metrics[9:10],
                            "critic", 2)

    def _actor_update(self, actor: FlatGroup, am: "_MLP", name: str, slot: int):
        """backward of the policy loss from `d_actor_raw` (rows of the first H steps) through the heads and the actor
        MLP whose activations the rollout kept, then all-reduce / clip / Adam (dreamer_v3.py:298-304)"""
        ops, N, H, L = self.ops, self.N, self.H, self.L
        a = self.cfg.algo
        M1, M0 = (H + 1) * N, H * N
        traj2 = self.traj.view(M1, L)
        ops.zero(actor.grad)
        last = am.act[-1][:M0]
        ops.zero(self.d_actor_hidden)
        off = 0
        for i, ad in enumerate((self.AW,) if self.is_continuous else self.actions_dim):
            d = self.d_actor_raw[:, off:off + ad]
            ops.gemm(d, last, actor.gviews[f"mlp_heads.{i}.weight"], True, False)
            ops.col_sum(d, actor.gviews[f"mlp_heads.{i}.bias"])
            ops.gemm(d, actor.views[f"mlp_heads.{i}.weight"], self.d_actor_hidden, False, False, accumulate=True)
            off += ad
        am.backward(traj2[:M0], self.d_actor_hidden, None, False, M=M0)
        self._optimizer_step(name, actor, float(a.actor.clip_gradients or 0.0), a.actor.optimizer, slot)

    def _critic_update(self, critic: FlatGroup, cm: "_MLP", tm: "_MLP", v_logits: torch.Tensor, lam: torch.Tensor,
                       metric: torch.Tensor, name: str, slot: int):
        """two-hot regression of the critic on the lambda-values and on the target critic's values, discount-weighted
        (dreamer_v3.py:307-327); `v_logits` are `cm`'s logits on the whole trajectory (its activations are live)"""
        ops, N, H, L = self.ops, self.N, self.H, self.L
        a = self.cfg.algo
        M1, M0 = (H + 1) * N, H * N
        traj2 = self.traj.view(M1, L)
        t_logits = tm.forward(traj2[:M0])
        ops.twohot_mean(t_logits, TWOHOT_LOW, TWOHOT_HIGH, self.target_values)
        disc = self.discount.view(-1)[:M0]
        ops.twohot_loss_grad(v_logits[:M0], lam.view(-1), disc, 1.0 / M0, TWOHOT_LOW, TWOHOT_HIGH,
                             self.value_rows, self.d_critic_logits)
        ops.twohot_loss_grad(v_logits[:M0], self.target_values, disc, 1.0 / M0, TWOHOT_LOW, TWOHOT_HIGH,
                             self.value_rows, self.d_critic_logits, accumulate=True)
        ops.weighted_mean(self.value_rows, disc, 1.0 / M0, metric)
        ops.zero(critic.grad)
        cm.backward(traj2[:M0], self.d_critic_logits, None, False, M=M0)
        self._optimizer_step(name, critic, float(a.critic.clip_gradients or 0.0), a.critic.optimizer, slot)

    # ------------------------------------------------------------------ misc
    METRIC_NAMES = (
        "Loss/world_model_loss", "Loss/observation_loss", "Loss/reward_loss", "Loss/state_loss",
        "Loss/continue_loss", "State/kl", "State/post_entropy", "State/prior_entropy", "Loss/policy_loss",
        "Loss/value_loss",
    )

    def metrics_dict(self) -> Dict[str, torch.Tensor]:
        d = {n: self.metrics[i] for i, n in enumerate(self.METRIC_NAMES)}
        d["Grads/world_model"], d["Grads/actor"], d["Grads/critic"] = self.norms[0], self.norms[1], self.norms[2]
        return d

    def update_target(self, tau: float):
        """Target-critic EMA (reference: dreamer_v3.py:674-680, done by `main` before each train call)."""
        if tau >= 1.0:
            self.ops.copy(self.critic.flat, self.target.flat)
        else:
            self.ops.ema(self.target.flat, self.critic.flat, float(tau))
