"""Batched dense-layer stacks on `ops.bgemm`: the MLPs of the PPO, A2C, recurrent PPO, SAC and DroQ engines.

A `Linear` binds flat-group views of W [n, out, in], b [n, out] and their gradients, so n networks (1, or the stacked
critics) run in one launch per product.  A block says what follows a Linear.  A `Stack`'s buffers live in activation
sets (`Stack.acts`): one stack runs on several sets, and stacks of one shape (online and target critics) share a set.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

ACT_CODE = {"none": 0, "tanh": 2, "relu": 3}          # b200rl_ln_act_* activation codes


def stacked(flat: torch.Tensor, offset: int, n: int, stride: int, shape) -> torch.Tensor:
    """one [n, *shape] view of n equally laid out 1-D or 2-D tensors of `flat`, `stride` floats apart"""
    return torch.as_strided(flat, (n, *shape), (stride, *((shape[1], 1) if len(shape) == 2 else (1,))), offset)


class Linear:
    def __init__(self, W, b, gW=None, gb=None):
        self.W, self.b, self.gW, self.gb = W, b, gW, gb
        self.WT = W.transpose(1, 2)

    @classmethod
    def of(cls, group, wkey: str):
        """n = 1: a flat group's `wkey` and its bias; a convolution's [Cout, k, k, Cin] weight becomes [1, Cout, k*k*Cin]"""
        bkey, v, g = wkey[:-6] + "bias", group.views, group.gviews
        return cls(v[wkey].unsqueeze(0).flatten(2), v[bkey].unsqueeze(0), g[wkey].unsqueeze(0).flatten(2),
                   g[bkey].unsqueeze(0))

    def forward(self, ops, x, y, epi: str = "none"):
        ops.bgemm(x, self.WT, y, bias=self.b, epi=epi)

    def weight_grad(self, ops, d, x):
        ops.bgemm(d.transpose(1, 2), x, self.gW, rsum=self.gb)

    def input_grad(self, ops, d, dx: Sequence[tuple], accumulate: bool = False):
        """d: gradient w.r.t. the output; per (out, cols, epi, aux) of `dx`, the gradient w.r.t. the input columns `cols`
        (a slice; None: all) times the derivative `epi` of the producer's activation, whose output is `aux`"""
        for out, cols, epi, aux in dx:
            ops.bgemm(d, self.W if cols is None else self.W[:, :, cols], out, aux=aux, epi=epi, accumulate=accumulate)


class Act:
    """an activation fused as the product's epilogue; the base of the blocks"""

    def __init__(self, act: str):
        self.act = act

    def alloc(self, f):
        """the block's own buffers of an activation set; f(width=H) allocates one [n, rows, width]"""
        return {}

    def forward(self, ops, lin, x, y, a, mask):
        lin.forward(ops, x, y, self.act)

    def dx_epi(self, y):
        """(epi, aux) of the product that writes the gradient w.r.t. this block's output y"""
        return ("none", None) if self.act in ("none", None) else ("d" + self.act, y)

    def backward(self, ops, dy, y, a, mask, wgrad: bool):
        """the gradient w.r.t. the Linear's output, from dy (w.r.t. the block's output, times `dx_epi`)"""
        return dy


class LayerNormAct(Act):
    """LayerNorm(eps) -> act (n = 1), the backward in place on dy"""

    def __init__(self, group, key: str, eps: float, act: str):
        super().__init__(None)
        v, g = group.views, group.gviews
        self.gamma, self.beta, self.dgamma, self.dbeta = v[key + ".weight"], v[key + ".bias"], g[key + ".weight"], g[key + ".bias"]
        self.eps, self.code = eps, ACT_CODE[act]

    def alloc(self, f):
        return {"pre": f()}

    def forward(self, ops, lin, x, y, a, mask):
        ops.bgemm(x, lin.WT, a["pre"], bias=lin.b)
        ops.ln_act_fwd(a["pre"][0], self.gamma, self.beta, self.eps, self.code, y[0])

    def backward(self, ops, dy, y, a, mask, wgrad: bool):
        ops.ln_act_bwd(a["pre"][0], self.gamma, self.beta, self.eps, self.code, dy[0], dy[0], self.dgamma, self.dbeta)
        return dy


class DropoutLayerNormReLU(Act):
    """Dropout(p) -> LayerNorm(eps) -> ReLU of all n networks in one launch; gamma / beta (and gradients) are [n, H]
    views, `mask` the layer's [n, rows, words] keep mask of the call (None when p == 0)"""

    def __init__(self, p: float, eps: float, gamma, beta, dgamma=None, dbeta=None):
        super().__init__(None)
        self.p, self.eps, self.gamma, self.beta, self.dgamma, self.dbeta = p, eps, gamma, beta, dgamma, dbeta

    def alloc(self, f):
        return {"z": f(), "dz": f(), "stats": f(2)}

    def forward(self, ops, lin, x, y, a, mask):
        ops.bgemm(x, lin.WT, a["z"], bias=lin.b)
        ops.dropout_ln_relu_fwd(a["z"], mask, self.p, self.gamma, self.beta, self.eps, y, a["stats"])

    def backward(self, ops, dy, y, a, mask, wgrad: bool):
        ops.dropout_ln_relu_bwd(dy, y, a["z"], mask, self.p, a["stats"], self.gamma, a["dz"],
                                self.dgamma if wgrad else None, self.dbeta if wgrad else None)
        return a["dz"]


class Stack:
    """(Linear, block) layers; the last block's output is the stack's output.  `masks[i]`: layer i's dropout mask."""

    def __init__(self, ops, layers):
        self.ops, self.layers = ops, list(layers)

    def acts(self, rows: int, grads: bool = True) -> dict:
        """hidden outputs "h", their gradients "dh" (with `grads`) and each block's own buffers"""
        W = self.layers[0][0].W

        def f(i):
            return lambda w=None: torch.zeros(W.shape[0], rows, w or self.layers[i][0].W.shape[1], dtype=torch.float32,
                                              device=W.device)

        hidden = range(len(self.layers) - 1)
        return {"h": [f(i)() for i in hidden], "dh": [f(i)() for i in hidden] if grads else None,
                "blocks": [blk.alloc(f(i)) for i, (_, blk) in enumerate(self.layers)]}

    def forward(self, x, a: dict, out, masks: Optional[Sequence] = None):
        for i, (lin, blk) in enumerate(self.layers):
            y = a["h"][i] if i < len(self.layers) - 1 else out
            blk.forward(self.ops, lin, x, y, a["blocks"][i], _mask(masks, i))
            x = y

    def backward(self, dout, x, a: dict, dx: Sequence[tuple] = (), accumulate: bool = False, wgrad: bool = True,
                 masks: Optional[Sequence] = None):
        """dout: the gradient w.r.t. the output, times the last block's `dx_epi`.  Each layer's weight (and block
        parameter) gradient, when `wgrad`, precedes its input gradient; the first layer's goes to `dx` (`input_grad`)."""
        o, last = self.ops, len(self.layers) - 1
        d = self.layers[last][1].backward(o, dout, None, a["blocks"][last], _mask(masks, last), wgrad)
        for i in range(last, 0, -1):
            lin, below, h, dh = self.layers[i][0], self.layers[i - 1][1], a["h"][i - 1], a["dh"][i - 1]
            if wgrad:
                lin.weight_grad(o, d, h)
            lin.input_grad(o, d, [(dh, None, *below.dx_epi(h))])
            d = below.backward(o, dh, h, a["blocks"][i - 1], _mask(masks, i - 1), wgrad)
        if wgrad:
            self.layers[0][0].weight_grad(o, d, x)
        self.layers[0][0].input_grad(o, d, dx, accumulate)


def _mask(masks, i: int):
    return masks[i] if masks is not None and i < len(masks) else None
