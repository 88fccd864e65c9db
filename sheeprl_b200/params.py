"""Flat parameter groups in HBM.

Every optimiser group (world model / actor / critic) lives in ONE contiguous fp32 buffer so that the
gradient-norm, clip+Adam and NCCL all-reduce each touch a single region (28 B/param of traffic for
the whole clip+Adam, SURVEY.md §8d).  The named tensors the reference exposes through `state_dict()`
(layout: SURVEY.md §8b) are *views* into that buffer, so checkpoints keep the reference's key names
and shapes and `nn.Parameter.data` can alias them.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Mapping, Tuple

import torch

ALIGN = 64  # floats; keeps every tensor 256-byte aligned for vector loads / TMA


class FlatGroup:
    def __init__(self, shapes: Mapping[str, Tuple[int, ...]], device, with_optimizer: bool = True):
        self.shapes = OrderedDict((k, tuple(v)) for k, v in shapes.items())
        self.offsets: Dict[str, int] = {}
        off = 0
        for k, shp in self.shapes.items():
            self.offsets[k] = off
            n = 1
            for s in shp:
                n *= s
            off += (n + ALIGN - 1) // ALIGN * ALIGN
        self.numel = off
        self.device = torch.device(device)
        self.flat = torch.zeros(off, dtype=torch.float32, device=device)
        self.views = self._views(self.flat)
        if with_optimizer:
            self.grad = torch.zeros_like(self.flat)
            self.exp_avg = torch.zeros_like(self.flat)
            self.exp_avg_sq = torch.zeros_like(self.flat)
            self.gviews = self._views(self.grad)
        self.grad_avg = None                                              # RMSprop(centered=True) only: alloc_grad_avg()
        self.step = 0                                                     # host mirror of step_t
        self.step_t = torch.zeros(1, dtype=torch.int32, device=device)    # device-side Adam step (graph-safe)

    def _views(self, flat: torch.Tensor) -> "OrderedDict[str, torch.Tensor]":
        out = OrderedDict()
        for k, shp in self.shapes.items():
            n = 1
            for s in shp:
                n *= s
            out[k] = flat[self.offsets[k]: self.offsets[k] + n].view(shp)
        return out

    def load(self, state: Mapping[str, torch.Tensor]):
        missing = set(self.shapes) - set(state)
        extra = set(state) - set(self.shapes)
        if missing or extra:
            raise KeyError(f"state dict mismatch: missing={sorted(missing)} unexpected={sorted(extra)}")
        with torch.no_grad():
            for k, v in self.views.items():
                if tuple(state[k].shape) != tuple(v.shape):
                    raise ValueError(f"shape mismatch for {k}: {tuple(state[k].shape)} vs {tuple(v.shape)}")
                v.copy_(state[k])

    def state_dict(self) -> "OrderedDict[str, torch.Tensor]":
        return OrderedDict((k, v.detach().clone()) for k, v in self.views.items())

    def optimizer_views(self):
        return self._views(self.exp_avg), self._views(self.exp_avg_sq)

    def alloc_grad_avg(self) -> torch.Tensor:
        """the one optimizer buffer not every group needs (centered RMSprop's grad_avg), allocated on first use"""
        if self.grad_avg is None:
            self.grad_avg = torch.zeros_like(self.flat)
        return self.grad_avg

    def adam_kwargs(self, weight_decay: float = 0.0) -> dict:
        """`ops.adam_step`'s optional arguments: the L2 weight decay of the optimizer handle attached to this group
        (`B200Adam`, built from the same optimizer config), or `weight_decay` when no handle is attached.  Without decay
        the call keeps the plain Adam form."""
        opt = getattr(self, "optimizer", None)
        wd = float((opt.param_groups[0].get("weight_decay") if opt is not None else weight_decay) or 0.0)
        return {"weight_decay": wd} if wd else {}
