"""TEST INFRASTRUCTURE — import harness for the REAL reference.

Imports the unmodified reference package from $SHEEPRL_REFERENCE_ROOT, else from oracle/_ref (placed there by
oracle/install_ref.py during build(); absent where no reference checkout was available) with permissive stubs for
the third-party packages this project does not depend on (lightning, hydra, omegaconf, gymnasium, torchmetrics, ...).
It is used ONLY to
  * run the tests that execute the reference itself (skipped when it is absent), and
  * generate the committed golden fixtures (oracle/make_golden*.py -> tests/golden/).
Nothing in the product package imports this module.

Recipe follows SURVEY.md Appendix C.
"""
from __future__ import annotations

import importlib
import importlib.abc
import importlib.machinery
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("SHEEPRL_REFERENCE_ROOT",
                                os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref"))
_STUB_ROOTS = {
    "lightning", "hydra", "omegaconf", "gymnasium", "torchmetrics", "moviepy",
    "lightning_utilities", "pytorch_lightning", "mlflow", "pygame", "dotenv_stub_never",
}


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "sheeprl"))


class _Meta(type):
    def __getattr__(cls, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        return _Meta(name, (), {})

    def __getitem__(cls, item):
        return cls

    def __call__(cls, *a, **k):  # instantiating a stub gives a plain object
        return type.__call__(cls) if cls.__init__ is object.__init__ else type.__call__(cls, *a, **k)


class _Loader(importlib.abc.Loader):
    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []

        def _ga(attr, _n=spec.name):
            if attr.startswith("__") and attr.endswith("__"):
                raise AttributeError(attr)
            return _Meta(attr, (), {})

        m.__getattr__ = _ga
        return m

    def exec_module(self, module):
        pass


class _Finder(importlib.abc.MetaPathFinder):
    def find_spec(self, name, path=None, target=None):
        if name.split(".")[0] in _STUB_ROOTS:
            try:  # a really-installed package wins
                for f in sys.meta_path:
                    if f is self:
                        continue
                    s = f.find_spec(name, path, target) if hasattr(f, "find_spec") else None
                    if s is not None:
                        return s
            except Exception:
                pass
            return importlib.machinery.ModuleSpec(name, _Loader(), is_package=True)
        return None


_installed = False


def install():
    """Install the stubs and import the reference `sheeprl` package. Idempotent."""
    global _installed
    if _installed:
        return
    if not reference_available():
        raise RuntimeError(f"reference not found at {REFERENCE_ROOT}")
    sys.meta_path.insert(0, _Finder())

    import lightning_utilities.core.imports as lui

    class RequirementCache:
        def __init__(self, req="", *a, **k):
            self.req = str(req)

        def __bool__(self):
            return self.req.startswith("torch")

    lui.RequirementCache = RequirementCache
    import pytorch_lightning.utilities as plu

    plu.rank_zero_only = lambda f: f
    import hydra.utils as hu

    def get_class(path):
        mod, _, name = path.rpartition(".")
        return getattr(importlib.import_module(mod), name)

    hu.get_class = get_class
    if REFERENCE_ROOT not in sys.path:
        sys.path.append(REFERENCE_ROOT)       # at the END: the reference ships its own top-level `tests` package
    import sheeprl  # noqa: F401
    import sheeprl.algos.dreamer_v3.agent as agent_mod

    agent_mod.get_single_device_fabric = lambda f: f
    _installed = True


class _Wrap(__import__("torch").nn.Module):
    """Mimics lightning's _FabricModule: exposes .module, forwards attributes, plain state_dict keys."""

    def __init__(self, m):
        super().__init__()
        self._forward_module = m

    @property
    def module(self):
        return self._forward_module

    def forward(self, *a, **k):
        return self._forward_module(*a, **k)

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self._forward_module, name)

    def state_dict(self, *a, **k):
        return self._forward_module.state_dict(*a, **k)

    def load_state_dict(self, *a, **k):
        return self._forward_module.load_state_dict(*a, **k)


class FakeFabric:
    def __init__(self, device="cpu"):
        import torch

        self.device = torch.device(device)
        self.world_size = 1
        self.global_rank = 0
        self.is_global_zero = True

    def setup_module(self, m):
        return _Wrap(m.to(self.device))        # Fabric.setup_module moves the module to its device

    def setup_optimizers(self, *o):
        return o if len(o) > 1 else o[0]

    def backward(self, loss):
        loss.backward()

    def all_gather(self, x):
        return x

    def clip_gradients(self, module, optimizer, max_norm, error_if_nonfinite=False):
        import torch

        return torch.nn.utils.clip_grad_norm_(module.parameters(), max_norm, error_if_nonfinite=error_if_nonfinite)

    def print(self, *a, **k):
        print(*a, **k)


class Shape:
    def __init__(self, shape):
        self.shape = tuple(shape)


class RecordingAggregator:
    disabled = False

    def __init__(self):
        self.values = {}

    def update(self, name, value):
        self.values[name] = float(value)


class NoiseQueue:
    """Replaces torch.multinomial inside the reference with argmax(probs / q) on injected q~Exp(1)
    (SURVEY.md Appendix B: identical to torch's CPU fast path). Pops tensors in call order."""

    def __init__(self, noises):
        self.noises = list(noises)
        self.i = 0
        self._orig = None

    def __enter__(self):
        import torch

        self._orig = torch.multinomial

        def fake(probs, num_samples, replacement=False, *, generator=None, out=None):
            q = self.noises[self.i]
            self.i += 1
            assert q.numel() == probs.numel(), (q.shape, probs.shape, self.i)
            return torch.argmax(probs / q.reshape(probs.shape), dim=-1, keepdim=True)

        torch.multinomial = fake
        return self

    def __exit__(self, *exc):
        import torch

        torch.multinomial = self._orig
        return False
