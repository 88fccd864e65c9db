"""Places the unmodified reference package (Eclectic-Sheep/sheeprl, pure Python) under `oracle/_ref/` (git-ignored) so
that bench.py's baseline arms and the reference-harness tests can execute it on machines that do not have the reference
checkout.  The checkout is taken from $SHEEPRL_REFERENCE_SRC, else from a `reference/` directory next to this
repository, else from /root/reference (where the golden fixtures were generated); without one this is a no-op and
those arms / tests fall back or skip.

    python -m oracle.install_ref
"""
from __future__ import annotations

import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")


def source() -> str | None:
    for p in (os.environ.get("SHEEPRL_REFERENCE_SRC"), os.path.join(os.path.dirname(ROOT), "reference"), "/root/reference"):
        if p and os.path.isfile(os.path.join(p, "sheeprl", "__init__.py")):
            return p
    return None


def install() -> str | None:
    if os.path.isdir(os.path.join(DST, "sheeprl")):
        return DST
    src = source()
    if src is None:
        return None
    tmp = DST + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(os.path.join(src, "sheeprl"), os.path.join(tmp, "sheeprl"),
                    ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    os.replace(tmp, DST)
    return DST


if __name__ == "__main__":
    print(install())
