"""Make the unmodified reference example scripts importable against this package.

``install()`` puts ``dance_b200/shims`` on ``sys.path`` — a ``dance`` package with the reference's module tree whose leaves
re-export the H100-native classes, and a minimal ``scanpy`` exposing the ``pp`` functions the examples pass to
``AnnDataTransform`` — unless real ``dance`` / ``scanpy`` installations are importable.  ``run_example(path, argv)`` then
executes a script such as ``examples/single_modality/imputation/scgnn2.py`` as ``__main__``.

    python -m dance_b200.dropin /path/to/examples/single_modality/imputation/scgnn2.py --total_epoch 2 ...
"""
from __future__ import annotations

import importlib.util
import runpy
import sys
from pathlib import Path

SHIMS = Path(__file__).resolve().parent / "shims"


def install(force: bool = False) -> list:
    added = []
    for name in ("dance", "scanpy"):
        spec = None
        try:
            spec = importlib.util.find_spec(name)
        except (ImportError, ValueError):
            spec = None
        ours = spec is not None and spec.origin is not None and str(SHIMS) in str(spec.origin)
        if spec is None or ours or force:
            added.append(name)
    if added and str(SHIMS) not in sys.path:
        sys.path.insert(0, str(SHIMS))
    return added


def run_example(path: str, argv=()):
    install()
    old = sys.argv
    sys.argv = [str(path), *map(str, argv)]
    try:
        return runpy.run_path(str(path), run_name="__main__")
    finally:
        sys.argv = old


if __name__ == "__main__":
    if len(sys.argv) < 2:
        raise SystemExit("usage: python -m dance_b200.dropin <example.py> [script arguments]")
    run_example(sys.argv[1], sys.argv[2:])
