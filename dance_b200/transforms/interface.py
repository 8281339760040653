"""``AnnDataTransform(func, **kwargs)`` (reference dance/transforms/interface.py:9-68).  ``func`` may be a
callable or a dotted name; the scanpy functions the pipelines call (``scanpy.pp.normalize_total``, ``log1p``,
``filter_genes``, ``filter_cells`` and ``highly_variable_genes``) are dispatched to the GPU implementations in
:mod:`dance_b200.transforms.pp`, by name, whether or not scanpy itself is installed."""
from __future__ import annotations

import importlib
from typing import Callable, Union

from . import pp
from .base import BaseTransform

_GPU_DISPATCH = {"scanpy.pp.normalize_total": pp.normalize_total, "scanpy.pp.log1p": pp.log1p,
                 "scanpy.preprocessing._normalization.normalize_total": pp.normalize_total,
                 "scanpy.preprocessing._simple.log1p": pp.log1p,
                 "scanpy.pp.filter_genes": pp.filter_genes, "scanpy.pp.filter_cells": pp.filter_cells,
                 "scanpy.preprocessing._simple.filter_genes": pp.filter_genes, "scanpy.preprocessing._simple.filter_cells": pp.filter_cells,
                 "scanpy.pp.highly_variable_genes": pp.highly_variable_genes,
                 "scanpy.preprocessing._highly_variable_genes.highly_variable_genes": pp.highly_variable_genes}


class AnnDataTransform(BaseTransform):
    _DISPLAY_ATTRS = ("func", "func_kwargs")

    def __init__(self, func: Union[Callable, str], **kwargs):
        super().__init__()
        self.func = func
        self.func_kwargs = kwargs

    @property
    def func(self) -> Callable:
        return self._func

    @func.setter
    def func(self, func: Union[Callable, str]):
        if isinstance(func, str):
            if func in _GPU_DISPATCH:
                self._display_name = func
                self._func = _GPU_DISPATCH[func]
                return
            func_scope, func_name = func.rsplit(".", 1)
            func = getattr(importlib.import_module(func_scope), func_name)
        if not callable(func):
            raise TypeError(f"Interfaced function must be callable, got {type(func)}: {func!r}")
        full = f"{func.__module__}.{func.__name__}"
        self._display_name = full
        self._func = _GPU_DISPATCH.get(full, func)

    def __repr__(self):
        return f"{self.name}(func={self._display_name}, func_kwargs={self.func_kwargs})"

    def __call__(self, data):
        self.func(data.data, **self.func_kwargs)
