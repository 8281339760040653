"""Minimal stand-ins for ``anndata.AnnData`` and ``dance.data.Data`` — just the surface the hot-path
transforms and models touch (SURVEY App. D; reference dance/data/base.py:84-108, 131-168, 203-272, 415-475,
817-851).  When the real ``anndata`` is importable, pass a real AnnData: ``Data`` only uses attribute access.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Union

import numpy as np
import scipy.sparse as sp
import torch

from .matrix import SpotDistance


class AnnDataLite:
    """Attribute bag with the AnnData field names (X, obs, var, obsm, varm, obsp, varp, layers, uns).

    ``X`` may live on the DEVICE between operators: a transform that computes on the GPU takes ``device_X()`` and hands its
    result back with ``set_device_X()``; the host copy is only rebuilt when somebody reads ``.X`` (a Compose of k device
    operators moves the N×G matrix over PCIe once in and once out instead of 2k times).  ``layers`` entries may be device
    tensors as well (``get_layer_host`` materialises them)."""

    def __init__(self, X, obs=None, var=None, obsm=None, varm=None, obsp=None, varp=None, layers=None, uns=None):
        self._X_host, self._X_dev = None, None
        self.X = X
        n, g = X.shape
        self.obs = obs if obs is not None else {}
        self.var = var if var is not None else {}
        # like AnnData: positional string names are fixed at construction and survive subsetting
        if isinstance(self.obs, dict) and "names" not in self.obs:
            self.obs["names"] = np.array([str(i) for i in range(n)])
        if isinstance(self.var, dict) and "names" not in self.var:
            self.var["names"] = np.array([str(i) for i in range(g)])
        self.obsm, self.varm = dict(obsm or {}), dict(varm or {})
        self.obsp, self.varp = dict(obsp or {}), dict(varp or {})
        self.layers, self.uns = _LazyHostDict(layers or {}), dict(uns or {})

    # ---- X: host view with an optional device-resident master copy -------------------------------------------------------
    @property
    def X(self):
        if self._X_host is None and self._X_dev is not None:
            self._X_host = self._X_dev.cpu().numpy()
        return self._X_host

    @X.setter
    def X(self, value):
        if isinstance(value, torch.Tensor) and value.is_cuda:
            self._X_dev, self._X_host = value, None
        else:
            self._X_host, self._X_dev = value, None

    def device_X(self, device=None) -> torch.Tensor:
        """float32 CUDA tensor of X (uploaded once; later device operators reuse it)."""
        if self._X_dev is None:
            if not torch.cuda.is_available():
                raise RuntimeError("dance_b200 needs a CUDA device (there is no CPU fallback)")
            X = self._X_host
            if sp.issparse(X):
                X = X.toarray()
            self._X_dev = torch.as_tensor(np.ascontiguousarray(X, dtype=np.float32)).to(device or "cuda")
        return self._X_dev

    def set_device_X(self, t: torch.Tensor):
        """Install a device result as the new X; the host copy becomes stale and is rebuilt on the next ``.X`` read."""
        self._X_dev, self._X_host = t, None

    @property
    def n_obs(self):
        return self.shape[0]

    @property
    def n_vars(self):
        return self.shape[1]

    @property
    def shape(self):
        return tuple((self._X_dev if self._X_dev is not None else self._X_host).shape)

    def copy(self):
        import copy
        new = copy.copy(self)
        new._X_host = None if self._X_host is None else self._X_host.copy()
        new._X_dev = None if self._X_dev is None else self._X_dev.clone()
        for k in ("obs", "var", "obsm", "varm", "obsp", "varp", "uns"):
            setattr(new, k, copy.deepcopy(getattr(self, k)))
        new.layers = _LazyHostDict({k: (v.clone() if isinstance(v, torch.Tensor) else copy.deepcopy(v)) for k, v in self.layers.raw_items()})
        return new

    def __getstate__(self):
        # pickling (the reference caches the whole Data object, datasets/base.py:117-120): everything on the host
        d = dict(self.__dict__)
        d["_X_host"], d["_X_dev"] = self.X, None
        d["layers"] = _LazyHostDict({k: self.layers[k] for k in self.layers})
        return d

    def _names(self, table, n, key="names"):
        import pandas as pd
        if hasattr(table, "index"):
            return pd.Index(table.index.astype(str))
        if isinstance(table, dict) and key in table:
            return pd.Index(np.asarray(table[key]).astype(str))
        return pd.Index([str(i) for i in range(n)])

    @property
    def var_names(self):
        """Gene identifiers: ``var["names"]`` (or the index of a DataFrame ``var``); defaults to "0".."g-1"."""
        return self._names(self.var, self.n_vars)

    @property
    def obs_names(self):
        return self._names(self.obs, self.n_obs)

    def _positions(self, index, names):
        index = np.asarray(index)
        if index.dtype == bool:
            return np.flatnonzero(index)
        if index.dtype.kind in "iu":
            return index.astype(np.int64)
        keep = names.get_indexer(index.astype(str))
        if (keep < 0).any():
            raise KeyError("unknown names in subset")
        return keep.astype(np.int64)

    @staticmethod
    def _take(table, keep, n):
        if hasattr(table, "iloc"):
            return table.iloc[keep]
        if isinstance(table, dict):
            return {k: (np.asarray(v)[keep] if np.ndim(v) >= 1 and len(v) == n else v) for k, v in table.items()}
        return table

    def _subset_X(self, rows=None, cols=None):
        if self._X_dev is not None:
            from . import ops
            dev = self._X_dev.device
            r = None if rows is None else torch.as_tensor(rows, dtype=torch.int64, device=dev)
            c = None if cols is None else torch.as_tensor(cols, dtype=torch.int32, device=dev)
            self.set_device_X(ops.subset(self._X_dev, r, c))
        else:
            X = self._X_host
            X = X if rows is None else X[rows]
            self._X_host = X if cols is None else X[:, cols]

    def _inplace_subset_var(self, index):
        """Keep the genes selected by a boolean mask, integer positions or names, in the order given (AnnData._inplace_subset_var)."""
        g = self.n_vars
        keep = self._positions(index, self.var_names)
        self._subset_X(cols=keep)
        self.var = self._take(self.var, keep, g)
        self.varm = {k: self._take(v, keep, g) if hasattr(v, "iloc") else v[keep] for k, v in self.varm.items()}
        self.varp = {k: v[keep][:, keep] for k, v in self.varp.items()}
        self.layers = _LazyHostDict({k: (v[:, torch.as_tensor(keep, device=v.device)] if isinstance(v, torch.Tensor) else v[:, keep])
                                     for k, v in self.layers.raw_items()})

    def _inplace_subset_obs(self, index):
        """Keep the cells selected by a boolean mask, integer positions or names (AnnData._inplace_subset_obs)."""
        n = self.n_obs
        keep = self._positions(index, self.obs_names)
        self._subset_X(rows=keep)
        self.obs = self._take(self.obs, keep, n)
        self.obsm = {k: self._take(v, keep, n) if hasattr(v, "iloc") else v[keep] for k, v in self.obsm.items()}
        self.obsp = {k: v[keep][:, keep] for k, v in self.obsp.items()}
        self.layers = _LazyHostDict({k: (v[torch.as_tensor(keep, device=v.device)] if isinstance(v, torch.Tensor) else v[keep])
                                     for k, v in self.layers.raw_items()})


class _LazyHostDict(dict):
    """``layers`` container: values may be device tensors (masks written by CellwiseMaskData); reading an entry returns the host
    ndarray the reference's callers expect (converted once and cached), ``raw_items`` gives the stored objects."""

    def __getitem__(self, k):
        v = dict.__getitem__(self, k)
        if isinstance(v, torch.Tensor):
            v = v.cpu().numpy()
            dict.__setitem__(self, k, v)
        return v

    def get(self, k, default=None):
        return self[k] if k in self else default

    def raw(self, k):
        return dict.__getitem__(self, k)

    def raw_items(self):
        return [(k, dict.__getitem__(self, k)) for k in self.keys()]

    def items(self):
        return [(k, self[k]) for k in self.keys()]

    def values(self):
        return [self[k] for k in self.keys()]


_CONFIG_KEYS = ("feature_mod", "feature_channel", "feature_channel_type", "label_mod", "label_channel", "label_channel_type")


class Data:
    """``dance.data.Data`` stand-in: holds a reference to the AnnData(-like) object, contiguous
    train | val | test splits, the ``dance_config`` dict and the typed accessors."""

    def __init__(self, data, train_size: Optional[Union[int, str]] = None, val_size: int = 0, test_size: int = -1):
        self._data = data
        if "dance_config" not in data.uns:
            data.uns["dance_config"] = {}
        self._split_idx_dict: Dict[str, List[int]] = {}
        n = data.shape[0]
        if train_size == "all":
            self._split_idx_dict["train"] = list(range(n))
        elif train_size is not None:
            sizes = {"train": train_size, "val": val_size, "test": test_size}
            if list(sizes.values()).count(-1) > 1:
                raise ValueError("Only one split size may be -1")
            known = sum(v for v in sizes.values() if v != -1)
            sizes = {k: (n - known if v == -1 else v) for k, v in sizes.items()}
            start = 0
            for k in ("train", "val", "test"):
                self._split_idx_dict[k] = list(range(start, start + sizes[k]))
                start += sizes[k]

    # -- AnnData mirrors ---------------------------------------------------------
    @property
    def data(self):
        return self._data

    @property
    def config(self) -> Dict[str, Any]:
        return self._data.uns["dance_config"]

    @property
    def shape(self):
        return self._data.shape

    @property
    def num_cells(self):
        return self._data.shape[0]

    @property
    def num_features(self):
        return self._data.shape[1]

    def get_split_idx(self, name: str, error_on_miss: bool = False):
        if name in self._split_idx_dict:
            return self._split_idx_dict[name]
        if error_on_miss:
            raise KeyError(f"Unknown split {name!r}. Please set the split inddices via set_split_idx first.")
        return None

    def set_split_idx(self, name: str, idx: Sequence[int]):
        self._split_idx_dict[name] = list(idx)

    def filter_by_mask(self, mask, update_splits: bool = True):
        """Keep the cells where ``mask`` is True and renumber the split indices accordingly (data/base.py:694-770)."""
        mask = np.asarray(mask)
        if mask.dtype != bool:
            raise ValueError(f"Mask must be boolean, got dtype {mask.dtype}")
        if len(mask) != self.shape[0]:
            raise ValueError(f"Mask length ({len(mask)}) must match number of cells ({self.shape[0]})")
        if mask.all():
            return self
        new_pos = np.cumsum(mask) - 1
        self._data._inplace_subset_obs(mask)
        if update_splits:
            self._split_idx_dict = {k: [int(new_pos[i]) for i in v if mask[i]] for k, v in self._split_idx_dict.items()}
        return self

    train_idx = property(lambda self: self.get_split_idx("train"))
    val_idx = property(lambda self: self.get_split_idx("val"))
    test_idx = property(lambda self: self.get_split_idx("test"))

    # -- config --------------------------------------------------------------------
    def set_config(self, *, overwrite: bool = False, **kwargs):
        self.set_config_from_dict(kwargs, overwrite=overwrite)

    def set_config_from_dict(self, config_dict: Dict[str, Any], *, overwrite: bool = False):
        for k, v in config_dict.items():
            if k not in _CONFIG_KEYS:
                raise KeyError(f"Unknown config option {k!r}, available options are {_CONFIG_KEYS}")
            if k in self.config and self.config[k] != v and not overwrite:
                raise KeyError(f"Config option {k!r} already set to {self.config[k]!r}; pass overwrite=True to replace it")
            self.config[k] = v

    # -- accessors -------------------------------------------------------------------
    def get_feature(self, *, split_name: Optional[str] = None, return_type: str = "numpy", channel: Optional[str] = None,
                    channel_type: Optional[str] = "obsm", mod: Optional[str] = None):
        if mod is not None:
            raise NotImplementedError("multi-modal (MuData) access is out of scope (SURVEY §2)")
        if channel is None:
            feature = self._data.X
            channel_type = "X"
        else:
            channel_type = channel_type or "obsm"
            if channel_type == "X":
                feature = self._data.X
            else:
                feature = getattr(self._data, channel_type)[channel]
        if return_type == "default":
            if split_name is not None:
                raise ValueError("split_name is not supported when return_type='default'")
            return feature
        if channel_type == "uns" and not (sp.issparse(feature) or isinstance(feature, (np.ndarray, torch.Tensor))):
            # an object kept in uns (graph-sc's CellFeatureGraph) is handed over as it is: the reference indexes no uns entry by
            # split and leaves a non-array one unconverted (data/base.py:454-467)
            return feature
        if isinstance(feature, SpotDistance):   # handed through unmaterialised unless a torch / sparse matrix is asked for
            if split_name is not None:
                idx = self.get_split_idx(split_name, error_on_miss=True)
                feature = feature[idx][:, idx] if channel_type == "obsp" else feature[idx]
            if return_type == "numpy":
                return feature
            feature = feature.toarray()
        if return_type == "sparse":
            feature = sp.csr_matrix(feature)
        else:
            if sp.issparse(feature):
                feature = feature.toarray()
            elif hasattr(feature, "values") and not isinstance(feature, (np.ndarray, torch.Tensor)):
                feature = feature.values
            feature = np.asarray(feature) if not isinstance(feature, torch.Tensor) else feature
        if split_name is not None:
            idx = self.get_split_idx(split_name, error_on_miss=True)
            feature = feature[idx][:, idx] if channel_type == "obsp" else feature[idx]
        if return_type == "torch" and not isinstance(feature, torch.Tensor):
            feature = torch.from_numpy(np.ascontiguousarray(feature))
        return feature

    def _get(self, kind: str, split_name, return_type):
        mods = self.config.get(f"{kind}_mod")
        channels = self.config.get(f"{kind}_channel")
        types = self.config.get(f"{kind}_channel_type")
        if isinstance(channels, list):
            n = len(channels)
            types = types if isinstance(types, list) else [types] * n
            return [self.get_feature(split_name=split_name, return_type=return_type, channel=c, channel_type=t) for c, t in zip(channels, types)]
        return self.get_feature(split_name=split_name, return_type=return_type, channel=channels, channel_type=types, mod=mods)

    def get_x(self, split_name: Optional[str] = None, return_type: str = "numpy"):
        return self._get("feature", split_name, return_type)

    def get_y(self, split_name: Optional[str] = None, return_type: str = "numpy"):
        return self._get("label", split_name, return_type)

    def get_data(self, split_name: Optional[str] = None, return_type: str = "numpy"):
        """(features, labels) of a split (data/base.py get_data)."""
        return self.get_x(split_name, return_type), self.get_y(split_name, return_type)

    def get_train_data(self, return_type: str = "numpy"):
        return self.get_data("train", return_type)
