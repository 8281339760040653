"""Dataset classes with the reference's names, constructor arguments, split / label conventions and cache behaviour
(dance/datasets/base.py:78-158, singlemodality.py, spatial.py; SURVEY App. D) that serve SYNTHETIC data: the reference's
loaders download from the network, which the air-gapped GPU box cannot.  Sizes come from the environment
(``DANCE_B200_SYNTH="cells=10000,genes=2000,types=10"``), the values from :mod:`dance_b200.synth` (a pure function of seed,
cell and gene index).

``load_data(transform, cache)`` follows ``BaseDataset.load_data``: the processed ``Data`` object is pickled to
``<root>/cache/<md5(dataset repr + transform.hexdigest())>.pkl`` (SURVEY §8f row 4) and read back on the next call."""
from __future__ import annotations

import hashlib
import logging
import os
import pickle
from typing import Optional

import numpy as np
import pandas as pd

from . import synth
from .data import AnnDataLite, Data
from .transforms.base import BaseTransform

logger = logging.getLogger("dance_b200.datasets")


def synth_config() -> dict:
    cfg = {"cells": 10000, "genes": 2000, "types": 10, "seed": 0, "density": 0.10}
    for item in filter(None, os.environ.get("DANCE_B200_SYNTH", "").split(",")):
        k, v = item.split("=")
        cfg[k.strip()] = float(v) if k.strip() == "density" else int(v)
    return cfg


class BaseDataset:
    """load_data / cache protocol of dance/datasets/base.py:78-149."""

    def __init__(self, root: str = "./", full_download: bool = False):
        self.root = root

    def hexdigest(self) -> str:
        return hashlib.md5((repr(self) + repr(sorted(synth_config().items()))).encode()).hexdigest()

    def __repr__(self):
        attrs = ", ".join(f"{k}={v!r}" for k, v in sorted(vars(self).items()) if not k.startswith("_"))
        return f"{type(self).__name__}({attrs})"

    def _cache_path(self, transform) -> str:
        cache_dir = os.path.join(self.root, "cache")
        os.makedirs(cache_dir, exist_ok=True)
        key = self.hexdigest() + ("" if transform is None else transform.hexdigest())
        return os.path.join(cache_dir, hashlib.md5(key.encode()).hexdigest() + ".pkl")

    def load_raw_data(self):
        raise NotImplementedError

    def _raw_to_dance(self, raw) -> Data:
        raise NotImplementedError

    def load_data(self, transform: Optional[BaseTransform] = None, cache: bool = False, redo_cache: bool = False) -> Data:
        path = self._cache_path(transform) if cache else None
        if cache and not redo_cache and os.path.isfile(path):
            with open(path, "rb") as f:
                data = pickle.load(f)
            logger.info(f"Loading cached data at {path}")
            return data
        data = self._raw_to_dance(self.load_raw_data())
        if transform is not None:
            if not isinstance(transform, BaseTransform):
                raise TypeError(f"transform has to be inherited from BaseTransform, got {type(transform)}: {transform!r}.")
            transform(data)
        if cache:
            with open(path, "wb") as f:
                pickle.dump(data, f, protocol=pickle.HIGHEST_PROTOCOL)
            logger.info(f"Saved processed data to cache: {path}")
        return data


def _counts(cfg, n=None):
    n = cfg["cells"] if n is None else n
    X = synth.expression_counts(n, cfg["genes"], seed=cfg["seed"], density=cfg["density"], n_types=cfg["types"]).numpy()
    types = synth.cell_types(n, seed=cfg["seed"], n_types=cfg["types"]).numpy()
    var = {"names": np.array([f"Gene{i:05d}" for i in range(cfg["genes"])])}
    return X, types, var


class ImputationDataset(BaseDataset):
    """singlemodality.py:447-580: raw counts, ``Data(adata, train_size=int(n_obs · train_size))``."""

    def __init__(self, data_dir="data", dataset="human_stemcell", train_size=0.1):
        super().__init__(data_dir)
        self.data_dir, self.dataset, self.train_size = data_dir, dataset, train_size

    def load_raw_data(self):
        X, types, var = _counts(synth_config())
        return AnnDataLite(X, obs={"names": np.array([str(i) for i in range(len(X))]), "latent_type": types}, var=var)

    def _raw_to_dance(self, adata):
        return Data(adata, train_size=int(adata.n_obs * self.train_size))


class CellTypeAnnotationDataset(BaseDataset):
    """singlemodality.py:33-347: dense float32 expression, one-hot label DataFrame in ``obsm["cell_type"]``, training cells
    first then test cells (``Data(adata, train_size=n_train, val_size=…)``)."""

    def __init__(self, full_download=False, train_dataset=None, test_dataset=None, species=None, tissue=None, valid_dataset=None,
                 train_dir="train", test_dir="test", valid_dir="valid", map_path="map", data_dir="./", train_as_valid=False,
                 val_size=0.0, test_size=None, filetype: str = "csv"):
        super().__init__(data_dir)
        self.data_dir, self.species, self.tissue = data_dir, species, tissue
        self.train_dataset, self.test_dataset, self.val_size = train_dataset, test_dataset, val_size

    def load_raw_data(self):
        cfg = synth_config()
        X, types, var = _counts(cfg)
        tot = X.sum(1, keepdims=True)
        X = np.log1p(np.where(tot > 0, X * (1e4 / np.maximum(tot, 1e-30)), X)).astype(np.float32)
        labels = pd.DataFrame(np.eye(cfg["types"], dtype=np.float32)[types], columns=[f"type{t}" for t in range(cfg["types"])],
                              index=[str(i) for i in range(len(X))])
        return AnnDataLite(X, obs={"names": np.array([str(i) for i in range(len(X))])}, var=var, obsm={"cell_type": labels})

    def _raw_to_dance(self, adata):
        n = adata.n_obs
        n_test = n // 5
        n_val = int((n - n_test) * self.val_size)
        return Data(adata, train_size=n - n_test - n_val, val_size=n_val, test_size=n_test)


class ClusteringDataset(BaseDataset):
    """singlemodality.py:350-441: labels in ``obsm["Group"]``, ``train_size="all"``."""

    def __init__(self, data_dir: str = "./data", dataset: str = "mouse_bladder_cell"):
        super().__init__(data_dir)
        self.data_dir, self.dataset = data_dir, dataset

    def load_raw_data(self):
        X, types, var = _counts(synth_config())
        return AnnDataLite(X, obs={"names": np.array([str(i) for i in range(len(X))])}, var=var,
                           obsm={"Group": np.asarray(types)})     # a 1-D label vector, as the reference's h5 "Y" (:428-439)

    def _raw_to_dance(self, adata):
        data = Data(adata, train_size="all")
        data.set_config(label_channel="Group")
        return data


class SpatialLIBDDataset(BaseDataset):
    """spatial.py: ``obsm["spatial"]``, ``obsm["spatial_pixel"]``, ``uns["image"]``, ``obs["label"]`` (consumed at
    transforms/graph/spatial_graph.py:17-18,37-39 and spagcn.py:724-729); spots on a jittered hex grid, a smooth random image."""

    def __init__(self, root=".", full_download=False, data_id="151673", data_dir="data/spatial"):
        super().__init__(root)
        self.data_id, self.data_dir = data_id, data_dir

    def load_raw_data(self):
        cfg = synth_config()
        X, types, var = _counts(cfg)
        n = len(X)
        xy = synth.spatial_coordinates(n, seed=cfg["seed"]).numpy().astype(np.float32)
        pix = np.round(xy).astype(np.int64)
        side = int(pix.max()) + 64
        rng = np.random.default_rng(cfg["seed"])
        coarse = rng.random((side // 64 + 2, side // 64 + 2, 3))
        img = (np.kron(coarse, np.ones((64, 64, 1)))[:side, :side] * 255).astype(np.uint8)
        return AnnDataLite(X, obs={"names": np.array([str(i) for i in range(n)]), "label": types}, var=var,
                           obsm={"spatial": xy, "spatial_pixel": pix}, uns={"image": img})

    def _raw_to_dance(self, adata):
        data = Data(adata, train_size="all")
        return data
