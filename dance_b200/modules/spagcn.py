"""SpaGCN on the H100-native kernels — host-side mirror of ``dance/modules/spatial/spatial_domain/spagcn.py``
(GraphConvolution :337-366, SimpleGCDEC :369-584, calculate_p / search_l :249-287, SpaGCN :700-892).

The layer is ``z = adj_exp · (X · W) + b`` with a DENSE ``adj_exp = exp(-D² / 2l²)`` (N×N, ``torch.spmm`` on a dense
matrix at spagcn.py:359).  ``X`` and ``adj_exp`` never change during training, so this implementation builds
``AX = adj_exp · X`` ONCE with the tensor-core GEMM and trains on ``z = AX · W + b`` — the N²·h product leaves the epoch
loop, and the backward pass needs only ``dW = AXᵀ · dz`` (re-association of the same fp32 sums, parity ≤1e-4 pinned by
tests/test_gpu_spagcn.py against the reference's own ``fit``).

Reference quirks reproduced on purpose:
* ``SimpleGCDEC.fit`` creates its optimiser BEFORE ``self.mu`` exists (:464-495), so ``mu`` is never trained there;
  ``fit_with_init`` creates it afterwards and trains ``mu`` too (:544-547).
* ``q**(alpha+1.0)/2.0`` (:395) is ``(q^(alpha+1))/2``, not the Student-t exponent.
* the stop rule (:527-534) compares the labels of consecutive epochs, checked only when ``(epoch-1) % update_interval == 0``.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from .. import ops, spatial_ops
from ..engine import FlatParams
from ..leiden import leiden, neighbor_graph
from ..matrix import SpotDistance


def _dev(a, device, dtype=torch.float32) -> torch.Tensor:
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=dtype).contiguous()
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(device)


def calculate_p(adj, l: float) -> float:
    """``mean_i Σ_j exp(-adj_ij²/2l²) - 1`` (spagcn.py:249-251); one reduction kernel, the N×N exponentials are never stored
    (nor, for a ``SpotDistance``, the distances)."""
    n = adj.shape[0]
    if isinstance(adj, SpotDistance):
        acc = spatial_ops.spatial_exp_adj_sum(*adj.device_coords(), l)
    else:
        _, acc = ops.exp_adj(adj, l, want_matrix=False, want_sum=True)
    return float(acc.item()) / n - 1.0


def search_l(p: float, adj, start: float = 0.01, end: float = 1000, tol: float = 0.01, max_run: int = 100, device="cuda"):
    """Bisection on ``l`` so that ``calculate_p(adj, l) ≈ p`` — same control flow and return values as spagcn.py:254-287."""
    adj = adj if isinstance(adj, SpotDistance) else _dev(adj, device)
    run = 0
    p_low = calculate_p(adj, start)
    p_high = calculate_p(adj, end)
    if p_low > p + tol:
        return None
    elif p_high < p - tol:
        return None
    elif abs(p_low - p) <= tol:
        return start
    elif abs(p_high - p) <= tol:
        return end
    while (p_low + tol) < p < (p_high - tol):
        run += 1
        if run > max_run:
            return None
        mid = (start + end) / 2
        p_mid = calculate_p(adj, mid)
        if abs(p_mid - p) <= tol:
            return mid
        if p_mid <= p:
            start, p_low = mid, p_mid
        else:
            end, p_high = mid, p_mid
    return None


def _refine_labels(pred: torch.Tensor, dis: torch.Tensor, num_nbs: int) -> torch.Tensor:
    """Majority vote over each spot's ``num_nbs`` + 1 nearest spots (itself included), device-agnostic torch:
    relabel when the spot's own label holds fewer than num_nbs/2 of those votes and some label holds more than num_nbs/2
    (spagcn.py:322-333).  ``pred`` int64 labels in 0..K-1; ties in distance go to the lower index (the reference's quicksort
    leaves them unspecified)."""
    return _refine_votes(pred, torch.sort(dis, dim=1, stable=True).indices[:, :num_nbs + 1], num_nbs)


def _refine_votes(pred: torch.Tensor, idx: torch.Tensor, num_nbs: int) -> torch.Tensor:
    """The vote of :func:`_refine_labels` given each spot's nearest spots ``idx`` [n, num_nbs + 1]."""
    votes = torch.nn.functional.one_hot(pred[idx], int(pred.max().item()) + 1).sum(1)
    self_cnt = votes.gather(1, pred.view(-1, 1)).squeeze(1)
    max_cnt, major = votes.max(1)
    flip = (self_cnt < num_nbs / 2) & (max_cnt > num_nbs / 2)
    return torch.where(flip, major, pred)


def refine(sample_id, pred, dis, shape: str = "hexagon"):
    """Optional post-processing of the domain labels (module-level ``refine`` of the reference, spagcn.py:290-334): returns the
    refined labels as a list in ``sample_id`` order.  ``dis`` is the spot-to-spot distance matrix (numpy, tensor or
    ``SpotDistance``; the last ranks the same fp32 distances on the device without forming the matrix)."""
    if shape == "hexagon":
        num_nbs = 6
    elif shape == "square":
        num_nbs = 4
    else:
        raise ValueError("Shape not recognized, shape='hexagon' for Visium data, 'square' for ST data.")   # the reference logs and then fails on an unbound name
    labels, inv = np.unique(np.asarray(pred), return_inverse=True)
    if isinstance(dis, SpotDistance):
        idx = spatial_ops.spatial_nearest(*dis.device_coords(), num_nbs + 1).long()
        out = _refine_votes(torch.as_tensor(inv, dtype=torch.int64, device=idx.device), idx, num_nbs)
        return labels[out.cpu().numpy()].tolist()
    dis_t = (dis if isinstance(dis, torch.Tensor) else torch.as_tensor(np.ascontiguousarray(dis))).to("cuda")   # no CPU path
    out = _refine_labels(torch.as_tensor(inv, dtype=torch.int64, device=dis_t.device), dis_t, num_nbs)
    return labels[out.cpu().numpy()].tolist()


def _fingerprint(a) -> tuple:
    """Cheap content key of an array (shape + a strided sample + two moments): detects in-place mutation between calls without a
    full pass over an N×N matrix."""
    t = a if isinstance(a, torch.Tensor) else np.asarray(a)
    flat = t.reshape(-1)
    n = flat.shape[0]
    step = max(1, n // 4096)
    sample = flat[::step][:4096]
    if isinstance(sample, torch.Tensor):
        sample = sample.detach().double().cpu().numpy()
    sample = np.asarray(sample, dtype=np.float64)
    return (tuple(t.shape), float(sample.sum()), float((sample * sample).sum()), float(sample[-1]) if len(sample) else 0.0)


class SimpleGCDEC:
    """One graph convolution + DEC clustering head; explicit forward/backward on the C-ABI kernels."""

    def __init__(self, nfeat: int, nhid: int, alpha: float = 0.2, device: str = "cuda", precision: Optional[str] = None,
                 seed: Optional[int] = None):
        self.nfeat, self.nhid, self.alpha = int(nfeat), int(nhid), float(alpha)
        self.device = torch.device("cuda" if device in ("cpu", "auto") else device)   # the reference default is "cpu"
        if self.device.type != "cuda":
            raise RuntimeError("dance_b200 runs on CUDA devices only")
        self.precision = precision
        self.params = FlatParams([("gc.weight", (self.nfeat, self.nhid)), ("gc.bias", (self.nhid, ))], self.device)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        stdv = 1.0 / np.sqrt(self.nhid)                                             # GraphConvolution.reset_parameters :351-355
        self.params.p["gc.weight"].copy_((torch.rand((self.nfeat, self.nhid), generator=gen) * 2 - 1) * stdv)
        self.params.p["gc.bias"].copy_((torch.rand((self.nhid, ), generator=gen) * 2 - 1) * stdv)
        self.mu_params: Optional[FlatParams] = None
        self.n_clusters: Optional[int] = None
        self.trajectory = []
        self.epochs_run = 0
        self._bound = None
        self.last_loss: Optional[torch.Tensor] = None

    # ---- parameters -------------------------------------------------------------------------
    @property
    def mu(self) -> torch.Tensor:
        if self.mu_params is None:
            raise AttributeError("mu is determined by fit() (spagcn.py:387)")
        return self.mu_params.p["mu"]

    def set_mu(self, mu):
        mu = _dev(mu, self.device)
        self.n_clusters = int(mu.shape[0])
        self.mu_params = FlatParams([("mu", (self.n_clusters, self.nhid))], self.device)
        self.mu_params.p["mu"].copy_(mu)

    def state_dict(self):
        sd = {k: v.detach().clone() for k, v in self.params.p.items()}
        if self.mu_params is not None:
            sd["mu"] = self.mu.detach().clone()
        return sd

    def load_state_dict(self, sd):
        self.params.p["gc.weight"].copy_(_dev(sd["gc.weight"], self.device))
        self.params.p["gc.bias"].copy_(_dev(sd["gc.bias"], self.device))
        if "mu" in sd:
            self.set_mu(sd["mu"])

    # ---- graph binding ----------------------------------------------------------------------
    def bind(self, X, adj):
        """Upload ``X`` [N, nfeat] and the dense ``adj`` [N, N] and form ``AX = adj · X`` once.  A ``SpotDistance`` ``adj`` (the
        exponentiated form, ``l`` set) forms ``AX`` from the coordinates; its key is the coordinates' digest and ``l``."""
        spots = isinstance(adj, SpotDistance)
        if spots:   # identity AND content: an in-place edit of X / adj re-binds
            key = (id(X), _fingerprint(X), adj.fingerprint())
        else:
            key = (id(X), id(adj), _fingerprint(X), _fingerprint(adj))
        if self._bound is not None and self._bound[0] == key:
            return
        Xd = _dev(X, self.device)
        if spots and adj.l is None:
            raise ValueError("bind: a SpotDistance adjacency must be the exponentiated form (SpaGCN.calc_adj_exp)")
        Ad = adj if spots else _dev(adj, self.device)
        if tuple(Ad.shape) != (Xd.shape[0], Xd.shape[0]) or Xd.shape[1] != self.nfeat:
            raise ValueError(f"bind: X {tuple(Xd.shape)} / adj {tuple(Ad.shape)} do not fit nfeat={self.nfeat}")
        if spots:
            self.AX = spatial_ops.spatial_exp_adj_matmul(*adj.device_coords(self.device), adj.l, Xd)
        else:
            self.AX = ops.gemm(Ad, Xd, precision=self.precision)
        self.n = Xd.shape[0]
        self._bound = (key, X, adj)          # keeps the host objects alive so that id() stays unique
        n, h = self.n, self.nhid
        self._z = torch.empty((n, h), dtype=torch.float32, device=self.device)
        self._dz = torch.empty((n, h), dtype=torch.float32, device=self.device)
        self._labels = torch.empty(n, dtype=torch.int32, device=self.device)
        self._labels_last = torch.empty(n, dtype=torch.int32, device=self.device)
        self._loss = torch.zeros(1, dtype=torch.float32, device=self.device)

    def _features(self) -> torch.Tensor:
        return ops.gemm(self.AX, self.params.p["gc.weight"], bias=self.params.p["gc.bias"], out=self._z, precision=self.precision)

    def forward(self, X, adj) -> Tuple[torch.Tensor, torch.Tensor]:
        self.bind(X, adj)
        z = self._features()
        return z, ops.dec_q(z, self.mu, self.alpha)

    __call__ = forward

    def predict(self, X, adj):
        z, q = self.forward(X, adj)
        return z.clone(), q

    def target_distribution(self, q: torch.Tensor) -> torch.Tensor:
        return ops.dec_target(q)

    def loss_function(self, p: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
        """Forward-only KL (spagcn.py:399-406) on given p/q — diagnostic; training uses the fused loss+gradient kernel."""
        return torch.mean(torch.sum(p * torch.log(p / (q + 1e-6)), dim=1))

    # ---- training ---------------------------------------------------------------------------
    def _init_labels(self, features: torch.Tensor, X, init, n_clusters, n_neighbors, res, init_spa, init_labels):
        if init_labels is not None:
            return np.asarray(init_labels).astype(np.int64)
        if init == "kmeans":   # same third-party call as the reference (:471-480); initialisation only, not the hot path
            base = features.cpu().numpy() if init_spa else np.asarray(X, dtype=np.float32)
            from sklearn.cluster import KMeans
            return KMeans(int(n_clusters), n_init=20).fit_predict(base).astype(np.int64)
        if init == "louvain":   # sc.pp.neighbors(n_neighbors, use_rep="X") + sc.tl.leiden(resolution=res) (:481-492), on the device
            X0 = features if init_spa else _dev(X, self.device)
            labels = leiden(neighbor_graph(X0.contiguous(), int(n_neighbors)), resolution=float(res)).labels
            return labels.cpu().numpy().astype(np.int64)
        raise ValueError(f"unknown init {init!r}")

    def _centers(self, features: torch.Tensor, y: np.ndarray) -> torch.Tensor:
        """Group means in sorted-label order (``Mergefeature.groupby("Group").mean()``, :499-503)."""
        uniq, inv = np.unique(y, return_inverse=True)
        inv_d = torch.as_tensor(inv, dtype=torch.int64, device=self.device)
        sums = torch.zeros((len(uniq), features.shape[1]), dtype=torch.float64, device=self.device)
        sums.index_add_(0, inv_d, features.double())
        cnt = torch.bincount(inv_d, minlength=len(uniq)).double().unsqueeze(1)
        return (sums / cnt).float()

    def _step(self, p: torch.Tensor, opt: str, lr: float, weight_decay: float, train_mu: bool):
        P, G = self.params.p, self.params.g
        z = self._features()
        ops.dec_kl_grad(z, self.mu, p, self.alpha, dz=self._dz, dmu=self.mu_params.g["mu"], loss=self._loss,
                        labels_out=self._labels)
        ops.gemm(self.AX, self._dz, transA=True, out=G["gc.weight"], precision=self.precision)
        ops.colsum(self._dz, out=G["gc.bias"])
        buckets = [self.params] + ([self.mu_params] if train_mu else [])
        for b in buckets:
            if opt == "sgd":
                b.step += 1
                ops.sgd_momentum_step(b.flat, b.grad, b.exp_avg, b.step, lr, 0.9, 0.0)
            else:
                b.adam_step(lr, weight_decay=weight_decay)
        self.last_loss = self._loss

    def _reset_optim(self):
        for b in (self.params, self.mu_params):
            if b is not None:
                b.step = 0
                b.exp_avg.zero_()
                b.exp_avg_sq.zero_()

    def fit(self, X, adj, lr=0.001, epochs=5000, update_interval=3, trajectory_interval=50, weight_decay=5e-4, opt="sgd",
            init="louvain", n_neighbors=10, res=0.4, n_clusters=10, init_spa=True, tol=1e-3, init_labels=None):
        """Mirror of ``SimpleGCDEC.fit`` (spagcn.py:427-539); ``init_labels`` bypasses the kmeans / leiden initialisation."""
        if opt not in ("sgd", "admin"):
            raise ValueError("opt must be 'sgd' or 'admin'")
        self.trajectory = []
        self.bind(X, adj)
        features = self._features()
        y_pred = self._init_labels(features, X, init, n_clusters, n_neighbors, res, init_spa, init_labels)
        self.set_mu(self._centers(features, y_pred))
        self.trajectory.append(y_pred)
        self._labels_last.copy_(torch.as_tensor(y_pred, dtype=torch.int32))
        self._reset_optim()
        p = None
        self.epochs_run = 0
        for epoch in range(epochs):
            if epoch % update_interval == 0:
                p = ops.dec_target(ops.dec_q(self._features(), self.mu, self.alpha))
            self._step(p, opt, lr, weight_decay, train_mu=False)
            self.epochs_run = epoch + 1
            if epoch % trajectory_interval == 0:
                self.trajectory.append(self._labels.cpu().numpy().astype(np.int64))
            check = epoch > 0 and (epoch - 1) % update_interval == 0
            if check:
                delta_label = float((self._labels != self._labels_last).sum().item()) / self.n
                if delta_label < tol:
                    break
            self._labels, self._labels_last = self._labels_last, self._labels
        return self

    def fit_with_init(self, X, adj, init_y, lr=0.001, epochs=5000, update_interval=1, weight_decay=5e-4, opt="sgd"):
        """Mirror of ``fit_with_init`` (spagcn.py:541-579): centres from ``init_y``, then every parameter incl. mu is trained."""
        if self.mu_params is None:
            raise AttributeError("fit_with_init needs an existing mu (the reference fails the same way, spagcn.py:555)")
        self.bind(X, adj)
        features = self._features()
        self.mu.copy_(self._centers(features, np.asarray(init_y)))
        self._reset_optim()
        p = None
        for epoch in range(epochs):
            if epoch % update_interval == 0:
                p = ops.dec_target(ops.dec_q(self._features(), self.mu, self.alpha))
            self._step(p, opt, lr, weight_decay, train_mu=True)
        return self


class SpaGCN:
    """Mirror of the reference ``SpaGCN`` clustering method (spagcn.py:700-892)."""

    def __init__(self, l: Optional[float] = None, device: str = "cuda", precision: Optional[str] = None, seed: Optional[int] = None):
        self.l, self.res = l, None
        self.device = "cuda" if device in ("cpu", "auto") else device
        self.precision, self.seed = precision, seed
        self.model: Optional[SimpleGCDEC] = None

    @staticmethod
    def preprocessing_pipeline(alpha: float = 1, beta: int = 49, dim: int = 50, log_level="INFO", dense: bool = True):
        """The reference's pipeline (spagcn.py:716-731); ``dense=False`` makes both graph transforms store the coordinate-backed
        ``SpotDistance`` instead of the N×N matrices."""
        from ..transforms import AnnDataTransform, CellPCA, Compose, FilterGenesMatch, SetConfig
        from ..transforms.graph import SpaGCNGraph, SpaGCNGraph2D
        return Compose(
            FilterGenesMatch(prefixes=["ERCC", "MT-"]),
            AnnDataTransform("scanpy.pp.normalize_total", target_sum=1e4),
            AnnDataTransform("scanpy.pp.log1p"),
            SpaGCNGraph(alpha=alpha, beta=beta, dense=dense),
            SpaGCNGraph2D(dense=dense),
            CellPCA(n_components=dim),
            SetConfig({
                "feature_channel": ["CellPCA", "SpaGCNGraph", "SpaGCNGraph2D"],
                "feature_channel_type": ["obsm", "obsp", "obsp"],
                "label_channel": "label",
                "label_channel_type": "obs"
            }),
            log_level=log_level,
        )

    def search_l(self, p, adj, start=0.01, end=1000, tol=0.01, max_run=100):
        return search_l(p, adj, start, end, tol, max_run, device=self.device)

    def set_l(self, l):
        self.l = l

    def search_set_res(self, x, l, target_num, start=0.4, step=0.1, tol=5e-3, lr=0.05, epochs=10, max_run=10):
        """Search the leiden resolution that yields ``target_num`` domains (spagcn.py:771-805; same control flow).  Each step fits
        with ``init="louvain"``, i.e. the device neighbour graph and Leiden (:mod:`dance_b200.leiden`)."""
        res = start
        clf = SpaGCN(l, device=self.device, precision=self.precision, seed=self.seed)
        old_num = len(set(clf.fit_predict(x, init_spa=True, init="louvain", res=res, tol=tol, lr=lr, epochs=epochs)))
        run = 0
        while old_num != target_num:
            old_sign = 1 if (old_num < target_num) else -1
            clf = SpaGCN(l, device=self.device, precision=self.precision, seed=self.seed)
            new_num = len(set(clf.fit_predict(x, init_spa=True, init="louvain", res=res + step * old_sign, tol=tol, lr=lr, epochs=epochs)))
            if new_num == target_num:
                res = res + step * old_sign
                return res
            new_sign = 1 if (new_num < target_num) else -1
            if new_sign == old_sign:
                res = res + step * old_sign
                old_num = new_num
            else:
                step = step / 2
            if run > max_run:
                return res
            run += 1
        self.res = res
        return res

    def calc_adj_exp(self, adj) -> torch.Tensor:
        """``exp(-adj²/(2 l²))`` on the device (spagcn.py:807-809); returns a CUDA tensor (the reference returns numpy), or for a
        ``SpotDistance`` its exponentiated form, still unmaterialised."""
        if isinstance(adj, SpotDistance):
            return adj.exp(self.l)
        out, _ = ops.exp_adj(_dev(adj, self.device), self.l, want_matrix=True, want_sum=False)
        return out

    def fit(self, x, y=None, *, num_pcs=50, lr=0.005, epochs=2000, weight_decay=0, opt="admin", init_spa=True, init="louvain",
            n_neighbors=10, n_clusters=None, res=0.4, tol=1e-3, init_labels=None):
        embed, adj = x
        self.num_pcs, self.res, self.lr, self.epochs, self.weight_decay, self.opt = num_pcs, res, lr, epochs, weight_decay, opt
        self.init_spa, self.init, self.n_neighbors, self.n_clusters, self.tol = init_spa, init, n_neighbors, n_clusters, tol
        if self.l is None:
            raise ValueError("l should be set before fitting the model!")
        self.model = SimpleGCDEC(embed.shape[1], embed.shape[1], device=self.device, precision=self.precision, seed=self.seed)
        self._adj_exp = self.calc_adj_exp(adj)
        self._fit_inputs = (embed, adj)
        self.model.fit(embed, self._adj_exp, lr=lr, epochs=epochs, weight_decay=weight_decay, opt=opt, init_spa=init_spa, init=init,
                       n_neighbors=n_neighbors, n_clusters=n_clusters, res=res, tol=tol, init_labels=init_labels)
        return self

    def predict_proba(self, x) -> torch.Tensor:
        embed, adj = x
        if getattr(self, "_fit_inputs", None) is not None and embed is self._fit_inputs[0] and adj is self._fit_inputs[1]:
            adj_exp = self._adj_exp                       # same objects as fit(): AX is still bound
        else:
            adj_exp = self.calc_adj_exp(adj)
        _, q = self.model.predict(embed, adj_exp)
        return q

    def predict(self, x) -> np.ndarray:
        return torch.argmax(self.predict_proba(x), dim=1).cpu().numpy()

    def fit_predict(self, x, y=None, **fit_kwargs) -> np.ndarray:
        self.fit(x, y, **fit_kwargs)
        return self.predict(x)

    @staticmethod
    def default_score_func(y_true, y_pred) -> float:
        """Adjusted Rand index (``BaseClusteringMethod._DEFAULT_METRIC = "ari"``, modules/base.py:46-47,168)."""
        from sklearn.metrics import adjusted_rand_score
        return float(adjusted_rand_score(np.asarray(y_true), np.asarray(y_pred)))

    def score(self, x, y, score_func=None) -> float:
        """Adjusted Rand index by default (``default_score_func``)."""
        pred = self.predict(x)
        return float((score_func or self.default_score_func)(np.asarray(y), pred))

    def fit_score(self, x, y, score_func=None, **fit_kwargs) -> float:
        self.fit(x, y, **fit_kwargs)
        return self.score(x, y, score_func)
