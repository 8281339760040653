"""scGNN 2.0 on the H100-native engines — host-side mirror of the reference module
``dance/modules/single_modality/imputation/scgnn2.py`` for the stages on the hot path.

Same names, argument meaning and return types as the reference:
  * ``ScGNN2(args, device).fit(x) / .predict() / .score(...)``          scgnn2.py:22-121
  * ``feature_AE_handler(X, TRS, args, param, model_state)``            scgnn2.py:275-335
  * ``graph_AE_handler(X_embed, CCC_graph, args, param)``               scgnn2.py:530-600
numpy in / numpy out at this boundary, everything in between stays in HBM.

  * ``clustering_handler`` / ``graph_celltype_regu_handler`` / ``cluster_AE_handler``       scgnn2.py:138-216, 716-752, 821-880
numpy in / numpy out at this boundary, everything in between stays in HBM.

Differences that are deliberate and documented in DESIGN.md:
  * the N×N decoder logits, the dense label matrix (scgnn2.py:557) and ``recon_graph`` are never
    materialised; ``graph_AE_handler`` returns the ``edgeList`` as an [N·k, 2] index array plus a
    weight array instead of a Python list of tuples, and ``CCC_graph_hat`` as None above
    ``dense_recon_max_cells`` cells;
  * the EM iterations never form the two dense N×N regulariser matrices of ``graph_celltype_regu_handler``: the Cluster-AE
    loss only needs their column sums inside each cluster (``ops.graph_regu_weights`` — including the reference's
    np.matrix-product quirk that makes the "normalised adjacency" deg_j / deg_i); Louvain runs in host C++ on the
    sparse graph (the reference densifies it for igraph), KMeans as Lloyd iterations on the device seeded by sklearn's
    k-means++ (same ``random_state=0``; above ``kmeans_init_max_cells`` cells on a fixed-seed subsample).
"""
from __future__ import annotations

import logging
from time import time
from typing import Any, Optional

import numpy as np
import torch

from .. import hostio, ops
from ..engine import FeatureAEEngine, GATEngine, GraphAEEngine

logger = logging.getLogger("dance_b200.scgnn2")


def _device(device: str = "auto") -> torch.device:
    if device in ("auto", "cuda", None):
        if not torch.cuda.is_available():
            raise RuntimeError("dance_b200 needs a CUDA device (there is no CPU fallback)")
        return torch.device("cuda", torch.cuda.current_device())
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"dance_b200 runs on CUDA devices only, got {device!r}")
    return dev


def feature_AE_handler(X, TRS, args, param, model_state=None):
    """Feature autoencoder stage (scgnn2.py:275-335): returns (X_embed, X_recon, checkpoint)."""
    logger.info("Starting Feature AE")
    dev = param["device"]
    batch_size = args.feature_AE_batch_size
    total_epoch = args.feature_AE_epoch[param["epoch_num"] > 0]
    p_drop = float(args.feature_AE_dropout_prob or 0.0)        # train_handler's masked_prob: F.dropout on the network input (scgnn2.py:1256)
    if getattr(args, "feature_AE_concat_prev_embed", None) and param["epoch_num"] > 0:
        raise NotImplementedError("feature_AE_concat_prev_embed is not built")
    pool = param.get("io_pool")
    resident = isinstance(X, torch.Tensor) and X.is_cuda
    if resident:                                   # already in HBM (EM iterations hand device tensors from stage to stage)
        Xd, host = X.float().contiguous(), None
    else:
        host = hostio.as_host_tensor(X)
        Xd = torch.empty(host.shape, dtype=torch.float32, device=dev)
    n, dim = Xd.shape
    ltmg = None
    if TRS is not None and np.any(TRS):
        ltmg = torch.as_tensor(TRS, dtype=torch.float32).to(dev)
    eng = FeatureAEEngine(dim, device=dev, lr=args.feature_AE_learning_rate, precision=param.get("precision"), seed=param.get("seed"))
    if param["epoch_num"] > 0 and model_state is not None:
        eng.load_state_dict(model_state["model"])
    # regu_type=["LTMG", "noregu"][epoch_num > 0]   (scgnn2.py:314)
    regu = "noregu" if param["epoch_num"] > 0 else "LTMG"
    batches = [(b0, min(n, b0 + batch_size)) for b0 in range(0, n, batch_size)]
    z_all = torch.empty(n, eng.EMB, dtype=torch.float32, device=dev)
    keep_dev = bool(param.get("keep_on_device"))          # EM loop: outputs stay in HBM, nothing is copied back
    recon_dev = torch.empty(n, dim, dtype=torch.float32, device=dev) if keep_dev else None
    recon_host = None if keep_dev else hostio.pinned_empty(pool, "feature_recon", (n, dim))
    up = hostio.Uploader(host, dev, pool, max_rows=batch_size) if host is not None else None
    down = None if keep_dev else hostio.Downloader(dev)
    main = torch.cuda.current_stream(dev)
    if total_epoch == 0:
        raise ValueError("feature_AE_epoch must be >= 1 (the reference's train_handler returns the last epoch's outputs)")
    for epoch in range(total_epoch):
        first, last = epoch == 0 and up is not None, epoch == total_epoch - 1
        eng.loss_acc.zero_()
        ready, queued = {}, 0
        lookahead = len(batches) if (up is not None and up.pinned) else 2
        slot_busy = [None, None]
        for b, (b0, b1) in enumerate(batches):
            if first:                                     # epoch 0 streams X in: batch b trains while b+1.. are in flight
                while queued < min(len(batches), b + 1 + lookahead):
                    q0, q1 = batches[queued]
                    ready[queued] = up.copy_rows(q0, q1, Xd[q0:q1])
                    queued += 1
                main.wait_event(ready.pop(b))
            slot = b & 1
            if slot_busy[slot] is not None:               # the download of batch b-2's reconstruction has left this buffer set
                main.wait_event(slot_busy[slot])
                slot_busy[slot] = None
            z, r = eng.train_step(Xd[b0:b1], None if ltmg is None else ltmg[b0:b1], args.feature_AE_regu_strength, regu, slot=slot,
                                  x_input=eng.input_dropout(Xd[b0:b1], p_drop) if p_drop > 0.0 else None)
            if last:
                z_all[b0:b1].copy_(z)
                if keep_dev:
                    recon_dev[b0:b1].copy_(r)
                else:
                    slot_busy[slot] = down.copy(r, recon_host[b0:b1])
        if logger.isEnabledFor(logging.INFO):
            logger.info(f"Epoch: {epoch+1}/{total_epoch}, Average loss: {eng.loss_acc.item() / n:.4f}")
    checkpoint = {"model": eng.state_dict(),
                  "optimizer": {"step": eng.params.step, "exp_avg": eng.params.exp_avg.clone(),
                                "exp_avg_sq": eng.params.exp_avg_sq.clone()}}
    param["_feature_AE_engine"] = eng
    nf = param["n_feature_orig"]
    if keep_dev:
        return z_all, recon_dev[:, :nf], checkpoint
    embed_host = hostio.pinned_empty(pool, "feature_embed", (n, eng.EMB))
    embed_host.copy_(z_all, non_blocking=True)
    down.synchronize()
    torch.cuda.current_stream(dev).synchronize()
    return embed_host.numpy(), recon_host.numpy()[:, :nf], checkpoint


def build_knn_graph(x_embed: torch.Tensor, neighborhood_factor):
    """feature2adj + preprocess_graph on device (scgnn2.py:650-689, 1191-1198).
    Returns (Â as CSR with the A+I pattern, knn index [N,k] int32, knn fp64 distances)."""
    n = x_embed.shape[0]
    k_tmp = neighborhood_factor if neighborhood_factor > 1 else round(n * neighborhood_factor)
    k = int(k_tmp - 1 if k_tmp == n else k_tmp)
    idx, dist = ops.knn(x_embed, k, include_rank0=False)
    return ops.knn_graph_build(idx), idx, dist


def graph_AE_handler(X_embed, CCC_graph, args, param, dense_recon_max_cells: int = 4096):
    """Graph autoencoder stage, GCN branch (scgnn2.py:530-600): returns (embed, recon_graph, edgeList, adj)."""
    logger.info("Starting Graph AE")
    if args.graph_AE_use_GAT and args.graph_AE_GAT_dropout:
        raise NotImplementedError("graph_AE_GAT_dropout > 0 is not built (the example default is 0)")
    if args.graph_AE_concat_prev_embed and param["epoch_num"] > 0:
        raise NotImplementedError("graph_AE_concat_prev_embed is not built")
    if args.graph_AE_retain_weights:
        raise NotImplementedError("graph_AE_retain_weights permutes node order in the reference (App. B); not built")
    dev = param["device"]
    pool = param.get("io_pool")
    if isinstance(X_embed, torch.Tensor) and X_embed.is_cuda:
        xe = X_embed.float().contiguous()
    else:
        xh = hostio.as_host_tensor(X_embed)
        xe = torch.empty(xh.shape, dtype=torch.float32, device=dev)
        xe.copy_(xh, non_blocking=True)
    if args.graph_AE_normalize_embed == "sum1":
        xin = xe / xe.sum(1, keepdim=True).clamp(min=1)                         # scgnn2.py:622-628
    elif args.graph_AE_normalize_embed == "binary":
        xin = (xe > xe.mean(0)).float()
    else:
        xin = xe
    # ``param["graph_cache"]`` (extension): a dict that keeps the kNN graph of a previous call on the SAME embedding — the
    # reference rebuilds it on every call (feature2adj, scgnn2.py:555); bench.py uses it to time the training epochs alone.
    cache = param.get("graph_cache")
    if cache is not None and cache.get("n") == xe.shape[0] and "A" in cache:
        A, knn_idx, knn_dist = cache["A"], cache["knn_idx"], cache["knn_dist"]
    else:
        A, knn_idx, knn_dist = build_knn_graph(xe, args.graph_AE_neighborhood_factor)
        if cache is not None:
            cache.clear()
            cache.update(n=xe.shape[0], A=A, knn_idx=knn_idx, knn_dist=knn_dist)
    n = xe.shape[0]
    # ``param["cell_order"] = "locality"`` (extension): the epochs run on a relabelled copy of the graph in which cells are grouped
    # by nearest embedding centroid (ops.locality_order) — the aggregate's gathers then stay L2-resident; outputs are un-permuted
    perm = inv = None
    A_run = A
    if param.get("cell_order") == "locality" and not args.graph_AE_use_GAT:
        if cache is not None and "A_run" in cache:
            perm, inv, A_run = cache["perm"], cache["inv"], cache["A_run"]
        else:
            perm, inv = ops.locality_order(xe, n_anchors=int(param.get("cell_order_anchors", 64)))
            A_run = ops.knn_graph_build(inv[knn_idx[perm].long()].to(torch.int32).contiguous())
            if cache is not None:
                cache.update(perm=perm, inv=inv, A_run=A_run)
    adj_sum = A.nnz - n                                                         # Σ adj_train (no diagonal)
    pos_weight = float(n * n - adj_sum) / adj_sum                               # scgnn2.py:567
    norm = n * n / float((n * n - adj_sum) * 2)                                 # scgnn2.py:568-569
    labels = ops.CSR(A_run.rowptr, A_run.colidx, None, A_run.shape)             # A + I: pattern of Â, unit entries
    xin = xin.contiguous() if perm is None else xin[perm].contiguous()
    out_kw = dict(pool=pool, cache=cache, keep_dev=bool(param.get("keep_on_device")))
    if args.graph_AE_use_GAT:
        # edge_index = edgeList (i → its k neighbours), directed, no self loops (scgnn2.py:560-563); the kernels
        # index the graph by TARGET node, i.e. the transpose of the regular kNN-list CSR
        k = knn_idx.shape[1]
        src_csr = ops.CSR(torch.arange(0, n * k + 1, k, dtype=torch.int32, device=dev), knn_idx.reshape(-1).contiguous(), None, (n, n))
        T, _ = ops.csr_transpose(src_csr)
        Tt, t_perm = ops.csr_transpose(T)
        geng = GATEngine(xe.shape[1], args.gat_hid_embed, args.graph_AE_embedding_size, args.gat_multi_heads, device=dev,
                         lr=args.graph_AE_learning_rate, precision=param.get("precision"), seed=param.get("seed"))
        z = None
        for epoch in range(args.graph_AE_epoch):
            z = geng.train_step(xin, T, Tt, t_perm, labels)                         # loss_function: plain BCE (scgnn2.py:581)
            if logger.isEnabledFor(logging.INFO):
                logger.info(f"Epoch: {epoch+1}/{args.graph_AE_epoch}, Current loss: {geng.loss.item():.4f}")
        param["_graph_AE_engine"] = geng
        return _graph_ae_outputs(z, n, knn_idx, knn_dist, A, dense_recon_max_cells, **out_kw)
    eng = GraphAEEngine(xe.shape[1], args.graph_AE_embedding_size, device=dev, lr=args.graph_AE_learning_rate,
                        precision=param.get("precision"), seed=param.get("seed"))
    gen = torch.Generator(device=dev)
    gen.manual_seed(int(param.get("seed") or 0))
    eps = torch.empty(n, args.graph_AE_embedding_size, dtype=torch.float32, device=dev)
    z = None
    for epoch in range(args.graph_AE_epoch):
        eps.normal_(generator=gen)                                              # torch.randn_like(std), scgnn2.py:397
        z, _, _ = eng.train_step(xin, A_run, labels, norm, pos_weight, eps if perm is None else eps[perm].contiguous())
        if logger.isEnabledFor(logging.INFO):
            logger.info(f"Epoch: {epoch+1}/{args.graph_AE_epoch}, Current loss: {eng.loss.item():.4f}")
    param["_graph_AE_engine"] = eng
    if inv is not None:
        z = z[inv].contiguous()                                                 # back to the caller's cell order
    return _graph_ae_outputs(z, n, knn_idx, knn_dist, A, dense_recon_max_cells, **out_kw)


def _graph_ae_outputs(z, n, knn_idx, knn_dist, A, dense_recon_max_cells, pool=None, cache=None, keep_dev=False):
    """(graph_embed, recon_graph | None, edgeList, adj) like scgnn2.py:597-600.  ``edgeList`` is ([N·k, 2] int64 pairs, fp64
    weights 1/(d+1e-16)) instead of a Python list of tuples; ``adj`` the 0/1 union-symmetrised adjacency without diagonal."""
    if keep_dev:
        return z, None, (knn_idx, knn_dist), A
    embed_host = hostio.pinned_empty(pool, "graph_embed", tuple(z.shape))
    embed_host.copy_(z, non_blocking=True)
    recon = (z @ z.t()).cpu().numpy() if n <= dense_recon_max_cells else None   # InnerProductDecoder output, small N only
    if cache is not None and "edge_list" in cache:
        edge_list, adj = cache["edge_list"], cache["adj"]
    else:
        k = knn_idx.shape[1]
        src = torch.arange(n, device=z.device, dtype=torch.int64).repeat_interleave(k)
        edge_index = torch.stack([src, knn_idx.reshape(-1).long()], 1).cpu().numpy()
        edge_w = (1.0 / (knn_dist.reshape(-1).double() + 1e-16)).cpu().numpy()  # scgnn2.py:686
        edge_list = (edge_index, edge_w)
        import scipy.sparse as sp
        rp = A.rowptr.long()
        rows = torch.repeat_interleave(torch.arange(n, device=z.device), rp[1:] - rp[:-1])
        off = A.colidx.long() != rows                                           # drop the diagonal of A + I on the device
        counts = torch.zeros(n + 1, dtype=torch.int64, device=z.device)
        counts[1:] = torch.bincount(rows[off], minlength=n)
        indptr = torch.cumsum(counts, 0).cpu().numpy()
        indices = A.colidx[off].cpu().numpy()
        adj = sp.csr_matrix((np.ones(indices.shape[0], dtype=np.float32), indices, indptr), shape=(n, n))
        if cache is not None:
            cache["edge_list"], cache["adj"] = edge_list, adj
    torch.cuda.current_stream(z.device).synchronize()
    return embed_host.numpy(), recon, edge_list, adj


def _edge_list_arrays(edgeList):
    """edgeList as ([E, 2] int pairs, [E] weights) — accepts this module's array form or the reference's list of (i, j, w) tuples."""
    if isinstance(edgeList, tuple) and len(edgeList) == 2 and hasattr(edgeList[0], "shape"):
        idx, w = edgeList
        if isinstance(idx, torch.Tensor):      # device form (knn_idx [N, k] int32, knn_dist [N, k] fp64) from keep_on_device
            n, k = idx.shape
            src = np.repeat(np.arange(n), k)
            return np.stack([src, idx.cpu().numpy().reshape(-1).astype(np.int64)], 1), 1.0 / (w.cpu().numpy().reshape(-1) + 1e-16)
        return np.asarray(idx), np.asarray(w)
    arr = np.asarray(edgeList, dtype=np.float64)
    return arr[:, :2].astype(np.int64), arr[:, 2]


def generateLouvainCluster(edgeList, n_nodes: Optional[int] = None):
    """Louvain communities of the undirected weighted kNN graph (scgnn2.py:193-215): returns (labels list, n_communities).
    networkx.Graph.add_weighted_edges_from keeps ONE weight per undirected pair (the last one written; both directions carry
    the same 1/(d+1e-16)), loops dropped — here: the elementwise maximum of W and Wᵀ in CSR, then ``b2_louvain_csr_host``."""
    import scipy.sparse as sp
    idx, w = _edge_list_arrays(edgeList)
    n = int(idx.max()) + 1 if n_nodes is None else n_nodes
    keep = idx[:, 0] != idx[:, 1]
    W = sp.csr_matrix((w[keep], (idx[keep, 0], idx[keep, 1])), shape=(n, n))
    W = W.maximum(W.T).tocsr()
    W.sort_indices()
    labels, nc, _ = ops.louvain_host(W.indptr, W.indices, W.data)
    return labels.tolist(), nc


def trimClustering(listResult, minMemberinCluster=5, maxClusterNumber=30):
    """scgnn2.py:230-254: clusters that are too small or numbered ≥ maxClusterNumber are merged into one label.  (The reference
    counts members starting from 0 — ``numDict[item] = 0`` on first sight — so "fewer than 5" means ≤ 5 cells; kept.)  Labels are
    renumbered contiguously afterwards: the reference's ``cluster_output_handler`` would index past its list otherwise."""
    lab = np.asarray(listResult).copy()
    ids, counts = np.unique(lab, return_counts=True)
    size = len(ids)
    drop = [c for c in range(size) if (dict(zip(ids, counts)).get(c, 0) - 1) < minMemberinCluster or c >= maxClusterNumber]
    lab[np.isin(lab, drop)] = maxClusterNumber
    _, lab = np.unique(lab, return_inverse=True)
    return lab.tolist()


def cluster_output_handler(listResult):
    lab = np.asarray(listResult)
    return list(listResult), [np.nonzero(lab == c)[0].tolist() for c in range(len(set(lab.tolist())))]


def _normalizer(X, base, axis=0):
    from sklearn.preprocessing import minmax_scale
    upper, lower = np.quantile(base, q=0.9), np.quantile(base, q=0.1)
    if upper != lower:
        return minmax_scale(X, feature_range=(lower, upper), axis=axis)
    return minmax_scale(X, feature_range=(np.quantile(base, q=0), np.quantile(base, q=1)), axis=axis)


def kmeans_fit_predict(embed, k: int, device, seed: int = 0, init_max_cells: int = 200_000):
    """``KMeans(n_clusters=k, n_init="auto", random_state=0).fit_predict(embed)`` (scgnn2.py:186): k-means++ seeding by
    sklearn's own routine on the host (on a fixed-seed subsample above ``init_max_cells`` cells), Lloyd iterations on the device."""
    from sklearn.cluster import kmeans_plusplus
    xe = embed if isinstance(embed, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(embed, dtype=np.float32))
    xe = xe.to(device).float().contiguous()
    n = xe.shape[0]
    if n > init_max_cells:
        sel = np.sort(np.random.RandomState(seed).choice(n, init_max_cells, replace=False))
        host = xe[torch.from_numpy(sel).to(device)].cpu().numpy()
    else:
        host = xe.cpu().numpy()
    host = host - host.mean(0)                      # KMeans centres the data before seeding (sklearn _kmeans.py: X -= X_mean)
    # KMeans.fit hands its RandomState(random_state) straight to the k-means++ routine (sklearn _kmeans.py, _init_centroids)
    centers, _ = kmeans_plusplus(host.astype(np.float32), k, random_state=np.random.RandomState(seed))
    mean = xe.mean(0, keepdim=True)
    xc = (xe - mean).contiguous()
    C0 = torch.from_numpy(np.ascontiguousarray(centers, dtype=np.float32)).to(device)
    labels, _, _ = ops.kmeans(xc, C0)
    return labels


def clustering_handler(edgeList, args, param):
    """scgnn2.py:138-190: Louvain on the kNN graph fixes the cluster COUNT (k = round(max(k_louvain·resolution, 2))), KMeans on
    the chosen embedding gives the labels."""
    logger.info("Start Clustering")
    ge, fe = param["graph_embed"], param["feature_embed"]
    to_np = lambda a: a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    if args.clustering_embed == "feature":
        embed = fe
    elif args.clustering_embed == "both":
        embed = np.concatenate((to_np(ge), _normalizer(to_np(fe), base=to_np(ge), axis=0)), axis=1).astype(np.float32)
    else:
        if args.clustering_embed != "graph":
            logger.error("clustering_embed argument not recognized, using graph embed")
        embed = ge
    param["clustering_embed"] = embed
    n = embed.shape[0]
    listResult, _ = generateLouvainCluster(edgeList, n)
    k_louvain = len(np.unique(listResult))
    logger.info(f" Louvain clusters count: {k_louvain}")
    resolution = 0.8 if n < 2000 else 0.5
    param["k_float"] = max(k_louvain * resolution, 2)
    k = round(param["k_float"])
    logger.info(f" Adjusted clusters count: {k}")
    if not args.clustering_louvain_only:
        if args.clustering_method == "KMeans":
            listResult = kmeans_fit_predict(embed, k, param["device"], seed=0,
                                            init_max_cells=param.get("kmeans_init_max_cells", 200_000)).cpu().numpy().tolist()
        elif args.clustering_method == "AffinityPropagation":
            from sklearn.cluster import AffinityPropagation          # O(N²) host method, small data only — same call as the reference
            listResult = AffinityPropagation(random_state=args.seed).fit_predict(to_np(embed)).tolist()
    if len(set(listResult)) > 30 or len(set(listResult)) <= 1:
        logger.info(f" Stopping: Number of clusters is {len(set(listResult))}")
        listResult = trimClustering(listResult, minMemberinCluster=5, maxClusterNumber=30)
    logger.info(f"Total Cluster Number: {len(set(listResult))}")
    return cluster_output_handler(listResult)


def graph_celltype_regu_handler(adj, cluster_labels, device=None):
    """scgnn2.py:716-724 without the two dense N×N matrices: returns what the Cluster-AE loss takes from them, per cell —
    (w_graph [N], w_celltype [N]) = their column sums inside the cell's cluster.  The reference's "normalised" adjacency is
    deg_j / deg_i (it multiplies np.matrix objects, see csrc/em.cu), so w_graph_j = deg_j · Σ_{i∈cluster(j)} 1/deg_i; the
    same-cluster indicator is a true ndarray, row-normalised elementwise, whose column sums inside the cluster are 1."""
    lab = torch.as_tensor(np.asarray(cluster_labels), dtype=torch.int32)
    if isinstance(adj, ops.CSR):
        A = adj
    else:                                                                       # scipy 0/1 adjacency without diagonal
        A = ops.CSR.from_scipy(adj, device, with_values=False)
    lab = lab.to(A.rowptr.device)
    w_graph = ops.graph_regu_weights(A, lab)
    return w_graph, torch.ones_like(w_graph)


def cluster_AE_handler(X_recon, TRS, clusterIndexList, args, param, model_state):
    """scgnn2.py:821-880: one Cluster-AE per cluster, initialised from the Feature-AE weights, trained on the cluster's rows of
    X_recon with the "Celltype" regulariser; returns the stitched reconstruction (numpy, or a device tensor under
    ``keep_on_device``).  Clusters larger than ``cluster_AE_batch_size`` are trained in mini-batches with the full-cluster
    regulariser weights (the reference's dense [cluster × cluster] @ [batch × gene] product requires a single batch)."""
    logger.info("Starting Cluster AE")
    dev = param["device"]
    bs, epochs = args.cluster_AE_batch_size, args.cluster_AE_epoch
    p_drop = float(args.cluster_AE_dropout_prob or 0.0)        # train_handler's masked_prob (scgnn2.py:1256) for the Cluster-AE runs
    to_dev = lambda a: a.float().contiguous() if (isinstance(a, torch.Tensor) and a.is_cuda) else hostio.as_host_tensor(a).to(dev)
    Xr = to_dev(X_recon)
    xd = param.get("_x_dropout_dev")
    if xd is None:
        xd = to_dev(param["x_dropout"])
        param["_x_dropout_dev"] = xd
    w_graph, w_ct = param["impute_regu"]
    roww = (0.3 + 0.3 * w_graph + 0.1 * w_ct).contiguous()
    out = torch.zeros_like(Xr)
    nf = param["n_feature_orig"]
    for ci, members in enumerate(clusterIndexList):
        logger.info(f"Training cluster {ci+1}/{len(clusterIndexList)} -> size = {len(members)}")
        if len(members) == 0:
            continue
        rows = torch.as_tensor(np.asarray(members), dtype=torch.int64, device=dev)
        xc, xdc, wc = Xr[rows].contiguous(), xd[rows][:, :nf].contiguous(), roww[rows].contiguous()
        eng = FeatureAEEngine(Xr.shape[1], device=dev, lr=args.cluster_AE_learning_rate, precision=param.get("precision"))
        eng.load_state_dict(model_state["model"])
        m = xc.shape[0]
        rc = torch.empty_like(xc)
        for epoch in range(epochs):
            eng.loss_acc.zero_()
            for b0 in range(0, m, bs):
                b1 = min(m, b0 + bs)
                _, r = eng.train_step(xc[b0:b1], None, args.cluster_AE_regu_strength, "Celltype", row_weight=wc[b0:b1],
                                      x_dropout=xdc[b0:b1], x_input=eng.input_dropout(xc[b0:b1], p_drop) if p_drop > 0.0 else None)
                if epoch == epochs - 1:
                    rc[b0:b1].copy_(r)
        out[rows] = rc
    if param.get("keep_on_device"):
        return out
    host = hostio.pinned_empty(param.get("io_pool"), "cluster_recon", tuple(out.shape))
    host.copy_(out)
    return host.numpy()


class ScGNN2:
    """Drop-in for ``dance.modules.single_modality.imputation.scgnn2.ScGNN2`` (pre-EM stage + EM iterations)."""

    def __init__(self, args, device: str = "auto", precision: Optional[str] = None, seed: Optional[int] = None):
        self.args = args
        self.device = _device(device)
        self.precision = precision
        self.seed = seed

    def fit(self, x: np.ndarray):
        args = self.args
        epochs = args.total_epoch
        param = {"device": self.device, "tik": time(), "precision": self.precision, "seed": self.seed}
        logger.info(f"Using device: {param['device']}")
        trs_mat = None  # the reference passes an all-zero TRS (scgnn2.py:40)
        logger.info("Pre EM runs")
        param["epoch_num"] = 0
        param["total_epoch"] = epochs
        param["n_feature_orig"] = x.shape[1]
        param["x_dropout"] = x
        # inside fit() every stage hands DEVICE tensors to the next one (no N×G round trips between handlers); only the final
        # imputed matrix is copied back.  The public handlers keep their numpy-in / numpy-out contract when called directly.
        param["keep_on_device"] = True
        param["io_pool"] = hostio.IOPool()
        x_embed, x_feature_recon, model_state = feature_AE_handler(x, trs_mat, args, param)
        graph_embed, _, edge_list, adj = graph_AE_handler(x_embed, None, args, param)
        x_imputed = x_feature_recon
        logger.info("Entering main loop")
        for i in range(epochs):
            logger.info(f"\n==========> scGNN Epoch {i+1}/{epochs} <==========")
            param["epoch_num"] = i + 1
            param["feature_embed"], param["graph_embed"] = x_embed, graph_embed
            cluster_labels, cluster_lists_of_idx = clustering_handler(edge_list, args, param)
            param["impute_regu"] = graph_celltype_regu_handler(adj, cluster_labels, self.device)
            x_imputed = cluster_AE_handler(x_feature_recon, trs_mat, cluster_lists_of_idx, args, param, model_state)
            x_embed, x_feature_recon, model_state = feature_AE_handler(x_imputed, trs_mat, args, param, model_state)
            graph_embed, _, edge_list, adj = graph_AE_handler(x_embed, None, args, param)
            self.cluster_labels = cluster_labels
        param["keep_on_device"] = False
        self.x_embed, self.graph_embed = x_embed.cpu().numpy(), graph_embed.cpu().numpy()
        self.edge_list, self.adj, self.model_state = edge_list, adj, model_state
        # the reference returns the LAST Cluster-AE output (x_imputed), or — with total_epoch = 0 — nothing at all
        # (self.x_imputed is unbound, scgnn2.py:68); here the pre-EM Feature-AE reconstruction is returned in that case
        self.x_imputed = x_imputed.cpu().numpy() if isinstance(x_imputed, torch.Tensor) else x_imputed
        param.pop("_x_dropout_dev", None)

    def predict(self, x: Optional[Any] = None) -> np.ndarray:
        return self.x_imputed

    def score(self, true_expr, imputed_expr, mask=None, metric="MSE", log1p=True, test_idx=None):
        """Imputation quality on the test cells, reference semantics (scgnn2.py:73-121): the prediction is optionally log1p-ed,
        entries under ``mask`` are overwritten with the truth (so they do not count), then RMSE over all test entries or
        PCC / MRE over the held-out (``~mask``) entries.  The default ``metric="MSE"`` is rejected like in the reference."""
        supported = ("RMSE", "PCC", "MRE")
        if metric not in supported:
            raise ValueError(f"scoring metric must be one of {set(supported)!r}")
        rows = torch.arange(len(true_expr)) if test_idx is None else torch.as_tensor(np.asarray(test_idx))
        truth = torch.as_tensor(true_expr)[rows].to(self.device)
        pred = torch.as_tensor(imputed_expr)[rows].to(self.device)
        pred = torch.log1p(pred) if log1p else pred.clone()
        held_out = None
        if mask is not None:
            seen = torch.as_tensor(np.asarray(mask))[rows].to(self.device)
            pred = torch.where(seen, truth.to(pred.dtype), pred)
            held_out = ~seen
        if metric == "RMSE":
            return float(torch.sqrt(torch.mean((truth - pred)**2)).item())
        if held_out is None:
            raise ValueError(f"metric {metric!r} is evaluated on the masked-out entries and needs `mask`")
        t, p = truth[held_out].double(), pred[held_out].double()
        if metric == "PCC":
            tc, pc = t - t.mean(), p - p.mean()
            return float((tc @ pc / torch.sqrt((tc @ tc) * (pc @ pc))).item())
        return float(torch.mean(torch.abs(p - t) / torch.abs(t).clamp(min=1e-10)).item())      # MRE
