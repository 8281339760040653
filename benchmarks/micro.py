"""Kernel micro-benchmarks (CUDA-event timed on the launching stream, L2 flushed between
iterations).  Prints one JSON line per kernel with achieved algorithmic GB/s or TFLOP/s."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dance_b200 import ops  # noqa: E402

PEAKS = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}   # NVIDIA H100 SXM data sheet (700 W); MEASURED_PEAKS.json overrides
try:
    PEAKS.update(json.load(open(Path(__file__).resolve().parent.parent / "MEASURED_PEAKS.json")))
except Exception:
    pass


def timeit(fn, iters=10, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts)), float(np.min(ts))


def random_knn_graph(n, k, dev, seed=0, local=None):
    g = torch.Generator(device=dev).manual_seed(seed)
    if local is None:
        idx = torch.randint(0, n, (n, k), device=dev, dtype=torch.int32, generator=g)
    else:  # neighbours within a window of `local` rows (cluster-sorted cells)
        base = (torch.arange(n, device=dev) // local * local).unsqueeze(1)
        idx = (base + torch.randint(0, local, (n, k), device=dev, generator=g)).clamp_(max=n - 1).to(torch.int32)
    return ops.knn_graph_build(idx.contiguous())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--only", type=str, default="")
    ap.add_argument("--out", type=str, default=None, help="also write every result line as one JSON list to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    only = set(args.only.split(",")) if args.only else None
    out = []

    def want(name):
        return only is None or name in only

    n = args.n
    if want("spmm"):
        for local in (None, 100_000, 4096):
            A = random_knn_graph(n, 15, dev, local=local)
            for F in (16, 32, 64, 128):
                X = torch.randn(n, F, device=dev)
                Y = torch.empty(n, F, device=dev)
                med, best = timeit(lambda: ops.spmm(A, X, out=Y), flush=flush)
                alg = A.nnz * 8 + (n + 1) * 4 + 2 * n * F * 4
                gather = A.nnz * F * 4
                out.append(dict(kernel="spmm_csr_f32", n=n, nnz=A.nnz, F=F, locality=local, ms=med, ms_best=best,
                                alg_GB=alg / 1e9, alg_GBps=alg / med / 1e6, frac_hbm=alg / med / 1e6 / PEAKS["hbm_gbs"],
                                gather_GBps=gather / med / 1e6))
                print(json.dumps(out[-1]), flush=True)
    if want("gemm"):
        for prec in ("fp32", "tf32x3", "tf32"):
            for (M, N, K, tA, tB) in ((12800, 512, 2000, 0, 1), (12800, 2000, 512, 0, 1), (12800, 128, 512, 0, 1),
                                       (12800, 512, 2000, 0, 0), (2000, 512, 12800, 1, 0), (512, 2000, 12800, 1, 0)):
                A = torch.randn((K, M) if tA else (M, K), device=dev)
                B = torch.randn((N, K) if tB else (K, N), device=dev)
                C = torch.empty(M, N, device=dev)
                med, best = timeit(lambda: ops.gemm(A, B, transA=bool(tA), transB=bool(tB), out=C, precision=prec), flush=flush)
                fl = 2.0 * M * N * K
                out.append(dict(kernel="gemm_f32", precision=prec, M=M, N=N, K=K, tA=tA, tB=tB, ms=med, ms_best=best,
                                TFLOPs=fl / med / 1e9))
                print(json.dumps(out[-1]), flush=True)
    if want("gae"):
        for nn in (20_000, 100_000):
            A = random_knn_graph(nn, 15, dev)
            L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
            z = torch.randn(nn, 16, device=dev) * 0.3
            mu, lv = torch.randn(nn, 16, device=dev) * 0.1, torch.randn(nn, 16, device=dev) * 0.1
            med, best = timeit(lambda: ops.gae_loss_grad(z, L, 0.5, 100.0, mu, lv), iters=3, warmup=1)
            out.append(dict(kernel="gae_loss_grad", n=nn, ms=med, pairs_per_s=nn * nn / med * 1e3))
            print(json.dumps(out[-1]), flush=True)
    if want("knn"):
        for nn, d in ((100_000, 128), (100_000, 50)):
            X = torch.randn(nn, d, device=dev) + torch.randn(10, d, device=dev)[torch.randint(0, 10, (nn, ), device=dev)] * 3
            med, best = timeit(lambda: ops.knn(X, 15, return_dist=False), iters=3, warmup=1)
            out.append(dict(kernel="knn_l2", n=nn, d=d, k=15, ms=med, TFLOPs=2.0 * nn * nn * d / med / 1e9))
            print(json.dumps(out[-1]), flush=True)
    if want("normalize"):
        for nn, g in ((200_000, 2000), ):
            X = torch.rand(nn, g, device=dev)
            med, best = timeit(lambda: ops.normalize_total_log1p_(X, target_sum=1e4), flush=flush)
            alg = 2.0 * nn * g * 4
            out.append(dict(kernel="normalize_total_log1p", n=nn, g=g, ms=med, alg_GBps=alg / med / 1e6,
                            frac_hbm=alg / med / 1e6 / PEAKS["hbm_gbs"]))
            print(json.dumps(out[-1]), flush=True)
    if want("cellgene"):
        nn, g = 100_000, 2000
        X = (torch.rand(nn, g, device=dev) < 0.1).float() * torch.rand(nn, g, device=dev)
        med, best = timeit(lambda: ops.cellgene_graph(X, True), iters=3, warmup=1)
        nnz = int((X != 0).sum().item())
        alg = 2.0 * nn * g * 4 + (2 * nnz + nn + g) * (8 + 8 + 4)            # two passes over X + the edge list written once
        out.append(dict(kernel="cellgene_graph (CellFeatureGraph)", n=nn, g=g, nnz=nnz, ms=med, alg_GBps=alg / med / 1e6,
                        frac_hbm=alg / med / 1e6 / PEAKS["hbm_gbs"]))
        print(json.dumps(out[-1]), flush=True)
    if want("pearson"):
        for nn, g in ((100_000, 2000), ):
            X = torch.randn(nn, g, device=dev)
            med, best = timeit(lambda: ops.pearson_corr(X), iters=3, warmup=1)
            out.append(dict(kernel="pearson_corr (FeatureFeatureGraph, fp64 SIMT Gram, upper triangle)", n=nn, g=g, ms=med,
                            fp64_TFLOPs=float(g) * (g + 64) * nn / med / 1e9))
            print(json.dumps(out[-1]), flush=True)
    if want("matnorm"):
        nn, g = 200_000, 2000
        X = torch.rand(nn, g, device=dev)
        Y = torch.empty_like(X)
        for mode, axis, passes in (("normalize", 0, 2), ("standardize", 0, 3), ("l2", 1, 2)):
            med, best = timeit(lambda: ops.matrix_normalize(X, mode, axis, -1.0, out=Y), flush=flush)
            alg = (passes + 1.0) * nn * g * 4
            out.append(dict(kernel="matrix_normalize", mode=mode, axis=axis, n=nn, g=g, ms=med, alg_GBps=alg / med / 1e6,
                            frac_hbm=alg / med / 1e6 / PEAKS["hbm_gbs"]))
            print(json.dumps(out[-1]), flush=True)
    if want("umap"):
        nn, k = 1_000_000, 15
        idx = torch.randint(0, nn, (nn, k), device=dev, dtype=torch.int32)
        idx[:, 0] = torch.arange(nn, device=dev, dtype=torch.int32)
        dist = torch.sort(torch.rand(nn, k, device=dev), dim=1).values
        dist[:, 0] = 0
        med, best = timeit(lambda: ops.umap_connectivities(idx, dist), iters=3, warmup=1)
        out.append(dict(kernel="umap_connectivities (smooth-kNN bisection + 2 CSR transposes + fuzzy union)", n=nn, k=k, ms=med,
                        edges_per_s=nn * k / med * 1e3))
        print(json.dumps(out[-1]), flush=True)
    if want("radius"):
        nn = 200_000
        xy = torch.rand(nn, 2, device=dev, dtype=torch.float64) * (nn**0.5) * 100
        med, best = timeit(lambda: ops.radius_graph(xy, 150.0), iters=3, warmup=1)
        out.append(dict(kernel="radius_graph (StagateGraph, brute force fp64)", n=nn, ms=med, pair_tests_per_s=2.0 * nn * nn / med * 1e3))
        print(json.dumps(out[-1]), flush=True)
    if want("gat"):
        nn, k = 200_000, 6
        A = random_knn_graph(nn, k, dev)
        T = ops.CSR(A.rowptr, A.colidx, None, A.shape)
        H = torch.randn(nn, 512, device=dev)
        a_s, a_t = torch.randn(512, device=dev) * 0.05, torch.randn(512, device=dev) * 0.05
        s_src, s_trg = ops.gat_scores(H, a_s, a_t, 1)
        med, best = timeit(lambda: ops.gat_aggregate_fwd(T, H, s_src, s_trg, 1, score_act="sigmoid", shift="segment"), flush=flush)
        alg = T.nnz * 4 + 2.0 * nn * 512 * 4 + T.nnz * 4
        out.append(dict(kernel="gat_aggregate_fwd (STAGATE layer, F=512)", n=nn, nnz=T.nnz, ms=med, alg_GBps=alg / med / 1e6,
                        frac_hbm=alg / med / 1e6 / PEAKS["hbm_gbs"], gather_GBps=T.nnz * 512 * 4 / med / 1e6))
        print(json.dumps(out[-1]), flush=True)
    if want("zinb"):
        nn, g = 100_000, 2000
        a, b, c = (torch.randn(nn, g, device=dev) for _ in range(3))
        y = torch.poisson(torch.rand(nn, g, device=dev) * 2)
        sf = torch.rand(nn, device=dev) + 0.5
        med, best = timeit(lambda: ops.zinb_loss_grad(a, b, c, y, sf, None, 1.0, 1.0), flush=flush)
        alg = (2 * 4 + 3) * nn * g * 4.0            # loss pass reads a,b,c,y; grad pass reads them again and writes three gradients
        out.append(dict(kernel="zinb_loss_grad (GraphSCI heads + NLL + gradients)", n=nn, g=g, ms=med, alg_GBps=alg / med / 1e6,
                        frac_hbm=alg / med / 1e6 / PEAKS["hbm_gbs"]))
        print(json.dumps(out[-1]), flush=True)
    if want("batchnorm"):
        nn, g = 200_000, 2000
        X = torch.randn(nn, g, device=dev)
        gam, bet, rm, rv = torch.ones(g, device=dev), torch.zeros(g, device=dev), torch.zeros(g, device=dev), torch.ones(g, device=dev)
        med, best = timeit(lambda: ops.batchnorm_fwd(X, gam, bet, rm, rv, True), flush=flush)
        alg = 4.0 * nn * g * 4                      # two statistics passes + read + write
        out.append(dict(kernel="batchnorm_fwd (training)", n=nn, c=g, ms=med, alg_GBps=alg / med / 1e6, frac_hbm=alg / med / 1e6 / PEAKS["hbm_gbs"]))
        print(json.dumps(out[-1]), flush=True)
    if want("dec"):
        nn, h, K = 1_000_000, 50, 10
        z, mu = torch.randn(nn, h, device=dev), torch.randn(K, h, device=dev)
        p = ops.dec_target(ops.dec_q(z, mu))
        med, best = timeit(lambda: ops.dec_kl_grad(z, mu, p), flush=flush)
        alg = nn * (2.0 * h + K) * 4
        out.append(dict(kernel="dec_kl_grad (SpaGCN DEC head: loss + dz + dmu + argmax)", n=nn, h=h, K=K, ms=med, alg_GBps=alg / med / 1e6,
                        frac_hbm=alg / med / 1e6 / PEAKS["hbm_gbs"]))
        print(json.dumps(out[-1]), flush=True)
    if want("pca"):
        nn, g, k = 100_000, 2000, 50
        X = torch.randn(nn, g, device=dev)
        med, best = timeit(lambda: ops.pca(X, k), iters=2, warmup=1)
        out.append(dict(kernel="pca (CellPCA: covariance GEMM + Jacobi eigensolver + projection)", n=nn, g=g, k=k, ms=med))
        print(json.dumps(out[-1]), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        json.dump(out, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
