#!/usr/bin/env python
"""bench.py — scGNN forward+backward throughput (cells/sec) on synthetic cell×gene data.

One "step" = one pass of the scGNN hot path over all cells of the configuration
(BASELINE.json: "scGNN 1M cells × 2000 genes", SURVEY §8d):
  1. one Feature-AE epoch over every cell (batch 12 800, LTMG-mode loss with the reference
     driver's all-zero TRS, Adam)                                  scgnn2.py:275-335, 1217-1295
  2. one Graph-AE (GCN branch) full-batch epoch on the 128-d embeddings over the prebuilt
     k=15 kNN graph: 2 projection GEMMs + 2 SpMM forward, the exact matrix-free N×N
     inner-product-decoder loss (pos-weighted BCE + KLD), backward, Adam   scgnn2.py:575-615
kNN search + graph assembly are outside the step (the reference rebuilds the graph once per
200 Graph-AE epochs) and are reported as `graph_build_s`.

  python bench.py --gpus N --steps K --warmup W            (N>1: launched under torchrun)
  python bench.py --impl reference ...                     (CPU arm: oracle port on host cores)
  python bench.py ... --dump-outputs DIR                   (also write the last timed step's outputs as DIR/<name>.npy)

Prints ONE JSON line (see the repository README / DESIGN.md for the field definitions).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

BATCH = 12800
K_NN = 15
EMB = 16


def load_peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.load(open(p))
        return dict(hbm_gbs=d["hbm_gbs"], bf16_tflops=d["bf16_tflops"], bf16_tflops_sustained=d.get("bf16_tflops_sustained"),
                    source="measured")
    # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 TFLOP/s dense BF16
    return dict(hbm_gbs=3350.0, bf16_tflops=989.0, bf16_tflops_sustained=None, source="H100 SXM data sheet")


# ------------------------------------------------------------------------------------ synthetic data
DATA_SEED = 0


def synth_expression(n, g, device, row_begin=0):
    """Rows [row_begin, row_begin+n) of the SURVEY §8d expression matrix (dance_b200.synth: every value is a hash of
    (seed, global cell index, gene), identical on every arm / device / sharding), log-normalised (normalize_total(1e4) + log1p)."""
    from dance_b200 import synth
    X = synth.expression_counts(n, g, seed=DATA_SEED, density=0.10, row_begin=row_begin, device=device)
    if X.is_cuda:
        from dance_b200 import ops
        ops.normalize_total_log1p_(X, target_sum=1e4, max_fraction=1.0)
    else:   # CPU arm: the reference formula (scanpy normalize_total + log1p), zero-count cells untouched
        tot = X.sum(1, keepdim=True)
        X = torch.log1p(torch.where(tot > 0, X * (1e4 / tot.clamp(min=1e-30)), X))
    return X


# ------------------------------------------------------------------------------------ clocks sampler
class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
    Q_OLD = Q.replace("clocks_event_reasons", "clocks_throttle_reasons")

    def __init__(self, gpu_index=0):
        self.rows, self.proc, self.gpu_index = [], None, gpu_index

    def start(self):
        try:
            q = self.Q
            probe = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(self.gpu_index)],
                                   capture_output=True, text=True, timeout=20)
            if probe.returncode != 0 or "not a valid" in (probe.stdout + probe.stderr).lower():
                q = self.Q_OLD
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "100",
                                          "-i", str(self.gpu_index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            if len(f) < 8:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[4:8]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# ------------------------------------------------------------------------------------ CPU (reference) arm
def cpu_reference_step_factory(n_cells, genes):
    """One scGNN step on `n_cells` cells on the host cores: Feature_AE epoch + Graph_AE GCN epoch with the dense N×N
    decoder / labels exactly like scgnn2.py:557,425,603-615.  When the reference tree is present (build container) the
    reference's OWN classes run through oracle/ref_loader.py (kind "reference": Feature_AE, train_handler, Graph_AE,
    gae_loss_function, preprocess_graph, feature2adj); on the GPU box (/root/reference absent) the pinned restatement
    oracle/port.py runs the same arithmetic (kind "port")."""
    from oracle import port, ref_loader
    torch.set_num_threads(os.cpu_count())
    X = synth_expression(n_cells, genes, "cpu")
    torch.manual_seed(0)
    if ref_loader.available():
        ref = ref_loader.scgnn2()
        cpu_reference_step_factory.kind = "reference"
        fae = ref.Feature_AE(dim=genes)
        opt = torch.optim.Adam(fae.parameters(), lr=1e-3)
        with torch.no_grad():
            z0, _ = fae(X)
        _, adj, _ = ref.feature2adj(z0.numpy(), K_NN, False)      # (adj, adj_train, edgeList), scgnn2.py:650-672
        adj_norm = ref.preprocess_graph(adj)                      # same sequence as graph_AE_handler, scgnn2.py:555-569
        import scipy.sparse as sp
        labels = torch.FloatTensor((adj + sp.eye(n_cells)).toarray())
        pw = float(n_cells * n_cells - adj.sum()) / adj.sum()
        norm = n_cells * n_cells / float((n_cells * n_cells - adj.sum()) * 2)
        gae = ref.Graph_AE(128, EMB, 0, 2, 64)
        gopt = torch.optim.Adam(gae.parameters(), lr=1e-2)
        loader = torch.utils.data.DataLoader(ref.ExpressionDataset(X.numpy()), batch_size=BATCH)
        trs = torch.zeros_like(X)
        param = {"device": "cpu", "epoch_num": 0, "total_epoch": 0, "n_feature_orig": genes}

        def step():
            _, z_all, _ = ref.train_handler(model=fae, train_loader=loader, optimizer=opt, TRS=trs, total_epoch=1, impute_regu=None,
                                            regu_type=["LTMG", "noregu"], regu_strength=0.9, masked_prob=0, param=param)
            gae.train()
            gopt.zero_grad()
            embed, gae_info, recon = gae(z_all.detach(), adj_norm, use_GAT=False)
            loss = ref.gae_loss_function(preds=recon, labels=labels, mu=gae_info[0], logvar=gae_info[1], n_nodes=n_cells, norm=norm,
                                         pos_weight=pw)
            loss.backward()
            gopt.step()
            return float(loss.item())

        return step
    cpu_reference_step_factory.kind = "port"
    fae = port.FeatureAE(genes)
    opt = torch.optim.Adam(fae.parameters(), lr=1e-3)
    with torch.no_grad():
        z0, _ = fae(X)
    adj, _ = port.feature2adj(z0.numpy(), K_NN)
    an = port.preprocess_graph(adj)
    adj_t = port.to_torch_sparse(an)
    pw, norm = port.gae_norm_constants(adj)
    import scipy.sparse as sp
    labels = torch.from_numpy((adj + sp.eye(n_cells)).toarray()).float()
    w = [torch.nn.Parameter(torch.empty(128, 32)), torch.nn.Parameter(torch.empty(32, EMB)), torch.nn.Parameter(torch.empty(32, EMB))]
    for p in w:
        torch.nn.init.xavier_uniform_(p)
    gopt = torch.optim.Adam(w, lr=1e-2)

    def step():
        _, z_all, _ = port.feature_ae_epoch(fae, opt, X, BATCH, "LTMG", 0.9)
        gopt.zero_grad()
        eps = torch.randn(n_cells, EMB)
        z, mu, logvar, _ = port.graph_ae_gcn_forward(z_all, w[0], w[1], w[2], adj_t, eps)
        loss = port.gae_loss(torch.mm(z, z.t()), labels, mu, logvar, n_cells, norm, pw)
        loss.backward()
        gopt.step()
        return float(loss.item())

    return step


def time_cpu(n_cells, genes, steps, warmup):
    """Times the CPU arm with the best of a few intra-op thread counts: on a 128-core host torch-CPU is ~10× SLOWER
    with 128 threads than with 32 for these shapes (measured), and the baseline should be the reference at its best."""
    step = cpu_reference_step_factory(n_cells, genes)
    cores = os.cpu_count()
    best_t, best_th = None, cores
    for th in sorted({cores, min(cores, 64), min(cores, 32), min(cores, 16)}, reverse=True):
        torch.set_num_threads(th)
        step()                      # doubles as warm-up
        t0 = time.perf_counter()
        step()
        dt = time.perf_counter() - t0
        if best_t is None or dt < best_t:
            best_t, best_th = dt, th
    torch.set_num_threads(best_th)
    time_cpu.threads = best_th
    time_cpu.kind = cpu_reference_step_factory.kind
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        step()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), ts


def cpu_sample_text(n_cpu, args):
    return (f"{n_cpu} of {args.cells} cells × {args.genes} genes (same generator, rows 0..{n_cpu - 1}); 1 step = Feature_AE epoch + Graph_AE GCN "
            f"epoch with the reference's dense {n_cpu}×{n_cpu} decoder (scgnn2.py:425,557) on torch-CPU, best of 16/32/64/all intra-op "
            f"threads; the O(N²) decoder makes the per-cell CPU cost at the full {args.cells} cells ≈{max(1, args.cells // n_cpu)}× higher than in this sample")


def run_reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    n_cpu = min(args.cpu_cells, args.cells)
    med, ts = time_cpu(n_cpu, args.genes, args.steps, max(1, min(args.warmup, 1)))
    val = n_cpu / med
    line = {
        "impl": "reference", "metric": "cells/sec fwd+bwd scGNN", "value": val, "unit": "cells/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": med * 1e3, "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args),
        "cpu_baseline": {"value": val, "unit": "cells/s", "cores": time_cpu.threads, "host_cores": os.cpu_count(), "kind": time_cpu.kind,
                         "sample": cpu_sample_text(n_cpu, args)},
        "e2e": {"value": val, "unit": "cells/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


def workload_config(args):
    """Identical for both arms (the driver compares it): what one step computes; HOW each arm evaluates the decoder (dense N×N on the
    CPU sample, matrix-free blockwise on the GPU) is an implementation property reported outside `config`."""
    return {"workload": f"scGNN {args.cells} cells × {args.genes} genes: Feature_AE epoch (batch {BATCH}) + Graph_AE GCN epoch with the exact "
                        f"all-pairs inner-product decoder loss, k={K_NN} kNN graph",
            "cells": args.cells, "genes": args.genes, "feature_ae_batch": BATCH, "knn_k": K_NN, "graph_ae_embedding": EMB,
            "data_seed": DATA_SEED, "density": 0.10,
            "l2_policy": "inputs larger than L2 (X is %.1f GB; every step streams it)" % (args.cells * args.genes * 4 / 1e9)}


# ------------------------------------------------------------------------------------ GPU arm
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", type=str, default="b200", choices=["b200", "reference"])
    ap.add_argument("--cells", type=int, default=1_000_000)
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--precision", type=str, default="tf32x3", choices=["tf32x3", "tf32", "fp32"])
    ap.add_argument("--cpu-cells", type=int, default=16384, help="bounded CPU sample (cells) for cpu_baseline / --impl reference")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--cell-order", type=str, default="locality", choices=["locality", "data"],
                    help="order of the cells inside the Graph-AE at N=1: grouped by nearest embedding centroid (L2-resident gathers) or as given")
    ap.add_argument("--comm", type=str, default="torch", choices=["torch", "native"],
                    help="collectives of the data path under N > 1: torch.distributed (NCCL) or the C-ABI's own NCCL communicator (b2_comm_*)")
    ap.add_argument("--no-checks", action="store_true", help="skip the fp64 spot checks and the 16-bit aggregate side measurement")
    ap.add_argument("--cuda-profiler", action="store_true", help="bracket the timed region with cudaProfilerStart/Stop (for ncu --profile-from-start off)")
    ap.add_argument("--dump-outputs", type=str, default=None, metavar="DIR",
                    help="write what the last timed step computed as DIR/<name>.npy (rank 0; fixed seeded row sample of the embeddings)")
    args = ap.parse_args()
    if args.warmup < 3 and args.impl == "b200":
        args.warmup = 3

    if args.impl == "reference":
        run_reference_arm(args)
        return

    from dance_b200 import ops
    from dance_b200.engine import FeatureAEEngine, GraphAEEngine
    from dance_b200.parallel import Comm, shard_bounds

    comm = Comm.from_env()
    rank, world = comm.rank, comm.world
    if world != args.gpus and args.gpus > 1:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torchrun --nproc-per-node {args.gpus}")
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    peaks = load_peaks()
    ops.set_default_precision(args.precision)

    N, G = args.cells, args.genes
    bounds = shard_bounds(N, world)
    r0, r1 = bounds[rank]
    n_loc = r1 - r0

    # ---- setup (outside the timed region) ------------------------------------------------
    from dance_b200 import hostio, synth
    from dance_b200.parallel import epoch_steps
    X = synth_expression(n_loc, G, dev, row_begin=r0)
    fp = synth.fingerprint(X)
    fae = FeatureAEEngine(G, device=dev, lr=1e-3, precision=args.precision, seed=0)
    gae = GraphAEEngine(128, EMB, device=dev, lr=1e-2, precision=args.precision, seed=1)
    n_steps = None
    dcomm = comm                                   # communicator of the data path (gradient all-reduce, operand all-gathers)
    if comm.enabled and args.comm == "native":
        from dance_b200.parallel import NativeComm
        dcomm = NativeComm(rank, world)
    if comm.enabled:
        fae.grad_hook = dcomm.allreduce_sum_
        gae.set_sharding(dcomm, bounds)
        n_steps = epoch_steps(bounds, BATCH)       # every rank issues the same number of gradient all-reduces per epoch
    z_all = torch.empty(n_loc, 128, dtype=torch.float32, device=dev)
    fae.train_epoch(X, BATCH, "LTMG", 0.9, None, z_all, None, n_steps=n_steps)   # also serves as the first warm-up epoch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    z_full = comm.all_gather_rows(z_all, bounds) if comm.enabled else z_all
    idx_loc, _ = ops.knn(z_full, K_NN, include_rank0=False, q_begin=r0, q_end=r1, return_dist=False)
    idx_full = comm.all_gather_rows(idx_loc, bounds) if comm.enabled else idx_loc
    perm = None
    if not comm.enabled and args.cell_order == "locality":
        # locality-preserving cell order for the aggregate (cells grouped by nearest centroid of the embedding): the Graph-AE runs in
        # this order — the graph, the decoder loss and the weight gradients are permutation-equivariant — see ops.locality_order
        perm, inv = ops.locality_order(z_all, n_anchors=64)
        idx_full = inv[idx_full[perm].long()].to(torch.int32)
    A_full = ops.knn_graph_build(idx_full.contiguous())
    torch.cuda.synchronize()
    graph_build_s = time.perf_counter() - t0
    nnz_total = A_full.nnz
    if comm.enabled:   # local row block of Â (column ids stay global)
        rp = A_full.rowptr[r0:r1 + 1].clone()
        e0, e1 = int(rp[0].item()), int(rp[-1].item())
        A = ops.CSR((rp - e0).contiguous(), A_full.colidx[e0:e1].contiguous(), A_full.vals[e0:e1].contiguous(), (n_loc, N))
        del A_full
    else:
        A = A_full
    labels = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    adj_sum = nnz_total - N
    pos_weight = float(N * N - adj_sum) / adj_sum
    norm = N * N / float((N * N - adj_sum) * 2)
    gen = torch.Generator(device=dev).manual_seed(99 + rank)
    eps = torch.empty(n_loc, EMB, dtype=torch.float32, device=dev)

    ops.reset_counters()

    z_perm = torch.empty_like(z_all) if perm is not None else None

    def gae_input():
        if perm is None:
            return z_all
        torch.index_select(z_all, 0, perm, out=z_perm)      # one 0.5 GB gather per step buys L2-resident gathers in 4 aggregates
        return z_perm

    last = {}

    def step(x_src):
        last["fae_loss"] = fae.train_epoch(x_src, BATCH, "LTMG", 0.9, None, z_all, None, n_steps=n_steps)
        eps.normal_(generator=gen)
        last["gae_z"], last["gae_mu"], last["gae_logvar"] = gae.train_step(gae_input(), A, labels, norm, pos_weight, eps)

    def timed(fn, k):
        comm.barrier()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(k):
            fn()
        e.record()
        torch.cuda.synchronize()
        comm.barrier()
        t = torch.tensor([s.elapsed_time(e)], device=dev)
        comm.allreduce_max_(t)
        return float(t.item())

    for _ in range(args.warmup):
        step(X)
    torch.cuda.synchronize()

    # ---- parity spot checks on the exact code paths the timed region runs (fp64 closed forms on sampled rows) ----------------
    checks = parity_checks(ops, gae, A, labels, norm, pos_weight, N, r0, n_loc, comm, dev) if not args.no_checks else None

    # ---- timed region: device-resident inputs -----------------------------------------------
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    launches_before = ops.counters()["launches"]
    if args.cuda_profiler:
        torch.cuda.profiler.start()
    total_ms = timed(lambda: step(X), args.steps)
    if args.cuda_profiler:
        torch.cuda.profiler.stop()
    launches = ops.counters()["launches"] - launches_before
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(Path(args.dump_outputs), last, z_all, gae, inv if perm is not None else None)
    ms_per_step = total_ms / args.steps
    value = N / (ms_per_step / 1e3)

    # ---- per-kernel timing pass (CUDA events around every launch; same work, separate pass) ----
    ops.enable_kernel_timing(True)
    step(X)
    torch.cuda.synchronize()
    ktimes = ops.kernel_times()
    ops.enable_kernel_timing(False)

    # ---- 16-bit-operand aggregate on the same graph (the bf16 configuration's SpMM; not part of the fp32-grade step) ----------
    spmm16 = None
    if world == 1 and not args.no_checks:
        S = gae._buffers(n_loc)["s1"]
        S16 = ops.to_x16(S, torch.bfloat16)
        out = torch.empty_like(S)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        ts = []
        for it in range(6):
            flush.zero_()                                   # evict L2 between timed launches
            s_, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s_.record()
            ops.spmm(A, S16, out=out)
            e_.record()
            torch.cuda.synchronize()
            if it:
                ts.append(s_.elapsed_time(e_))
        ms16 = float(np.median(ts))
        b16 = A.nnz * 8 + (n_loc + 1) * 4 + N * 32 * 2 + n_loc * 32 * 4
        spmm16 = {"kernel": "spmm_stream_kernel<bf16, 64 B rows> (Â·support, F=32, bf16 operand, fp32 accumulate/output)", "bound": "hbm",
                  "achieved": b16 / (ms16 * 1e-3) / 1e9, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                  "frac": b16 / (ms16 * 1e-3) / 1e9 / peaks["hbm_gbs"], "ms_per_launch": ms16, "algorithmic_bytes": b16, "l2_policy": "256 MB flush between launches", "peak_source": peaks["source"]}
        del flush, S16, out

    # ---- e2e: the public handlers (numpy in / numpy out), host-resident pinned X, copies inside the timed region ---------------
    e2e = None
    if not args.no_e2e:
        from types import SimpleNamespace
        from dance_b200.modules import scgnn2 as mod
        Xh = torch.empty((n_loc, G), dtype=torch.float32, pin_memory=True)
        Xh.copy_(X)
        Xnp = Xh.numpy()
        del X
        torch.cuda.empty_cache()
        hargs = SimpleNamespace(feature_AE_batch_size=BATCH, feature_AE_epoch=[1, 1], feature_AE_learning_rate=1e-3,
                                feature_AE_regu_strength=0.9, feature_AE_dropout_prob=0, feature_AE_concat_prev_embed=None,
                                graph_AE_epoch=1, graph_AE_use_GAT=False, graph_AE_GAT_dropout=0, graph_AE_learning_rate=1e-2,
                                graph_AE_embedding_size=EMB, graph_AE_concat_prev_embed=None, graph_AE_normalize_embed=None,
                                graph_AE_neighborhood_factor=K_NN, graph_AE_retain_weights=False, gat_multi_heads=2, gat_hid_embed=64)
        param = {"device": dev, "epoch_num": 0, "total_epoch": 0, "n_feature_orig": G, "precision": args.precision, "seed": 0,
                 "io_pool": hostio.IOPool(), "graph_cache": {}, "cell_order": "locality" if args.cell_order == "locality" else None}
        out_bytes = {}

        def e2e_step():
            x_embed, x_recon, _ = mod.feature_AE_handler(Xnp, None, hargs, param)
            g_embed, _, edge_list, adj = mod.graph_AE_handler(x_embed, None, hargs, param)
            out_bytes["d2h"] = x_embed.nbytes + x_recon.nbytes + g_embed.nbytes
            out_bytes["h2d"] = Xnp.nbytes + x_embed.nbytes

        if world == 1:
            e2e_step()      # first call: allocates the pinned output buffers and builds + caches the kNN graph (not part of a step)
            e2e_step()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                e2e_step()
            torch.cuda.synchronize()
            e2e_ms = (time.perf_counter() - t0) * 1e3 / args.steps
            e2e = {"value": N / (e2e_ms / 1e3), "unit": "cells/s", "ms_per_step": e2e_ms,
                   "h2d_bytes_per_step": int(out_bytes["h2d"]), "d2h_bytes_per_step": int(out_bytes["d2h"]),
                   "api": "dance_b200.modules.scgnn2.feature_AE_handler + graph_AE_handler (numpy in / numpy out), feature_AE_epoch=1, graph_AE_epoch=1",
                   "note": "host wall clock around the two public handler calls. X is a pinned numpy array; the handler streams it in batch by "
                           "batch on a side stream while earlier batches train and streams the N×G reconstruction back to pinned host memory "
                           "the same way; returns X_embed, X_recon, graph_embed, edgeList, adj as host arrays. The kNN graph of the step's "
                           "embedding is taken from param['graph_cache'] (built in the untimed first call), like the reference arm which "
                           "builds its graph outside the timed step; graph_build_s reports that cost."}
        else:
            # multi-GPU: the handlers are single-device; the sharded engines are driven with per-batch pinned uploads instead
            stage = [torch.empty((BATCH, G), dtype=torch.float32, device=dev) for _ in range(2)]
            up = hostio.Uploader(Xh, dev)
            main_stream = torch.cuda.current_stream()
            loss_host = torch.empty(2, dtype=torch.float32, pin_memory=True)
            from dance_b200.parallel import batch_schedule
            sched = batch_schedule(n_loc, BATCH, n_steps)

            def e2e_step_mg():
                fae.loss_acc.zero_()
                free = [None, None]
                evs = {}
                def issue(b):
                    if sched[b] is None:
                        return
                    if free[b & 1] is not None:
                        up.stream.wait_event(free[b & 1])
                    b0, b1 = sched[b]
                    evs[b] = up.copy_rows(b0, b1, stage[b & 1][:b1 - b0])
                issue(0)
                for b, rng in enumerate(sched):
                    if b + 1 < len(sched):
                        issue(b + 1)
                    if rng is None:
                        fae.idle_step()
                        continue
                    b0, b1 = rng
                    main_stream.wait_event(evs.pop(b))
                    z, _ = fae.train_step(stage[b & 1][:b1 - b0], None, 0.9, "LTMG")
                    z_all[b0:b1].copy_(z)
                    fr = torch.cuda.Event()
                    fr.record(main_stream)
                    free[b & 1] = fr
                eps.normal_(generator=gen)
                gae.train_step(z_all, A, labels, norm, pos_weight, eps)
                loss_host[0:1].copy_(fae.loss_acc, non_blocking=True)
                loss_host[1:2].copy_(gae.loss, non_blocking=True)

            e2e_step_mg()
            e2e_ms = timed(e2e_step_mg, args.steps) / args.steps
            e2e = {"value": N / (e2e_ms / 1e3), "unit": "cells/s", "ms_per_step": e2e_ms,
                   "h2d_bytes_per_step": int(N * G * 4), "d2h_bytes_per_step": 8 * world,
                   "api": "sharded engines (FeatureAEEngine.train_step / GraphAEEngine.train_step) under torch.distributed",
                   "note": "X pinned on each rank's host, copied batch-by-batch on a side stream (double-buffered) inside the timed region; "
                           "per-step D2H = the two loss scalars per rank (the numpy-returning handlers are single-device)"}
        del Xh

    if rank != 0:
        return

    # ---- roofline of the kernels (algorithmic bytes / flops from DESIGN.md §kernels) ------------
    def kt(name):
        d = ktimes.get(name)
        return (d["ms"] / d["n"], d["n"], d["ms"]) if d else (None, 0, 0.0)

    F = 32
    spmm_ms, spmm_n, spmm_total = kt("spmm_csr_f32")
    nnz_loc = A.nnz
    spmm_bytes = nnz_loc * 8 + (n_loc + 1) * 4 + N * F * 4 + n_loc * F * 4
    roof_spmm = None
    if spmm_ms:
        ach = spmm_bytes / (spmm_ms * 1e-3) / 1e9
        roof_spmm = {"kernel": "spmm_stream_kernel<f32, 128 B rows> (Â·support, F=32, fp32 operand; nnz-stream pipeline, cp.async-staged gathers)", "bound": "hbm", "achieved": ach, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                     "frac": ach / peaks["hbm_gbs"], "launches": spmm_n, "ms_per_launch": spmm_ms,
                     "algorithmic_bytes": spmm_bytes, "gather_bytes_through_l2": nnz_loc * F * 4, "peak_source": peaks["source"]}
    gemm_ms, gemm_n, gemm_total = kt("gemm_f32")
    fae_flops = 6.0 * n_loc * (G * 512 + 512 * 128 + 128 * 512 + 512 * G)       # fwd + dX + dW, 2 flops per MAC
    gcn_flops = 6.0 * n_loc * (128 * 32 + 32 * 2 * EMB)
    roof_gemm = None
    if gemm_ms:
        ach = (fae_flops + gcn_flops) / (gemm_total * 1e-3) / 1e12
        roof_gemm = {"kernel": "gemm_tc_kernel (wgmma tf32, %s)" % args.precision, "bound": "tensor", "achieved": ach,
                     "peak": peaks["bf16_tflops_sustained"] or peaks["bf16_tflops"], "unit": "TFLOP/s",
                     "frac": ach / (peaks["bf16_tflops_sustained"] or peaks["bf16_tflops"]), "launches": gemm_n,
                     "ms_total": gemm_total, "algorithmic_flops": fae_flops + gcn_flops, "peak_source": peaks["source"],
                     "note": "achieved = fp32-equivalent algorithmic FLOPs; tf32x3 issues 3 tensor-core products per algorithmic product "
                             "and tf32 runs at half the bf16 rate, so the ceiling of this mode is peak/6"}
    dec_ms, dec_n, dec_total = kt("gae_loss_grad_f32")
    phases = {k: {"ms": v["ms"], "launches": v["n"]} for k, v in sorted(ktimes.items(), key=lambda kv: -kv[1]["ms"])}
    dominant = max(ktimes.items(), key=lambda kv: kv[1]["ms"])[0] if ktimes else None
    roofline = roof_gemm if dominant == "gemm_f32" else (roof_spmm if dominant == "spmm_csr_f32" else None)
    if roofline is None:
        # the exact N×N decoder is SFU/issue-bound; report it on the tensor roofline with its matmul flops (2·d per logit, S and G·Z)
        dec_flops = 2.0 * 2 * EMB * float(n_loc) * N
        ach = dec_flops / (dec_total * 1e-3) / 1e12 if dec_total else 0.0
        roofline = {"kernel": "gae_allpairs_tc_kernel (matrix-free z·zᵀ BCE decoder: wgmma tf32 hi/lo split, S and G in registers, "
                              "row sweep over all 128×128 tiles)",
                    "bound": "tensor", "achieved": ach,
                    "peak": peaks["bf16_tflops_sustained"] or peaks["bf16_tflops"], "unit": "TFLOP/s",
                    "frac": ach / (peaks["bf16_tflops_sustained"] or peaks["bf16_tflops"]), "launches": dec_n, "ms_total": dec_total, "peak_source": peaks["source"],
                    "logits_per_s": float(n_loc) * N / (dec_total * 1e-3) if dec_total else None,
                    "note": "dominant kernel of the step; algorithmic flops = the two K=16 products per logit (S and G·Z) over ALL N² ordered "
                            "pairs. Its real ceiling is the per-logit elementwise work (2 MUFU + ~11 ALU instructions per logit), not the tensor "
                            "pipe or HBM; roofline_spmm / roofline_gemm are the HBM- and tensor-bound kernels"}

    cpu_baseline, matched = None, None
    if not args.no_cpu_baseline and world == 1:
        n_cpu = min(args.cpu_cells, N)
        med, ts = time_cpu(n_cpu, G, steps=2, warmup=1)
        cpu_baseline = {"value": n_cpu / med, "unit": "cells/s", "cores": time_cpu.threads, "host_cores": os.cpu_count(), "kind": time_cpu.kind,
                        "sample": cpu_sample_text(n_cpu, args), "s_per_step": med}
        # like-for-like line: the GPU arm on exactly the CPU arm's sample (same rows of the same matrix, same step)
        gm = gpu_step_ms(n_cpu, G, dev, args.precision)
        matched = {"cells": n_cpu, "gpu_cells_per_s": n_cpu / (gm / 1e3), "gpu_ms_per_step": gm, "cpu_cells_per_s": n_cpu / med,
                   "ratio": (n_cpu / (gm / 1e3)) / (n_cpu / med),
                   "note": "same-N comparison; the headline value / reference ratio is cross-N (GPU at the full size, CPU on this sample)"}

    line = {
        "metric": "cells/sec fwd+bwd scGNN", "value": value, "unit": "cells/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "f32 (wgmma 3xTF32 split GEMMs, fp32 everything else)" if args.precision == "tf32x3" else args.precision,
        "data": "synthetic",
        "config": workload_config(args),
        "implementation": {"decoder_loss": "exact-fused-blockwise (matrix-free, no N×N tensors)", "gemm_precision": args.precision,
                           "collectives": ("C-ABI NCCL communicator (b2_comm_*)" if args.comm == "native" else "torch.distributed NCCL") if world > 1 else None,
                           "parallelism": f"cells sharded ×{world}", "nnz": nnz_total, "data_fingerprint_rank0": fp,
                           "graph_ae_cell_order": ("locality (64 centroids)" if perm is not None else "data order")},
        "clocks": clocks, "e2e": e2e, "gpu_launches": launches // args.steps, "checks": checks,
        "roofline": roofline, "roofline_spmm": roof_spmm, "roofline_spmm_bf16": spmm16, "roofline_gemm": roof_gemm,
        "cpu_baseline": cpu_baseline, "matched_n": matched,
        "kernel_ms_per_step": phases, "graph_build_s": graph_build_s,
    }
    print(json.dumps(line), flush=True)


DUMP_ROWS = 65536


def dump_outputs(out_dir, last, z_all, gae, inv):
    """What a caller of the timed step receives after its last step, as float32 / float64 .npy files (≤ 64 MB in all): the two
    losses, the Feature-AE embedding and the Graph-AE z / mu / logvar on a fixed seeded sample of DUMP_ROWS cells (rows in the
    data's cell order, whatever order the Graph-AE ran in), and the Graph-AE weights after the step's Adam update."""
    out_dir.mkdir(parents=True, exist_ok=True)
    n = z_all.shape[0]
    rows = np.sort(np.random.default_rng(1234).choice(n, size=min(n, DUMP_ROWS), replace=False))
    rows_t = torch.from_numpy(rows).to(z_all.device)
    gae_rows = inv[rows_t].long() if inv is not None else rows_t           # position of each sampled cell in the Graph-AE's order
    arrays = {"cell_index": rows.astype(np.float64),
              "feature_ae_loss": last["fae_loss"].double().cpu().numpy(),
              "feature_ae_embedding": z_all[rows_t].float().cpu().numpy(),
              "graph_ae_loss": gae.loss.double().cpu().numpy()}
    for name in ("z", "mu", "logvar"):
        arrays[f"graph_ae_{name}"] = last[f"gae_{name}"][gae_rows].float().cpu().numpy()
    for name, w in gae.state_dict().items():
        arrays[f"graph_ae_{name.replace('.', '_')}"] = w.float().cpu().numpy()
    for name, a in arrays.items():
        np.save(out_dir / f"{name}.npy", a)


def gae_reference_rows(z, rowptr, colidx, norm, pw, rows, chunk=256):
    """fp64 closed form of gae_loss_function (scgnn2.py:603-612) for `rows` × all columns on the device (checker, plain torch):
    returns (Σ cost over those rows · norm / n², gradient rows).  cost = y·pw·softplus(−x) + (1−y)·softplus(x); labels symmetric ⇒
    ∂/∂z_i = 2·Σ_j c_ij z_j with c = σ(x) off the pattern and −pw·σ(−x) on it."""
    import torch.nn.functional as F
    zd = z.double()
    n = zd.shape[0]
    rp = rowptr.long()
    loss = 0.0
    out = torch.empty(len(rows), zd.shape[1], dtype=torch.float64, device=z.device)
    for a in range(0, len(rows), chunk):
        r = rows[a:a + chunk]
        x = zd[r] @ zd.t()
        c = torch.sigmoid(x)
        cost = F.softplus(x)
        cnt = rp[r + 1] - rp[r]
        loc = torch.repeat_interleave(torch.arange(len(r), device=z.device), cnt)
        start = torch.repeat_interleave(rp[r], cnt)
        within = torch.arange(int(cnt.sum()), device=z.device) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
        cols = colidx.long()[start + within]
        xe = x[loc, cols]
        cost[loc, cols] = pw * F.softplus(-xe)
        c[loc, cols] = -pw * torch.sigmoid(-xe)
        loss += float(cost.sum())
        out[a:a + chunk] = 2.0 * (c @ zd)
    return norm * loss / (float(n) * n), out * (norm / (float(n) * n))


def parity_checks(ops, gae, A, labels, norm, pos_weight, N, r0, n_loc, comm, dev):
    """Spot checks of the code paths the timed region runs, at the benchmark's own size: (1) decoder gradient rows of the full-size
    call (the j_splits == 1 / non-atomic epilogue branch at 1 GPU) and the loss of a row block against the fp64 closed form;
    (2) aggregate rows against an fp64 gather-sum.  Raises on a mismatch."""
    b = gae._buffers(n_loc)
    z_loc = b["z"]
    z_all = gae._gather(z_loc, "z")
    out = {"z_finite": bool(torch.isfinite(z_all).all()), "z_absmax": float(z_all.abs().max()), "train_loss": float(gae.loss.item())}
    assert out["z_finite"], f"Graph-AE embedding is not finite after the warm-up steps: {out}"
    g = torch.Generator(device=dev).manual_seed(7)
    rows_loc = torch.randint(0, n_loc, (96, ), device=dev, generator=g)
    loss = torch.zeros(1, dtype=torch.float32, device=dev)
    gcomm = getattr(gae, "comm", None)
    if gcomm is not None and gcomm.enabled:
        # what GraphAEEngine.train_step runs under sharding: this rank's share of the block-pair schedule, partial gradients for ALL
        # rows, summed over ranks
        from dance_b200.parallel import shard_bounds
        sb0, sb1 = shard_bounds(ops.gae_sym_super_blocks(N), gcomm.world)[gcomm.rank]
        dzf = torch.empty(N, z_loc.shape[1], dtype=torch.float32, device=dev)
        ops.gae_loss_grad_sym(z_all, labels, norm, pos_weight, sb0, sb1, dz_full=dzf, loss=loss, row_begin=r0, n_rows=n_loc)
        gcomm.allreduce_sum_(dzf)
        gcomm.allreduce_sum_(loss)
        dz = dzf[r0:r0 + n_loc]
        out["decoder_path"] = "pair-sharded symmetric decoder + all-reduce(dz)"
    else:
        dz = torch.empty(n_loc, z_loc.shape[1], dtype=torch.float32, device=dev)
        ops.gae_loss_grad(z_all, labels, norm, pos_weight, dz=dz, loss=loss, row_begin=r0, n_rows=n_loc)
    # reference rows need the label pattern of the sampled rows in GLOBAL numbering: shift the local CSR rows
    class _Shift:   # minimal view: rowptr indexable by global row id
        pass
    rp_full = torch.zeros(N + 1, dtype=A.rowptr.dtype, device=dev)
    rp_full[r0:r0 + n_loc + 1] = A.rowptr
    if r0 + n_loc < N:
        rp_full[r0 + n_loc + 1:] = A.rowptr[-1]
    _, ref_rows = gae_reference_rows(z_all, rp_full, A.colidx, norm, pos_weight, rows_loc + r0)
    out["dz_finite"] = bool(torch.isfinite(dz).all())
    err = float((dz[rows_loc].double() - ref_rows).norm() / ref_rows.norm())
    out["decoder_grad_rel_err_96_rows"] = err
    assert err < 1e-4, f"decoder gradient mismatch at full size: rel err {err}"      # north_star tolerance; typical 5e-7 … 7e-6
    # loss of a 512-row block through the same entry point (row-sharded form) against fp64
    blk = torch.arange(0, min(512, n_loc), device=dev)
    sub = ops.CSR(A.rowptr[:len(blk) + 1].contiguous(), A.colidx[:int(A.rowptr[len(blk)].item())].contiguous(), None, (len(blk), N))
    lb, _, _, _ = ops.gae_loss_grad(z_all, sub, norm, pos_weight, row_begin=r0, n_rows=len(blk))
    ref_l, _ = gae_reference_rows(z_all, rp_full, A.colidx, norm, pos_weight, blk + r0)
    out["decoder_loss_rel_err_512_rows"] = abs(lb.item() - ref_l) / abs(ref_l)
    assert out["decoder_loss_rel_err_512_rows"] < 1e-5, f"decoder loss mismatch: {lb.item()} vs {ref_l}"
    # aggregate rows
    S = gae._gather(b["s1"], "s1")
    Y = ops.spmm(A, S)
    rp = A.rowptr.long()
    rr = rows_loc[:32]
    e = 0.0
    for i in rr.tolist():
        cols = A.colidx[rp[i]:rp[i + 1]].long()
        ref = (A.vals[rp[i]:rp[i + 1]].double()[:, None] * S[cols].double()).sum(0)
        e = max(e, float((Y[i].double() - ref).norm() / ref.norm().clamp(min=1e-30)))
    out["spmm_rel_err_32_rows"] = e
    assert e < 1e-5, f"aggregate mismatch: {e}"
    out["decoder_loss"] = float(loss.item())
    return out


def gpu_step_ms(n, G, dev, precision, steps=5):
    """Device-timed ms per scGNN step on the first `n` cells of the dataset (the CPU arm's sample) — single GPU."""
    from dance_b200 import ops
    from dance_b200.engine import FeatureAEEngine, GraphAEEngine
    X = synth_expression(n, G, dev)
    fae = FeatureAEEngine(G, device=dev, lr=1e-3, precision=precision, seed=0)
    gae = GraphAEEngine(128, EMB, device=dev, lr=1e-2, precision=precision, seed=1)
    z_all = torch.empty(n, 128, dtype=torch.float32, device=dev)
    fae.train_epoch(X, BATCH, "LTMG", 0.9, None, z_all, None)
    idx, _ = ops.knn(z_all, K_NN, include_rank0=False, return_dist=False)
    A = ops.knn_graph_build(idx)
    labels = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    adj_sum = A.nnz - n
    pw, norm = float(n * n - adj_sum) / adj_sum, n * n / float((n * n - adj_sum) * 2)
    eps = torch.randn(n, EMB, device=dev)

    def step():
        fae.train_epoch(X, BATCH, "LTMG", 0.9, None, z_all, None)
        gae.train_step(z_all, A, labels, norm, pw, eps)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        step()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


if __name__ == "__main__":
    main()
