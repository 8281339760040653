"""world_size-2 gloo tests (CPU) of the cell-sharded decomposition used on N GPUs (dance_b200/parallel.py,
GraphAEEngine.set_sharding): shard bounds, uneven all-gather, and — with the oracle's torch-CPU arithmetic in
place of the CUDA kernels — that the row-sharded GCN forward/backward + all-reduce reproduces the unsharded
loss and weight gradients, and that data-parallel Feature-AE gradients sum to the global-batch gradient."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, fn_name, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    sys.path.insert(0, str(ROOT))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        q.put((rank, globals()[fn_name](rank, world)))
    finally:
        dist.destroy_process_group()


def _run(fn_name, world=2):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, fn_name, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return out


def test_shard_bounds():
    from dance_b200.parallel import shard_bounds
    for n, w in ((10, 3), (7, 8), (1_000_000, 8), (5, 1)):
        b = shard_bounds(n, w)
        assert b[0][0] == 0 and b[-1][1] == n and all(b[i][1] == b[i + 1][0] for i in range(w - 1))
        sizes = [e - s for s, e in b]
        assert max(sizes) - min(sizes) <= 1


def _gather_case(rank, world):
    from dance_b200.parallel import Comm, shard_bounds
    comm = Comm()
    bounds = shard_bounds(11, world)   # uneven: 6 + 5
    full = torch.arange(11 * 3, dtype=torch.float32).view(11, 3)
    a, b = bounds[rank]
    out = comm.all_gather_rows(full[a:b].clone(), bounds)
    t = torch.tensor([float(rank + 1)])
    comm.allreduce_sum_(t)
    return bool(torch.equal(out, full)) and t.item() == 3.0 and comm.world == 2


def test_all_gather_rows_uneven_gloo():
    assert all(_run("_gather_case").values())


def _sharded_gcn_case(rank, world):
    """Row-sharded Graph-AE step with the communication pattern of GraphAEEngine.train_step."""
    from dance_b200.parallel import Comm, shard_bounds
    from oracle import port
    comm = Comm()
    n, d, e = 203, 16, 16
    X = torch.from_numpy(port.synthetic_embedding(n, d=d, n_clusters=3, seed=2))
    adj, _ = port.feature2adj(X.numpy(), 8)
    an = port.preprocess_graph(adj)
    pw, norm = port.gae_norm_constants(adj)
    torch.manual_seed(0)
    w1, w2, w3 = (torch.nn.init.xavier_uniform_(torch.empty(d, 32)), torch.nn.init.xavier_uniform_(torch.empty(32, e)),
                  torch.nn.init.xavier_uniform_(torch.empty(32, e)))
    eps = torch.randn(n, e)
    # unsharded reference (autograd)
    W = [w.clone().requires_grad_() for w in (w1, w2, w3)]
    loss_ref, *_ = port.graph_ae_gcn_loss(X, *W, an, adj, eps=eps)
    loss_ref.backward()

    bounds = shard_bounds(n, world)
    a, b = bounds[rank]
    A_loc = torch.from_numpy(an[a:b].toarray())                      # local row block of Â, global columns
    L_loc = torch.from_numpy((adj + sp.eye(n)).tocsr()[a:b].toarray()).float()
    x, ep = X[a:b], eps[a:b]
    gather = lambda t: comm.all_gather_rows(t.contiguous(), bounds)
    # forward
    s1 = x @ w1
    h1 = torch.relu(A_loc @ gather(s1))
    w23 = torch.cat([w2, w3], 1)
    ml = A_loc @ gather(h1 @ w23)
    mu, lv = ml[:, :e], ml[:, e:]
    z = mu + ep * torch.exp(lv)
    z_all = gather(z)
    # loss share of this shard: rows local × all columns (constants use the global n)
    logits = z @ z_all.t()
    bce = torch.nn.functional.binary_cross_entropy_with_logits(logits, L_loc, pos_weight=L_loc * pw, reduction="sum")
    kld = -0.5 / n * torch.sum(1 + 2 * lv - mu.pow(2) - lv.exp().pow(2)) / n
    loss = norm * bce / (n * n) + kld
    # gradients wrt the local rows (L symmetric ⇒ factor 2 on the decoder part)
    sig = torch.sigmoid(logits)
    g = norm / (n * n) * (sig * (1 - L_loc) - pw * L_loc * (1 - sig))
    dz = 2 * g @ z_all
    cf = -0.5 / (n * n)
    dmu = cf * (-2 * mu) + dz
    dlv = cf * (2 - 2 * lv.exp().pow(2)) + dz * ep * torch.exp(lv)
    dml = torch.cat([dmu, dlv], 1)
    ds2 = A_loc @ gather(dml)                                        # Âᵀ·dY on local rows = Â_loc·gather(dY) (Â symmetric)
    g23 = h1.t() @ ds2
    dh1 = (ds2 @ w23.t()) * (h1 > 0)
    ds1 = A_loc @ gather(dh1)
    g1 = x.t() @ ds1
    flat = torch.cat([g1.reshape(-1), g23.reshape(-1), loss.reshape(1)])
    comm.allreduce_sum_(flat)
    g1r, g23r, lossr = flat[:d * 32].view(d, 32), flat[d * 32:-1].view(32, 2 * e), flat[-1]
    rel = lambda p, q: (torch.norm(p - q) / torch.norm(q)).item()
    return (abs(lossr.item() - loss_ref.item()) / abs(loss_ref.item()), rel(g1r, W[0].grad), rel(g23r[:, :e], W[1].grad),
            rel(g23r[:, e:], W[2].grad))


def test_sharded_gcn_matches_unsharded_gloo():
    for rank, errs in _run("_sharded_gcn_case").items():
        assert max(errs) < 1e-5, (rank, errs)


def _dp_feature_ae_case(rank, world):
    """Sum-reduced per-shard gradients == gradient of the loss over the union batch (loss uses reduction='sum')."""
    from dance_b200.parallel import Comm, shard_bounds
    from oracle import port
    comm = Comm()
    X = torch.from_numpy(port.synthetic_expression(64, 24, density=0.3, seed=1))
    torch.manual_seed(0)
    model = port.FeatureAE(24)
    ref = port.FeatureAE(24)
    ref.load_state_dict(model.state_dict())
    _, r = ref(X)
    port.feature_ae_loss(r, X, "LTMG", 0.9, torch.zeros_like(X)).backward()
    a, b = shard_bounds(64, world)[rank]
    _, r = model(X[a:b])
    port.feature_ae_loss(r, X[a:b], "LTMG", 0.9, torch.zeros_like(X[a:b])).backward()
    flat = torch.cat([p.grad.reshape(-1) for p in model.parameters()])
    comm.allreduce_sum_(flat)
    flat_ref = torch.cat([p.grad.reshape(-1) for p in ref.parameters()])
    return (torch.norm(flat - flat_ref) / torch.norm(flat_ref)).item()


def test_symmetric_decoder_schedule_covers_every_block_pair_once():
    """The decoder's super-blocks (csrc/gae_tc.cu) restated on the host: over all super-blocks every ordered pair of 128-row blocks
    appears exactly once, the work per super-block is balanced, and contiguous super-block ranges (the multi-GPU shards) partition it."""
    from dance_b200.parallel import shard_bounds, sym_schedule, sym_super_blocks
    for nb in list(range(1, 14)) + [31, 32, 61]:
        nsb = (nb + 1) // 2
        assert sym_super_blocks(nb * 128) == nsb and sym_super_blocks(nb * 128 - 5) == nsb
        seen = {}
        loads = []
        for sb in range(nsb):
            tiles = sym_schedule(nb, sb)
            loads.append(len(tiles))
            for I, J in tiles:
                key = (I, J)
                assert key not in seen, (nb, key)
                seen[key] = sb
                assert I in (sb, nb - 1 - sb)
        assert len(seen) == nb * nb, nb
        full = [l for l, sb in zip(loads, range(nsb)) if sb != nb - 1 - sb]
        if full:
            assert max(full) - min(full) <= 2, (nb, loads)
        for world in (2, 3):
            parts = [sum(loads[a:b]) for a, b in shard_bounds(nsb, world)]
            assert sum(parts) == sum(loads)


def _pair_sharded_decoder_case(rank, world):
    """Pair-sharded decoder gradient (GraphAEEngine.train_step under sharding): each rank evaluates the tiles of its super-blocks —
    dZ_I += G·Z_J — into a full-size buffer; the all-reduced sum equals the dense gradient and the loss shares add up to the dense
    loss.  torch-CPU arithmetic in place of the CUDA kernel."""
    from dance_b200.parallel import Comm, shard_bounds, sym_schedule, sym_super_blocks
    comm = Comm()
    torch.manual_seed(0)
    n, d, B = 333, 16, 32                         # small blocks so that several super-blocks exist
    z = torch.randn(n, d, dtype=torch.float64) * 0.5
    nb = (n + B - 1) // B
    nsb = (nb + 1) // 2
    sb0, sb1 = shard_bounds(nsb, world)[rank]
    dz = torch.zeros(n, d, dtype=torch.float64)
    loss = torch.zeros(1, dtype=torch.float64)
    for sb in range(sb0, sb1):
        for I, J in sym_schedule(nb, sb):
            ri, rj = slice(I * B, min(n, (I + 1) * B)), slice(J * B, min(n, (J + 1) * B))
            S = z[ri] @ z[rj].t()
            G = torch.sigmoid(S)
            dz[ri] += G @ z[rj]
            loss += torch.nn.functional.softplus(S).sum()
    dz *= 2
    comm.allreduce_sum_(dz)
    comm.allreduce_sum_(loss)
    S = z @ z.t()
    ref = 2 * torch.sigmoid(S) @ z
    return (torch.norm(dz - ref) / torch.norm(ref)).item(), abs(loss.item() - torch.nn.functional.softplus(S).sum().item()) / loss.item()


def test_pair_sharded_decoder_matches_dense_gloo():
    for rank, errs in _run("_pair_sharded_decoder_case").items():
        assert max(errs) < 1e-12, (rank, errs)


def _uneven_epoch_case(rank, world):
    """Feature-AE data parallelism with uneven shards (ADVICE r1): 21 cells on 2 ranks, batch 5 → 11 / 10 rows = 3 / 2 local
    batches.  Driving FeatureAEEngine.train_epoch's schedule (parallel.batch_schedule + idle steps) with the oracle's torch-CPU
    model in place of the CUDA kernels: every rank issues epoch_steps() all-reduces (no hang) and the replicas stay identical
    and equal to single-process training on the union batches."""
    from dance_b200.parallel import Comm, batch_schedule, epoch_steps, shard_bounds
    from oracle import port
    comm = Comm()
    n, g, bs = 21, 12, 5
    X = torch.from_numpy(port.synthetic_expression(n, g, density=0.4, seed=3))
    bounds = shard_bounds(n, world)
    steps = epoch_steps(bounds, bs)
    a, b = bounds[rank]
    torch.manual_seed(0)
    model = port.FeatureAE(g)
    ref = port.FeatureAE(g)
    ref.load_state_dict(model.state_dict())
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    ropt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    sched = batch_schedule(b - a, bs, steps)
    n_coll = 0
    for rng in sched:
        opt.zero_grad()
        if rng is not None:
            xb = X[a:b][rng[0]:rng[1]]
            _, r = model(xb)
            port.feature_ae_loss(r, xb, "LTMG", 0.9, torch.zeros_like(xb)).backward()
        flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in model.parameters()])
        comm.allreduce_sum_(flat)
        n_coll += 1
        o = 0
        for p in model.parameters():
            p.grad = flat[o:o + p.numel()].view_as(p).clone()
            o += p.numel()
        opt.step()
    # single-process reference: step s trains on the union of every rank's s-th batch
    for s in range(steps):
        rows = []
        for ra, rb in bounds:
            sc = batch_schedule(rb - ra, bs, steps)[s]
            if sc is not None:
                rows += list(range(ra + sc[0], ra + sc[1]))
        ropt.zero_grad()
        xb = X[rows]
        _, r = ref(xb)
        port.feature_ae_loss(r, xb, "LTMG", 0.9, torch.zeros_like(xb)).backward()
        ropt.step()
    pf = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
    rf = torch.cat([p.detach().reshape(-1) for p in ref.parameters()])
    return n_coll, steps, len([s for s in sched if s is None]), (torch.norm(pf - rf) / torch.norm(rf)).item()


def test_uneven_shards_issue_equal_collectives_gloo():
    out = _run("_uneven_epoch_case")
    assert out[0][0] == out[1][0] == out[0][1] == 3
    assert out[0][2] == 0 and out[1][2] == 1          # rank 1 pads one idle step
    assert max(v[3] for v in out.values()) < 1e-5


def test_data_parallel_feature_ae_gradients_gloo():
    assert max(_run("_dp_feature_ae_case").values()) < 1e-5


def test_symmetric_decoder_step_ranges_cover_every_tile_once():
    """The decoder cuts each super-block's J sweep into step ranges (one CTA each): for every block count and every number of
    parts the union of the parts' tiles is the super-block's tile list, without overlap — including more parts than steps."""
    from dance_b200.parallel import sym_schedule, sym_step_range, sym_steps, sym_super_blocks
    for nb in (1, 2, 3, 8, 13, 16, 17, 64, 65):
        seen = set()
        for sb in range(sym_super_blocks(nb * 128)):
            steps = sym_steps(nb, sb)
            flat = [t for st in steps for t in st]
            assert sorted(flat) == sorted(sym_schedule(nb, sb)) and all(steps[i] for i in range(len(steps)))
            for splits in (1, 2, 3, 5, 8, len(steps) + 3):
                parts = [sym_step_range(len(steps), p, splits) for p in range(splits)]
                assert parts[0][0] == 0 and parts[-1][1] == len(steps) and all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
                got = [t for s0, s1 in parts for st in steps[s0:s1] for t in st]
                assert got == flat
            assert not seen.intersection(flat)
            seen.update(flat)
        assert len(seen) == nb * nb                     # every ordered block pair exactly once over all super-blocks


def test_spmm_stream_partition_balances_rows_and_nonzeros():
    """Row ranges of the nnz-stream aggregate's warps: a partition of the rows in order, balanced by (non-zeros + rows) up to one
    row — for uniform degrees, hub rows, long runs of empty rows and an all-empty matrix."""
    from dance_b200.parallel import spmm_stream_partition
    rng = np.random.default_rng(0)
    cases = [rng.integers(20, 40, 5000), np.r_[rng.integers(0, 5, 3000), 9000, rng.integers(0, 5, 3000)], np.r_[np.zeros(4000, int), rng.integers(1, 60, 500), np.zeros(700, int)],
             np.zeros(300, int), np.array([5])]
    for deg in cases:
        rp = np.r_[0, np.cumsum(deg)]
        for W in (1, 7, 64, 1000):
            parts = spmm_stream_partition(rp, W)
            assert parts[0][0] == 0 and parts[-1][1] == len(deg) and all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
            load = np.array([rp[r1] - rp[r0] + (r1 - r0) for r0, r1 in parts])
            assert load.sum() == deg.sum() + len(deg)
            assert load.max() <= (deg.sum() + len(deg)) / W + deg.max() + 2      # at most one row over the even share


def test_spmm_stream_traversal_emulation_matches_csr_product():
    """Control flow of spmm_stream_kernel restated on the host — per warp: 32-entry blocks of its non-zero stream, consumed in
    order with a (row, row_end) cursor that emits a row whenever row_end ≤ position, NPI lane groups splitting each run, tail emission
    of rows that end at the stream's end — against the CSR product.  Guards the algorithm (block / row boundary cases), not the CUDA."""
    import scipy.sparse as sp
    from dance_b200.parallel import spmm_stream_partition
    rng = np.random.default_rng(1)
    n, c, F, BLK, NPI = 700, 300, 8, 32, 4
    deg = rng.integers(0, 50, n)
    deg[50:120] = 0; deg[300] = 900; deg[400:432] = 32; deg[-40:] = 0
    rows = np.repeat(np.arange(n), deg)
    m = sp.csr_matrix((rng.normal(size=rows.size), (rows, rng.integers(0, c, rows.size))), shape=(n, c))
    m.sum_duplicates(); m.sort_indices()
    X = rng.normal(size=(c, F))
    rp, ci, va = m.indptr.astype(np.int64), m.indices, m.data
    Y = np.full((n, F), np.nan)
    for R0, R1 in spmm_stream_partition(rp, 13):
        if R0 >= R1:
            continue
        E0, E1 = rp[R0], rp[R1]
        nblk = -(-(E1 - E0) // BLK)
        r, rend = R0, rp[R0 + 1]
        acc = np.zeros((NPI, F))                       # one partial sum per lane group

        def emit():
            nonlocal r, rend, acc
            Y[r] = acc.sum(0)
            acc = np.zeros((NPI, F))
            r += 1
            rend = rp[min(r + 1, n)]
        for b in range(nblk):
            eb, eend = E0 + b * BLK, min(E1, E0 + (b + 1) * BLK)
            e = eb
            while True:
                while r < R1 and rend <= e:
                    emit()
                if e >= eend or r >= R1:
                    break
                run_end = min(rend, eend)
                for k in range(e, run_end):
                    acc[(k - e) % NPI] += va[k] * X[ci[k]]
                e = run_end
        while r < R1:
            emit()
    assert not np.isnan(Y).any() and np.allclose(Y, m @ X, rtol=1e-12, atol=1e-12)
