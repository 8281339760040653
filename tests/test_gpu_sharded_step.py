"""The cell-sharded scGNN step on one GPU: P ranks emulated by P threads of this process, each with its own engine.

Under ``GraphAEEngine.set_sharding`` a rank runs the SpMMs on its row block of Â over all-gathered operands, the pair-sharded
decoder ``gae_loss_grad_sym`` (its super-blocks of the block-pair schedule into a full-size dz, all-reduced), and all-reduces
the weight gradients and the loss; the data-parallel Feature-AE all-reduces each step's gradient, with idle steps on ranks whose
shard has fewer batches.  Those are the device code paths of a multi-GPU run.  :class:`LockstepComm` stands in for
``parallel.Comm``: the ranks take turns, exactly one running between two collectives (they share ``ops``' cached workspace and
the default stream), and the last rank to reach a collective reduces in rank order and hands every rank the result.

The pair-sharded decoder is tested directly against float64 and against the row-form call, with exact checks of the rows a rank
must leave at zero and of the KLD rows; the sharded Graph-AE step against float64 (every step, from the GPU's own weights), against
the unsharded engine and across ranks; the data-parallel Feature-AE epoch against float64 on the union batches.
"""
import threading
import time

import pytest
import torch

from conftest import rel_err
from oracle import scgnn_step_ref as R
from retain_weights_ref import decoder_loss_grad, gae_constants
from step_compare import adam_reference, param_views, row_rel_err


# ---------------------------------------------------------------------------------------------------- lock-step communicator
class _Released(Exception):
    """Unwinds a rank after another rank failed."""


class Lockstep:
    """What the emulated ranks share: whose turn it is, the number of finished collectives, the collective of this round and
    the tensors the ranks deposited for it, and the first failure."""

    def __init__(self, world: int, timeout: float):
        self.world, self.timeout = world, timeout
        self.cond = threading.Condition()
        self.turn, self.round, self.kind, self.deposits = 0, 0, None, []
        self.error = None                          # (rank or None, exception)

    def fail(self, rank, exc):
        with self.cond:
            if self.error is None:
                self.error = (rank, exc)
            self.cond.notify_all()

    def wait(self, pred, what: str):
        """Under ``cond``: block until ``pred()``; a failure elsewhere or ``timeout`` seconds without it unwinds this rank."""
        if not self.cond.wait_for(lambda: self.error is not None or pred(), self.timeout):
            if self.error is None:
                self.error = (None, TimeoutError(f"no progress for {self.timeout:g} s while waiting for {what}"))
            self.cond.notify_all()
        if self.error is not None:
            raise _Released()

    def arrive(self, rank: int, kind: str, payload, resolve=None):
        """``rank`` (holding the baton) reaches collective ``kind`` ("exit": its function returned) and passes the baton on.  The
        last rank calls ``resolve(deposits)`` with every rank's payload in rank order and gives the baton back to rank 0; each rank
        then continues when its turn comes again."""
        with self.cond:
            assert self.turn == rank, (self.turn, rank)
            if self.kind is None:
                self.kind = kind
            elif kind != self.kind:
                raise RuntimeError(f"rank {rank} reached {kind!r} where rank 0 reached {self.kind!r} (collective #{self.round})")
            self.deposits.append(payload)
            rnd = self.round
            if rank + 1 < self.world:
                self.turn = rank + 1
            else:
                if resolve is not None:
                    resolve(self.deposits)
                self.kind, self.deposits = None, []
                self.round, self.turn = rnd + 1, 0
            self.cond.notify_all()
            if kind != "exit":
                self.wait(lambda: self.round > rnd and self.turn == rank, f"collective #{rnd} ({kind}) on rank {rank}")


class LockstepComm:
    """``parallel.Comm``'s interface over :class:`Lockstep`: sums and maxima in fixed rank order, written into every rank's
    tensor; row gathers into ``out`` when it is given (``GraphAEEngine._gather`` relies on that)."""

    def __init__(self, rank: int, world: int, shared: Lockstep):
        self.rank, self.world, self.shared = rank, world, shared
        self.enabled = world > 1

    @staticmethod
    def _same(ts):
        if any(t.shape != ts[0].shape or t.dtype != ts[0].dtype for t in ts):
            raise RuntimeError(f"collective over mismatched tensors {[(tuple(t.shape), t.dtype) for t in ts]}")

    def _reduce(self, kind, t, op):
        def resolve(ts):
            self._same(ts)
            acc = ts[0].clone()
            for u in ts[1:]:
                acc = op(acc, u)
            for u in ts:
                u.copy_(acc)
        self.shared.arrive(self.rank, kind, t, resolve)
        return t

    def allreduce_sum_(self, t):
        return self._reduce("allreduce_sum", t, torch.add)

    def allreduce_max_(self, t):
        return self._reduce("allreduce_max", t, torch.maximum)

    def all_gather_rows(self, local, bounds, out=None):
        if not self.enabled:
            return local
        if out is None:
            out = torch.empty((bounds[-1][1], local.shape[1]), dtype=local.dtype, device=local.device)

        def resolve(deps):
            for r, (loc, _) in enumerate(deps):
                if loc.shape[0] != bounds[r][1] - bounds[r][0]:
                    raise RuntimeError(f"rank {r} contributed {loc.shape[0]} rows to a gather of bounds {bounds[r]}")
            full = torch.cat([loc for loc, _ in deps])
            for _, o in deps:
                o.copy_(full)
        self.shared.arrive(self.rank, "all_gather_rows", (local, out), resolve)
        return out

    def barrier(self):
        self.shared.arrive(self.rank, "barrier", None)


def run_ranks(world: int, fn, timeout: float = 120.0):
    """``fn(comm)`` on ``world`` emulated ranks, one thread each; returns their results in rank order.  Rank 0 runs first.  The
    first exception of any rank is raised here, after every thread has stopped."""
    shared = Lockstep(world, timeout)
    out = [None] * world

    def body(rank):
        try:
            with shared.cond:
                shared.wait(lambda: shared.turn == rank, f"rank {rank}'s first turn")
            out[rank] = fn(LockstepComm(rank, world, shared))
            shared.arrive(rank, "exit", None)
        except _Released:
            pass
        except BaseException as e:          # noqa: B036 — handed to the caller's thread
            shared.fail(rank, e)

    threads = [threading.Thread(target=body, args=(r, ), name=f"rank{r}", daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if shared.error is not None:
        rank, exc = shared.error
        if rank is not None:
            exc.add_note(f"raised on emulated rank {rank} of {world}")
        raise exc
    return out


def test_lockstep_sum_and_max_in_rank_order():
    """float32 (1e8 + 1) − 1e8 is 0 and (1e8 − 1e8) + 1 is 1: the sum is taken in rank order, identically on every rank."""
    vals = [torch.tensor([1e8, 2.0, -3.0]), torch.tensor([1.0, -5.0, 7.0]), torch.tensor([-1e8, 4.0, 0.5])]

    def fn(comm):
        s, m = vals[comm.rank].clone(), vals[comm.rank].clone()
        assert comm.allreduce_sum_(s) is s and comm.allreduce_max_(m) is m
        return s, m
    want_sum = (vals[0] + vals[1]) + vals[2]
    want_max = torch.maximum(torch.maximum(vals[0], vals[1]), vals[2])
    assert want_sum[0].item() == 0.0
    for s, m in run_ranks(3, fn):
        assert torch.equal(s, want_sum) and torch.equal(m, want_max)


def test_lockstep_all_gather_rows_uneven_into_out():
    from dance_b200.parallel import shard_bounds
    bounds = shard_bounds(11, 3)                       # 4 + 4 + 3 rows
    full = torch.arange(33, dtype=torch.float32).view(11, 3)

    def fn(comm):
        a, b = bounds[comm.rank]
        out = torch.full((11, 3), float("nan"))
        got = comm.all_gather_rows(full[a:b].clone(), bounds, out=out)
        return got is out, out, comm.all_gather_rows(full[a:b].clone(), bounds)
    for same, out, fresh in run_ranks(3, fn):
        assert same and torch.equal(out, full) and torch.equal(fresh, full)


def test_lockstep_runs_one_rank_between_collectives():
    log = []

    def fn(comm):
        for step in range(3):
            log.append((step, comm.rank, 0))
            time.sleep(0.005)
            log.append((step, comm.rank, 1))
            comm.barrier()
    run_ranks(3, fn)
    assert log == [(s, r, p) for s in range(3) for r in range(3) for p in (0, 1)]


def test_lockstep_raising_rank_fails_the_caller_promptly():
    """A rank that raises between collectives releases the ranks waiting for it: the caller sees its exception at once, not a
    timeout, and no thread is left behind."""
    def fn(comm):
        t = torch.ones(2)
        comm.allreduce_sum_(t)
        if comm.rank == 1:
            raise ValueError("rank 1 broke")
        comm.allreduce_sum_(t)
    t0 = time.monotonic()
    before = threading.active_count()
    with pytest.raises(ValueError, match="rank 1 broke"):
        run_ranks(3, fn, timeout=30.0)
    assert time.monotonic() - t0 < 10.0
    assert threading.active_count() == before


def test_lockstep_mismatched_collectives_and_timeout_fail():
    def skip(comm):
        if comm.rank != 2:
            comm.barrier()
    with pytest.raises(RuntimeError, match="reached 'exit' where rank 0 reached 'barrier'"):
        run_ranks(3, skip, timeout=30.0)

    def slow(comm):
        if comm.rank == 0:
            time.sleep(1.0)
        comm.barrier()
    with pytest.raises(TimeoutError):
        run_ranks(2, slow, timeout=0.2)


# ---------------------------------------------------------------------------------------------------- shared GPU helpers
PRECISIONS = ["fp32", "tf32x3"]
BATCH, K_NN, EMB = 12800, 15, 16        # bench.py
BT = 128                                # row block of the tensor-core decoder (csrc/gae_tc.cu)

MEASURED = []        # (case, quantity, error, bound): every comparison made, for setting the bounds below


def _check(case, what, err, tol):
    MEASURED.append((case, what, float(err), tol))
    assert err < tol, f"{case}: {what} error {err:.3g} exceeds {tol:.3g}"


def _compare(case, what, got, ref, tol, kind):
    """Norm-wise error; for a matrix also the worst row, and for a gradient matrix the worst column (as in test_gpu_scgnn_step)."""
    _check(case, what, rel_err(got, ref), tol[kind])
    if got.dim() == 2:
        _check(case, what + " rows", row_rel_err(got, ref), tol[kind + "_row"])
        if kind in ("grad", "dact"):
            _check(case, what + " cols", row_rel_err(got.t(), torch.as_tensor(ref).t()), tol[kind + "_col"])


def _row_block(A, r0, r1):
    """Rows [r0, r1) of a CSR as a rank holds them: row pointers from 0, its own column ids (global) and values."""
    from dance_b200 import ops
    e0, e1 = int(A.rowptr[r0]), int(A.rowptr[r1])
    vals = None if A.vals is None else A.vals[e0:e1].contiguous()
    return ops.CSR((A.rowptr[r0:r1 + 1] - e0).contiguous(), A.colidx[e0:e1].contiguous(), vals, (r1 - r0, A.shape[1]))


def _clustered(cuda, n, dim, gen):
    """A clustered, non-negative (ReLU-like) embedding, scaled so that the logits and logvar stay out of saturation."""
    centres = torch.randn(10, dim, device=cuda, generator=gen) * 3
    lab = torch.randint(0, 10, (n, ), device=cuda, generator=gen)
    return ((torch.randn(n, dim, device=cuda, generator=gen) + centres[lab]).abs() * 0.1).contiguous()


def _graph(cuda, x, weighted):
    """The Graph-AE graph of x as bench.py builds it (k = 15, union-symmetrised, unit labels) or with retained weights:
    (adj, adj_t, labels, labels_t, norm, pos_weight)."""
    from dance_b200 import ops
    n = x.shape[0]
    idx, dist = ops.knn(x, K_NN, return_dist=weighted)
    if weighted:
        wg = ops.knn_graph_weighted_build(idx, dist)
        pw, norm = gae_constants(wg.sum_w.item(), n)
        return wg.adj, wg.adj_t, wg.labels, wg.labels_t, norm, pw
    A = ops.knn_graph_build(idx)
    adj_sum = A.nnz - n                                   # bench.py
    return A, A, ops.CSR(A.rowptr, A.colidx, None, A.shape), None, n * n / float((n * n - adj_sum) * 2), float(n * n - adj_sum) / adj_sum


def _dense(L):
    n = L.shape[0]
    return torch.sparse_csr_tensor(L.rowptr.long(), L.colidx.long(), L.vals.double(), (n, n)).to_dense()


# ---------------------------------------------------------------------------------------------------- pair-sharded decoder
# Bounds copied from the existing decoder tests: against float64 the loss 2e-6 and dz 2e-5 (test_decoder_matches_fp64_closed_form,
# test_gae_symmetric_decoder_pair_sharded), against the row-form call the loss 2e-6 and dz 1e-5 (test_gae_symmetric_decoder_pair_sharded).
DEC_TOL = dict(loss=2e-6, dz=2e-5, loss_row_form=2e-6, dz_row_form=1e-5)
GUARD = 64           # NaN rows after each output buffer: a write past the rows a call owns shows up there


@pytest.mark.gpu
@pytest.mark.parametrize("use_pw", [True, False], ids=["posweight", "plain"])
@pytest.mark.parametrize("labels", ["unit", "weighted"])
@pytest.mark.parametrize("n", [100, 129, 4900, 8200])
@pytest.mark.parametrize("d", [8, 16])
def test_pair_sharded_decoder(cuda, d, n, labels, use_pw):
    """gae_loss_grad_sym over every rank of a world of 1, 2, 3 and nsb + 1 ranks (the last one then has no super-block), with the
    J sweeps cut into the automatic, 3 and 7 step ranges.  n = 100: one 128-row block; 129: a 1-row tail block; 4 900: 39 blocks,
    the lone middle super-block; 8 200: 65 blocks.  mu / logvar and dmu / dlogvar are column slices of packed [rows, 2d] buffers,
    as the engine passes them.  The loss shares and the dz_full buffers summed over the ranks match float64 and the row-form call
    (the fp16 triangle); each rank's dz_full is exactly zero outside the rows of its super-blocks and of its labels, and its
    KLD rows equal the row-form call's bit for bit."""
    from dance_b200 import ops
    from dance_b200.parallel import shard_bounds, sym_super_blocks
    gen = torch.Generator(device=cuda).manual_seed(1000 * d + n)
    pts = _clustered(cuda, n, 16, gen)
    _, _, L, Lt, norm, pw = _graph(cuda, pts, labels == "weighted")
    z = (torch.randn(n, d, device=cuda, generator=gen) * d**-0.25).contiguous()     # logits of unit scale
    ml = torch.cat([torch.randn(n, d, device=cuda, generator=gen) * 0.3, torch.randn(n, d, device=cuda, generator=gen) * 0.1], 1)
    mu, lv = ml[:, :d], ml[:, d:]
    md, lvd = mu.double(), lv.double()
    kld = float(-0.5 / (n * n) * (1 + 2 * lvd - md**2 - lvd.exp()**2).sum())
    if labels == "unit":
        dec, ref_dz = R.gae_reference_rows(z, L.rowptr, L.colidx, norm if use_pw else 1.0, pw if use_pw else 1.0,
                                           torch.arange(n, device=cuda))
    else:
        dec, ref_dz = decoder_loss_grad(z, _dense(L), norm, pw, use_pw)
    ref_loss = dec + kld
    nsb, nb = ops.gae_sym_super_blocks(n), -(-n // BT)
    assert nsb == sym_super_blocks(n) == (nb + 1) // 2

    ops.set_path("gae", "tc")            # the row form's tensor-core triangle at every n (auto selects it from n² ≥ 2^22 on)
    try:
        ops.set_tuning("gae_splits", 0)
        dml_row = torch.empty(n, 2 * d, device=cuda)
        loss_row, dz_row, _, _ = ops.gae_loss_grad(z, L, norm, pw, mu, lv, use_pw, dmu=dml_row[:, :d], dlogvar=dml_row[:, d:],
                                                   labels_t=Lt)
        loss_row = loss_row.item()
        case = f"decoder d={d} n={n} {labels} use_pw={use_pw}"
        _check(case + " row form", "loss", abs(loss_row - ref_loss) / abs(ref_loss), DEC_TOL["loss"])
        _check(case + " row form", "dz", rel_err(dz_row, ref_dz), DEC_TOL["dz"])
        for world in sorted({1, 2, 3, nsb + 1}):
            sbs, rows = shard_bounds(nsb, world), shard_bounds(n, world)
            for splits in (0, 3, 7):
                ops.set_tuning("gae_splits", splits)
                at = f"{case} world={world} splits={splits}"
                total, dz_sum = 0.0, torch.zeros(n, d, dtype=torch.float64, device=cuda)
                for r, ((s0, s1), (r0, r1)) in enumerate(zip(sbs, rows)):
                    m = r1 - r0
                    dzf_buf = torch.full((n + GUARD, d), float("nan"), device=cuda)
                    dml_buf = torch.full((m + GUARD, 2 * d), float("nan"), device=cuda)
                    loss_r, dzf, _, _ = ops.gae_loss_grad_sym(z, _row_block(L, r0, r1), norm, pw, s0, s1, ml[r0:r1, :d], ml[r0:r1, d:],
                                                              use_pw, dz_full=dzf_buf[:n], dmu=dml_buf[:m, :d], dlogvar=dml_buf[:m, d:],
                                                              row_begin=r0, n_rows=m,
                                                              labels_t=None if Lt is None else _row_block(Lt, r0, r1))
                    owned = torch.zeros(n, dtype=torch.bool, device=cuda)
                    owned[r0:r1] = True
                    for sb in range(s0, s1):
                        for blk in (sb, nb - 1 - sb):
                            owned[blk * BT:(blk + 1) * BT] = True
                    stray = int((dzf[~owned].view(torch.int32) != 0).any(1).sum())
                    assert stray == 0, f"{at} rank {r}: {stray} rows outside super-blocks [{s0}, {s1}) and rows [{r0}, {r1}) not 0.0"
                    assert bool(dzf_buf[n:].isnan().all()), f"{at} rank {r}: write past row {n} of dz_full"
                    assert torch.equal(dml_buf[:m], dml_row[r0:r1]), f"{at} rank {r}: dmu / dlogvar differ from the row-form call"
                    assert bool(dml_buf[m:].isnan().all()), f"{at} rank {r}: write past row {m} of dmu / dlogvar"
                    total += loss_r.item()
                    dz_sum += dzf.double()
                _check(at, "loss", abs(total - ref_loss) / abs(ref_loss), DEC_TOL["loss"])
                _check(at, "dz", rel_err(dz_sum, ref_dz), DEC_TOL["dz"])
                _check(at, "loss vs row form", abs(total - loss_row) / abs(loss_row), DEC_TOL["loss_row_form"])
                _check(at, "dz vs row form", rel_err(dz_sum, dz_row), DEC_TOL["dz_row_form"])
    finally:
        ops.set_tuning("gae_splits", 0)
        ops.set_path("gae", "auto")


# ---------------------------------------------------------------------------------------------------- sharded Graph-AE step
# The bounds of test_gpu_scgnn_step.py's TOL (4-6x the largest error measured over seeds 0-2 of its cases on an H100 80 GB HBM3 at a
# 400 W power limit).  "act": z / mu / logvar; "dact": their loss gradients; "grad": the weight gradients; "_row" / "_col": the worst
# row / column; "adam_max": the worst element of the optimiser's move, in units of lr.
TOL = {
    "fp32": dict(loss=1e-6, act=3e-7, act_row=3e-6, dact=3e-6, dact_row=2e-5, dact_col=4e-6, grad=3e-5, grad_row=5e-5, grad_col=5e-5,
                 adam=2e-6, adam_max=1e-5),
    "tf32x3": dict(loss=3e-6, act=5e-6, act_row=2e-5, dact=2e-5, dact_row=1e-4, dact_col=3e-5, grad=5e-5, grad_row=1e-4,
                   grad_col=3e-4, adam=2e-6, adam_max=1e-5),
}
# The retained-weights graph (tf32x3), against float64 only: 4-6x the largest error measured over seeds 0-2 on an H100 80 GB HBM3 —
# loss 1.3e-5, z 9.1e-6 (its worst row 1.1e-5), dz / dmu / dlogvar 1.6e-5 (worst row 4.5e-4, worst column 2.0e-5), weight
# gradients 1.7e-5.  The unsharded engine is off from float64 by as much: on the same steps it agrees with the sharded one to 9e-7
# in z and 7e-5 in the worst gradient row (the "vs unsharded" checks, which keep the bounds above).  The other bounds are TOL's.
TOL_WEIGHTED_F64 = dict(TOL["tf32x3"], loss=6e-5, act=5e-5, act_row=6e-5, dact=8e-5, dact_row=2e-3, dact_col=1e-4, grad=8e-5)
STEPS = 3

# (world, precision, decoder branch, n).  "pair": the pair-sharded tensor-core decoder (auto at n² ≥ 2^24); "rows-cuda": the row form
# on the CUDA cores; "rows-tc": the row form on the tensor cores, a row subset (auto at n · n_rows ≥ 2^22); "weighted": the
# pair-sharded decoder on the retained-weights graph (real-valued, asymmetric labels with labels_t, Âᵀ ≠ Â).
GAE_CASES = ([(w, p, "pair", 5003) for w in (2, 3) for p in PRECISIONS] + [(w, p, "rows-cuda", 5003) for w in (2, 3) for p in PRECISIONS]
             + [(2, "tf32x3", "rows-tc", 3001), (3, "tf32x3", "weighted", 5003)])


def graph_ae_sharded_case(cuda, world, precision, branch, n, seed):
    from dance_b200 import ops
    from dance_b200.engine import GraphAEEngine
    from dance_b200.parallel import shard_bounds
    case = f"gae world={world} {precision} {branch} n={n} seed={seed}"
    tol = TOL[precision]
    weighted = branch == "weighted"
    gen = torch.Generator(device=cuda).manual_seed(seed)
    x = _clustered(cuda, n, 128, gen)
    adj, adj_t, labels, labels_t, norm, pw = _graph(cuda, x, weighted)
    eps = torch.randn(n, EMB, device=cuda, generator=gen)
    bounds = shard_bounds(n, world)
    assert len({b - a for a, b in bounds}) == 2                       # uneven shards
    pair = branch in ("pair", "weighted")
    if branch != "rows-cuda":
        assert pair == (n * n >= 1 << 24)
    if branch == "rows-tc":
        assert all(n * (b - a) >= 1 << 22 for a, b in bounds)

    def rank_fn(comm):
        a, b = bounds[comm.rank]
        eng = GraphAEEngine(128, EMB, device=cuda, lr=1e-2, precision=precision, seed=seed)
        eng.set_sharding(comm, bounds)
        loc = [x[a:b], _row_block(adj, a, b), _row_block(labels, a, b), norm, pw, eps[a:b]]
        kw = dict(adj_t=_row_block(adj_t, a, b), labels_t=_row_block(labels_t, a, b)) if weighted else {}
        hist = []
        for _ in range(STEPS):
            flat0 = eng.params.flat.clone()
            z, mu, lv = eng.train_step(*loc, **kw)
            buf = eng._buffers(b - a)
            dzf = eng._bufs.get(("dz_full", n))
            hist.append(dict(flat0=flat0, flat=eng.params.flat.clone(), grad=eng.params.grad.clone(), loss=eng.loss.clone(),
                             z=z.clone(), mu=mu.clone(), lv=lv.clone(), dz=buf["dz"].clone(), dml=buf["dml"].clone(),
                             dz_full=None if dzf is None else dzf.data_ptr(), n_bufs=len(eng._bufs)))
        return hist

    path = "cuda" if branch == "rows-cuda" else "auto"
    ops.set_path("gae", path)
    try:
        hists = run_ranks(world, rank_fn)
        full = GraphAEEngine(128, EMB, device=cuda, lr=1e-2, precision=precision, seed=seed)
        grads = []
        for k in range(STEPS):
            at = f"{case} step {k}"
            hk = [h[k] for h in hists]
            for r, h in enumerate(hk):
                assert (h["dz_full"] is not None) == pair, f"{at} rank {r}: pair-sharded decoder {'not ' if pair else ''}taken"
                assert h["n_bufs"] == hists[r][0]["n_bufs"] and h["dz_full"] == hists[r][0]["dz_full"], f"{at}: buffers not reused"
                for key in ("flat", "grad", "loss"):
                    assert torch.equal(h[key], hk[0][key]), f"{at}: rank {r}'s {key} differs from rank 0's"
            h0 = hk[0]
            cat = {key: torch.cat([h[key] for h in hk]) for key in ("z", "mu", "lv", "dz", "dml")}
            full.params.flat.copy_(h0["flat0"])
            w0 = full.state_dict()
            dec = None
            if weighted:
                dense = _dense(labels)
                dec = lambda zz: decoder_loss_grad(zz, dense, norm, pw)
            ref = R.graph_ae_step(x, adj.rowptr, adj.colidx, adj.vals, labels.rowptr, labels.colidx, norm, pw, w0, eps, decoder=dec)
            # the unsharded engine from the same weights (under auto its full-row decoder is the fp16 triangle, the sharded one
            # the tf32 sweep)
            z_u, mu_u, lv_u = full.train_step(x, adj, labels, norm, pw, eps, adj_t=adj_t if weighted else None, labels_t=labels_t)
            bu = full._buffers(n)
            unsharded = dict(loss=full.loss, z=z_u, mu=mu_u, lv=lv_u, dz=bu["dz"], dml=bu["dml"], grads=full.grads())
            mine = dict(loss=h0["loss"], z=cat["z"], mu=cat["mu"], lv=cat["lv"], dz=cat["dz"], dml=cat["dml"],
                        grads=param_views(full.params, h0["grad"]))
            f64 = dict(loss=ref["loss"], z=ref["z"], mu=ref["mu"], lv=ref["logvar"], dz=ref["dz"], grads=ref["grads"],
                       dml=torch.cat([ref["dmu"], ref["dlogvar"]], 1))
            for vs, other in (("", f64), (" vs unsharded", unsharded)):
                bound = TOL_WEIGHTED_F64 if weighted and vs == "" else tol
                lo = float(other["loss"]) if vs == "" else other["loss"].item()
                _check(at + vs, "loss", abs(mine["loss"].item() - lo) / abs(lo), bound["loss"])
                for name in ("z", "mu", "lv"):
                    _compare(at + vs, name, mine[name], other[name], bound, "act")
                _compare(at + vs, "dz", mine["dz"], other["dz"], bound, "dact")
                _compare(at + vs, "dmu", mine["dml"][:, :EMB], other["dml"][:, :EMB], bound, "dact")
                _compare(at + vs, "dlogvar", mine["dml"][:, EMB:], other["dml"][:, EMB:], bound, "dact")
                g_mine = {"gc1.weight": mine["grads"]["gc1.weight"], "gc2.weight": mine["grads"]["gc23.weight"][:, :EMB],
                          "gc3.weight": mine["grads"]["gc23.weight"][:, EMB:]}
                for key in ("gc1.weight", "gc2.weight", "gc3.weight"):
                    _compare(at + vs, f"d {key}", g_mine[key], other["grads"][key], bound, "grad")
            # the optimiser's move of this step, against float64 Adam over the GPU's own all-reduced gradients so far
            grads.append(h0["grad"])
            want = adam_reference(hists[0][0]["flat0"], grads, full.lr) - adam_reference(hists[0][0]["flat0"], grads[:-1], full.lr)
            moved = h0["flat"].double() - h0["flat0"].double()
            _check(at, "adam update", rel_err(moved, want), tol["adam"])
            _check(at, "adam update max/lr", float((moved - want).abs().max()) / full.lr, tol["adam_max"])
    finally:
        ops.set_path("gae", "auto")


@pytest.mark.gpu
@pytest.mark.parametrize("world,precision,branch,n", GAE_CASES, ids=[f"w{c[0]}-{c[1]}-{c[2]}" for c in GAE_CASES])
def test_sharded_graph_ae_steps(cuda, world, precision, branch, n):
    """Three GraphAEEngine steps per emulated rank under set_sharding (uneven shard_bounds), reusing the persistent buffers and
    the Adam state: after every step the concatenated z / mu / logvar and their gradients, the all-reduced weight gradients and
    loss against float64 from the weights at the start of the step and against the unsharded engine from the same weights, the
    optimiser's move against float64 Adam, and every rank's weights, gradients and loss bit-identical."""
    graph_ae_sharded_case(cuda, world, precision, branch, n, seed=0)


# ---------------------------------------------------------------------------------------------------- data-parallel Feature-AE
# test_gpu_scgnn_step.py's Feature-AE bounds (see its TOL; the gradients are ill-conditioned at initialisation), except fp32's worst
# gradient row, which takes the tf32x3 bound: on the 38 399- and 38 402-row union batches (seed 0) the worst row of d fc3.weight is off
# from float64 by 5.6e-2 in BOTH precisions, while the all-reduced gradient agrees with one single-device step on the same rows to
# 4e-6 in its worst row — the float32 forward's conditioning at three times the 12 800-row batch those bounds were measured at.
FAE_TOL = {
    "fp32": dict(loss=5e-6, grad=3e-4, grad_row=1e-1, grad_col=5e-3, adam=3e-6, adam_max=4e-5),
    "tf32x3": dict(loss=5e-6, grad=5e-4, grad_row=1e-1, grad_col=1e-2, adam=3e-6, adam_max=4e-5),
}
GENES = 2000
# (world, rows): 3 ranks of one batch each (12 800, 12 800, 12 799 rows); 2 ranks of 2 and 1 batches (12 801 + 12 800 rows, the
# second rank takes one idle step); 3 ranks of 2, 2 and 1 batches.
FAE_CASES = [(3, 3 * BATCH - 1), (2, 2 * BATCH + 1), (3, 3 * BATCH + 2)]


def feature_ae_dp_case(cuda, world, n_rows, precision, seed):
    from dance_b200 import ops, synth
    from dance_b200.engine import FeatureAEEngine
    from dance_b200.parallel import batch_schedule, epoch_steps, shard_bounds
    case = f"fae world={world} rows={n_rows} {precision} seed={seed}"
    tol = FAE_TOL[precision]
    X = synth.expression_counts(n_rows, GENES, seed=seed, density=0.10, device=cuda)
    ops.normalize_total_log1p_(X, target_sum=1e4, max_fraction=1.0)
    bounds = shard_bounds(n_rows, world)
    n_steps = epoch_steps(bounds, BATCH)
    scheds = [batch_schedule(b - a, BATCH, n_steps) for a, b in bounds]

    def rank_fn(comm):
        a, b = bounds[comm.rank]
        eng = FeatureAEEngine(GENES, device=cuda, lr=1e-3, precision=precision, seed=seed)
        steps = []

        def hook(g):
            flat0 = eng.params.flat.clone()
            comm.allreduce_sum_(g)
            steps.append((flat0, g.clone()))
        eng.grad_hook = hook
        loss = eng.train_epoch(X[a:b], BATCH, "LTMG", 0.9, None, n_steps=n_steps).clone()
        return dict(steps=steps, loss=loss, flat=eng.params.flat.clone())

    res = run_ranks(world, rank_fn)
    assert any(None in s for s in scheds) or all(len(s) == 1 for s in scheds)
    single = FeatureAEEngine(GENES, device=cuda, lr=1e-3, precision=precision, seed=seed)
    for r, out in enumerate(res):
        assert len(out["steps"]) == n_steps, f"{case}: rank {r} took {len(out['steps'])} steps of {n_steps}"
        assert torch.equal(out["flat"], res[0]["flat"]), f"{case}: rank {r}'s weights differ from rank 0's"
        for s in range(n_steps):
            assert torch.equal(out["steps"][s][1], res[0]["steps"][s][1]), f"{case}: rank {r}'s step-{s} gradient differs"
    for s in range(n_steps):
        flat0, g = res[0]["steps"][s]
        rows = torch.cat([torch.arange(a + sc[s][0], a + sc[s][1], device=cuda) for (a, _), sc in zip(bounds, scheds) if sc[s] is not None])
        ref = R.feature_ae_step(X[rows], param_views(single.params, flat0), "LTMG", 0.9, None)
        gv = param_views(single.params, g)
        for k in R.FEATURE_AE_PARAMS:
            _compare(f"{case} step {s}", f"d {k}", gv[k], ref["grads"][k], tol, "grad")
    ref_flat = adam_reference(res[0]["steps"][0][0], [g for _, g in res[0]["steps"]], single.lr)
    moved, want = res[0]["flat"].double() - res[0]["steps"][0][0].double(), ref_flat - res[0]["steps"][0][0].double()
    _check(case, "adam update", rel_err(moved, want), tol["adam"])
    _check(case, "adam update max/lr", float((moved - want).abs().max()) / single.lr, tol["adam_max"])
    if n_steps == 1:
        # one batch per rank: the all-reduced gradient is the gradient of one step on the concatenated batch (sum-reduced loss)
        seen = []
        single.grad_hook = lambda g: seen.append(g.clone())
        single.loss_acc.zero_()
        single.train_step(X, None, 0.9, "LTMG")
        total = sum(out["loss"].item() for out in res)
        _check(case, "loss vs one device", abs(total - single.loss_acc.item()) / abs(single.loss_acc.item()), tol["loss"])
        g1, gs = param_views(single.params, res[0]["steps"][0][1]), param_views(single.params, seen[0])
        for k in R.FEATURE_AE_PARAMS:
            _compare(f"{case} vs one device", f"d {k}", g1[k], gs[k], tol, "grad")


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("world,n_rows", FAE_CASES, ids=[f"w{c[0]}-rows{c[1]}" for c in FAE_CASES])
def test_data_parallel_feature_ae_epoch(cuda, world, n_rows, precision):
    """train_epoch per emulated rank with grad_hook = all-reduce and n_steps = epoch_steps: every rank takes every step (idle
    ones included), each step's reduced gradient matches float64 on the union of the ranks' batches of that step, the weights
    end bit-identical on every rank, and with one batch per rank the reduced gradient and summed loss match one step on the
    concatenated batch."""
    feature_ae_dp_case(cuda, world, n_rows, precision, seed=0)
