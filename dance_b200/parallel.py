"""Cell-sharded data parallelism over the GPUs of one box: one process per GPU,
``torch.distributed`` (NCCL over NVLink/NVSwitch on GPUs, gloo in the CPU tests) for the
plumbing.  The reference has no distributed path at all (SURVEY §2.2) — this is new.

Decomposition (SURVEY §8e):
  * cells (graph rows) are split into contiguous shards, one per rank;
  * Feature-AE: pure sample parallelism; ONE all-reduce(sum) of the flat gradient bucket per
    optimiser step (``FlatParams.grad`` is a single contiguous buffer);
  * Graph-AE (GCN): each rank owns its rows of Â (CSR rows local, column ids global); the narrow
    dense operand (N×32) is all-gathered before every SpMM, the decoder all-gathers z (N×16);
    weight gradients are all-reduced.  Â is symmetric, so the backward SpMM Âᵀ·dY restricted to
    the local rows is again ``Â_local · all_gather(dY)``.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n: int, world: int) -> List[Tuple[int, int]]:
    """Contiguous, balanced row ranges (first ``n % world`` shards get one extra row)."""
    base, rem = divmod(n, world)
    out, start = [], 0
    for r in range(world):
        size = base + (1 if r < rem else 0)
        out.append((start, start + size))
        start += size
    return out


def epoch_steps(bounds: List[Tuple[int, int]], batch_size: int) -> int:
    """Optimiser steps per data-parallel epoch = mini-batches of the LARGEST shard.  Every rank must issue this many gradient
    all-reduces per epoch: with uneven shards (e.g. 100 001 cells on 2 ranks, batch 12 500 → 5 and 4 local batches) a rank that
    stopped after its own batches would leave the others waiting in the collective."""
    return max((b - a + batch_size - 1) // batch_size for a, b in bounds)


def batch_schedule(n_local: int, batch_size: int, n_steps: Optional[int] = None) -> List[Optional[Tuple[int, int]]]:
    """Row ranges of one epoch over ``n_local`` rows; padded with ``None`` (= contribute a zero gradient) up to ``n_steps``."""
    sched: List[Optional[Tuple[int, int]]] = [(b0, min(n_local, b0 + batch_size)) for b0 in range(0, n_local, batch_size)]
    if n_steps is not None:
        if n_steps < len(sched):
            raise ValueError(f"n_steps={n_steps} is smaller than this rank's {len(sched)} local batches")
        sched += [None] * (n_steps - len(sched))
    return sched


def _sym_blocks(n_blocks: int, super_block: int) -> List[int]:
    return sorted({super_block, n_blocks - 1 - super_block})


def sym_schedule(n_blocks: int, super_block: int) -> List[Tuple[int, int]]:
    """Logit tiles (I, J) of 128-row blocks that super-block ``super_block`` of the pair-sharded decoder evaluates — the host-side
    statement of the work units of ``gae_allpairs_tc_kernel`` (csrc/gae_tc.cu), used to shard the decoder over ranks and to test it.

    A super-block is the row blocks sb and nb−1−sb (one block when they coincide); each row block sweeps every J.  Together the
    super-blocks cover every ordered pair of blocks exactly once, two row blocks of work each (one for a lone middle block)."""
    return [(I, J) for I in _sym_blocks(n_blocks, super_block) for J in range(n_blocks)]


def sym_steps(n_blocks: int, super_block: int) -> List[List[Tuple[int, int]]]:
    """The same tiles grouped by J-step: step s stages Z_J for J = s and evaluates it against the super-block's row blocks (in the
    kernel each row block is its own CTA; both walk the same steps)."""
    return [[(I, J) for I in _sym_blocks(n_blocks, super_block)] for J in range(n_blocks)]


def sym_step_range(n_steps: int, part: int, splits: int) -> Tuple[int, int]:
    """Steps [s0, s1) of a J sweep that CTA ``part`` of ``splits`` runs (``gae_allpairs_tc_kernel``: ⌈n_steps / splits⌉ steps per
    part, trailing parts may be empty): the decoder cuts sweeps into step ranges so that a grid fills a wave of SMs."""
    per = -(-n_steps // splits)
    return min(n_steps, part * per), min(n_steps, (part + 1) * per)


def spmm_stream_partition(rowptr, n_warps: int) -> List[Tuple[int, int]]:
    """Row ranges [R0, R1) the warps of the nnz-stream aggregate own (csrc/spmm_stream.cu): warp w takes the rows whose key
    rowptr[r] + r lies in [w·T/W, (w+1)·T/W), T = nnz + n_rows — balanced by non-zeros AND rows, so empty rows and hub rows cost
    what they cost.  Host restatement for tests; the kernel finds the boundaries with a warp-cooperative 32-ary search."""
    import numpy as np
    rp = np.asarray(rowptr, dtype=np.int64)
    n_rows = len(rp) - 1
    key = rp + np.arange(n_rows + 1)
    total = int(key[-1])
    out = []
    for w in range(n_warps):
        r0 = 0 if w == 0 else int(np.searchsorted(key, w * total // n_warps, side="left"))
        r1 = n_rows if w == n_warps - 1 else int(np.searchsorted(key, (w + 1) * total // n_warps, side="left"))
        out.append((r0, max(r0, r1)))
    return out


def sym_super_blocks(n: int, block: int = 128) -> int:
    return ((n + block - 1) // block + 1) // 2


class Comm:
    """Thin wrapper over a torch.distributed process group (or a no-op for world size 1)."""

    def __init__(self, group=None):
        self.enabled = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
        self.group = group
        self.rank = dist.get_rank(group) if self.enabled else 0
        self.world = dist.get_world_size(group) if self.enabled else 1

    @classmethod
    def from_env(cls, backend: Optional[str] = None) -> "Comm":
        """Initialise from the torchrun environment (RANK / WORLD_SIZE / MASTER_*)."""
        world = int(os.environ.get("WORLD_SIZE", "1"))
        if world > 1 and not dist.is_initialized():
            if backend is None:
                backend = "nccl" if torch.cuda.is_available() else "gloo"
            if backend == "nccl":
                torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
            dist.init_process_group(backend=backend)
        return cls()

    def allreduce_sum_(self, t: torch.Tensor) -> torch.Tensor:
        if self.enabled:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t

    def allreduce_max_(self, t: torch.Tensor) -> torch.Tensor:
        if self.enabled:
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        return t

    def all_gather_rows(self, local: torch.Tensor, bounds: List[Tuple[int, int]], out: Optional[torch.Tensor] = None):
        """Concatenate the ranks' row blocks [n_r, F] → [N, F] (row counts may differ by one)."""
        if not self.enabled:
            return local
        n_total = bounds[-1][1]
        F = local.shape[1]
        if out is None:
            out = torch.empty((n_total, F), dtype=local.dtype, device=local.device)
        local = local.contiguous()
        sizes = [b - a for a, b in bounds]
        if len(set(sizes)) == 1:
            dist.all_gather_into_tensor(out, local, group=self.group)
        else:
            # collectives need equal-sized contributions: pad every shard to the largest one, then compact
            mx = max(sizes)
            pad = torch.zeros((mx, F), dtype=local.dtype, device=local.device)
            pad[:local.shape[0]] = local
            buf = torch.empty((self.world * mx, F), dtype=local.dtype, device=local.device)
            dist.all_gather_into_tensor(buf, pad, group=self.group)
            for r, (a, b) in enumerate(bounds):
                out[a:b] = buf[r * mx:r * mx + (b - a)]
        return out

    def barrier(self):
        if self.enabled:
            dist.barrier(group=self.group)


class NativeComm:
    """The same collectives through the C-ABI's own NCCL communicator (``b2_comm_*``, csrc/comm.cu) — what a non-Python binder
    uses.  Drop-in for :class:`Comm` in the engines: ``allreduce_sum_`` / ``all_gather_rows`` / ``allreduce_max_`` / ``barrier``.
    The 128-byte NCCL id is created on rank 0 and handed to the other ranks through ``exchange`` (any callable that broadcasts
    bytes from rank 0; by default the torch.distributed process group that torchrun already set up — only for this bootstrap)."""

    def __init__(self, rank: int, world: int, exchange=None):
        import ctypes as C
        from . import ops
        self._ops, self._C = ops, C
        self.rank, self.world, self.enabled = rank, world, world > 1
        self._handle = C.c_void_p()
        lib = ops.lib()
        if not lib.b2_comm_available():
            raise RuntimeError("NativeComm: libnccl.so.2 could not be loaded")
        buf = (C.c_char * 128)()
        if rank == 0:
            ops.check(lib.b2_comm_unique_id(buf), "b2_comm_unique_id")
        raw = bytes(buf)
        if world > 1:
            if exchange is None:
                def exchange(b):
                    t = torch.frombuffer(bytearray(b), dtype=torch.uint8).clone()
                    if dist.get_backend() == "nccl":
                        t = t.cuda()
                    dist.broadcast(t, src=0)
                    return bytes(t.cpu().numpy().tobytes())
            raw = exchange(raw)
        idbuf = (C.c_char * 128).from_buffer_copy(raw)
        ops.check(lib.b2_comm_init_rank(C.byref(self._handle), idbuf, world, rank), "b2_comm_init_rank")

    def close(self):
        if self._handle:
            self._ops.lib().b2_comm_destroy(self._handle)
            self._handle = self._C.c_void_p()

    def allreduce_sum_(self, t: torch.Tensor) -> torch.Tensor:
        if self.enabled:
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError("NativeComm.allreduce_sum_: contiguous float32 tensor required")
            self._ops.check(self._ops.lib().b2_allreduce_sum_f32(self._handle, t.data_ptr(), t.numel(), self._ops._stream()), "b2_allreduce_sum_f32")
        return t

    def allreduce_max_(self, t: torch.Tensor) -> torch.Tensor:
        """max over ranks of a small non-negative vector, via gather + local max (timing bookkeeping only)."""
        if self.enabled:
            full = torch.empty(self.world * t.numel(), dtype=torch.float32, device=t.device)
            self._ops.check(self._ops.lib().b2_allgather_f32(self._handle, t.contiguous().data_ptr(), full.data_ptr(), t.numel(),
                                                             self._ops._stream()), "b2_allgather_f32")
            t.copy_(full.view(self.world, -1).max(0).values.view_as(t))
        return t

    def all_gather_rows(self, local: torch.Tensor, bounds, out: Optional[torch.Tensor] = None):
        if not self.enabled:
            return local
        n_total, F = bounds[-1][1], local.shape[1]
        if out is None:
            out = torch.empty((n_total, F), dtype=local.dtype, device=local.device)
        sizes = [b - a for a, b in bounds]
        mx = max(sizes)
        lib = self._ops.lib()
        if len(set(sizes)) == 1:
            self._ops.check(lib.b2_allgather_f32(self._handle, local.contiguous().data_ptr(), out.data_ptr(), mx * F, self._ops._stream()),
                            "b2_allgather_f32")
            return out
        pad = torch.zeros((mx, F), dtype=local.dtype, device=local.device)
        pad[:local.shape[0]] = local
        buf = torch.empty((self.world * mx, F), dtype=local.dtype, device=local.device)
        self._ops.check(lib.b2_allgather_f32(self._handle, pad.data_ptr(), buf.data_ptr(), mx * F, self._ops._stream()), "b2_allgather_f32")
        for r, (a, b) in enumerate(bounds):
            out[a:b] = buf[r * mx:r * mx + (b - a)]
        return out

    def barrier(self):
        if self.enabled:
            t = torch.zeros(1, dtype=torch.float32, device="cuda")
            self.allreduce_sum_(t)
            torch.cuda.current_stream().synchronize()
