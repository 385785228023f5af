"""1-D row-block data parallelism, one process per GPU (torch.distributed: nccl on GPUs,
gloo in CPU tests).

The reference has exactly one strategy (SURVEY §2b): Legate tiles the rows of A equally over
the processors (``align(y, pos)``, reference legate_sparse/csr.py:587-591), each GPU
gets the contiguous crd/vals slice of its rows and the x window it needs; the only NCCL call
upstream is a 1-element all-gather of per-GPU nnz (spgemm_csr_csr_csr.cu:43-62).

Here: every rank runs the same script (SPMD).  A matrix is split into row blocks
``bounds[r] .. bounds[r+1]``; x is replicated; each rank computes its block of y with the
local sm_90a kernel and — when a replicated result is needed (CG/GMRES) — the blocks are
all-gathered (NCCL over NVLink / NVSwitch).  Dense-vector reductions are done on the local
block and all-reduced.
"""
from __future__ import annotations

import os
from typing import Sequence

import numpy as np
import torch
import torch.distributed as td


def is_initialized() -> bool:
    return td.is_available() and td.is_initialized()


def world_size() -> int:
    return td.get_world_size() if is_initialized() else 1


def rank() -> int:
    return td.get_rank() if is_initialized() else 0


def init(backend: str | None = None) -> None:
    """Join the process group described by the torchrun environment (RANK/WORLD_SIZE/
    MASTER_ADDR/MASTER_PORT/LOCAL_RANK).  No-op for a single process."""
    if is_initialized() or int(os.environ.get("WORLD_SIZE", "1")) <= 1:
        return
    use_cuda = torch.cuda.is_available()
    if backend is None:
        backend = "nccl" if use_cuda else "gloo"
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    if use_cuda:
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        td.init_process_group(backend=backend, device_id=torch.device("cuda", local))
    else:
        td.init_process_group(backend=backend)


def shutdown() -> None:
    if is_initialized():
        td.destroy_process_group()


# ---------------------------------------------------------------------------- partitions
def row_block_bounds(nrows: int, nparts: int) -> np.ndarray:
    """Equal-row tiling (what Legate's ``align(y, pos)`` produces): block = ceil(n/G)."""
    nparts = max(int(nparts), 1)
    block = -(-int(nrows) // nparts) if nrows > 0 else 0
    b = np.minimum(np.arange(nparts + 1, dtype=np.int64) * block, nrows)
    return b.astype(np.int64)


def nnz_balanced_bounds(indptr, nparts: int) -> np.ndarray:
    """Row boundaries with ~equal nnz per part (binary search on indptr) — for skewed
    (power-law) matrices where equal rows starve some GPUs (SURVEY §8e)."""
    ip = indptr.detach().cpu().numpy() if isinstance(indptr, torch.Tensor) else np.asarray(indptr)
    nrows = ip.shape[0] - 1
    nnz = int(ip[-1])
    targets = (np.arange(1, nparts, dtype=np.float64) * (nnz / float(nparts))).astype(np.int64)
    cuts = np.searchsorted(ip, targets, side="left").astype(np.int64)
    b = np.concatenate([[0], np.clip(cuts, 0, nrows), [nrows]]).astype(np.int64)
    return np.maximum.accumulate(b)


def weight_balanced_bounds(weights, nparts: int) -> np.ndarray:
    """Row boundaries with ~equal total weight per part (weights: per-row work, e.g. the number of
    intermediate products of an SpGEMM row) — the generalisation of nnz_balanced_bounds."""
    w = weights.detach().to(torch.float64).cpu().numpy() if isinstance(weights, torch.Tensor) else np.asarray(weights, dtype=np.float64)
    nrows = w.shape[0]
    cum = np.concatenate([[0.0], np.cumsum(w)])
    targets = np.arange(1, nparts, dtype=np.float64) * (cum[-1] / float(nparts))
    cuts = np.searchsorted(cum, targets, side="left").astype(np.int64)
    b = np.concatenate([[0], np.clip(cuts, 0, nrows), [nrows]]).astype(np.int64)
    return np.maximum.accumulate(b)


# ---------------------------------------------------------------------------- collectives
def allgather_rows(local: torch.Tensor, bounds: Sequence[int]) -> torch.Tensor:
    """Gather the row blocks ``local`` (this rank owns rows bounds[rank]:bounds[rank+1])
    into the full replicated vector.  Blocks may be ragged; they are padded to the largest
    block so that a single all_gather_into_tensor (one NCCL all-gather) suffices."""
    G = world_size()
    n = int(bounds[-1])
    if G == 1:
        return local
    sizes = [int(bounds[i + 1] - bounds[i]) for i in range(G)]
    blk = max(sizes) if sizes else 0
    if blk == 0:
        return local.new_zeros(0)
    send = local
    if local.numel() != blk:
        send = local.new_zeros(blk)
        send[: local.numel()] = local
    recv = local.new_empty(G * blk)
    td.all_gather_into_tensor(recv, send.contiguous())
    if all(s == blk for s in sizes):
        return recv[:n] if G * blk != n else recv
    out = local.new_empty(n)
    for i in range(G):
        if sizes[i]:
            out[int(bounds[i]) : int(bounds[i + 1])] = recv[i * blk : i * blk + sizes[i]]
    return out


def allgather_into(full: torch.Tensor, bounds: Sequence[int]) -> torch.Tensor:
    """In-place variant: ``full`` already holds this rank's block at its row offset; after the
    call every rank holds every block.  Equal-size fast path needs no staging copy."""
    G = world_size()
    if G == 1:
        return full
    r = rank()
    sizes = [int(bounds[i + 1] - bounds[i]) for i in range(G)]
    blk = max(sizes)
    n = int(bounds[-1])
    if all(int(bounds[i]) == i * blk for i in range(G)) and G * blk == n:
        td.all_gather_into_tensor(full, full[r * blk : (r + 1) * blk])
        return full
    gathered = allgather_rows(full[int(bounds[r]) : int(bounds[r + 1])], bounds)
    full.copy_(gathered)
    return full


def allreduce_sum_(t: torch.Tensor) -> torch.Tensor:
    if world_size() > 1:
        td.all_reduce(t, op=td.ReduceOp.SUM)
    return t


def allgather_i64(value: int, device=None) -> np.ndarray:
    """All-gather of one int64 per rank (the reference's ncclAllGather of per-rank nnz,
    spgemm_csr_csr_csr.cu:43-62); returns the host array of the G values."""
    G = world_size()
    if G == 1:
        return np.array([int(value)], dtype=np.int64)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    cnt = torch.tensor([int(value)], dtype=torch.int64, device=device)
    cnts = torch.empty(G, dtype=torch.int64, device=device)
    td.all_gather_into_tensor(cnts, cnt)
    return cnts.cpu().numpy().astype(np.int64)


def allgather_varlen(local: torch.Tensor) -> tuple[torch.Tensor, np.ndarray]:
    """all-gather(v) of 1-D tensors of different lengths: returns (concatenation in rank
    order, per-rank counts).  Used for the SpGEMM C blocks; the count exchange is the
    analogue of the reference's ncclAllGather of per-rank nnz (spgemm_csr_csr_csr.cu:43-62)."""
    G = world_size()
    if G == 1:
        return local, np.array([local.numel()], dtype=np.int64)
    cnt = torch.tensor([local.numel()], dtype=torch.int64, device=local.device)
    cnts = torch.empty(G, dtype=torch.int64, device=local.device)
    td.all_gather_into_tensor(cnts, cnt)
    counts = cnts.cpu().numpy()
    blk = int(counts.max())
    send = local.new_zeros(blk)
    send[: local.numel()] = local
    recv = local.new_empty(G * blk)
    td.all_gather_into_tensor(recv, send)
    parts = [recv[i * blk : i * blk + int(counts[i])] for i in range(G)]
    return torch.cat(parts), counts


# ---------------------------------------------------------------------------- symmetric (peer) memory
class SymmVector:
    """A replicated vector whose copy on EVERY rank is mapped into every other rank's address
    space (torch symmetric memory: CUDA IPC / fabric handles over NVLink).  Kernels that produce
    a row block store it straight into all copies (b2s_spmv_csr_bcast / b2s_cg_pupdate_bcast):
    the all-gather is fused into the producing kernel; `barrier()` is the only collective."""

    def __init__(self, n: int, dtype: torch.dtype):
        import torch.distributed._symmetric_memory as symm

        dev = torch.device("cuda", torch.cuda.current_device())
        self.t = symm.empty(int(n), dtype=dtype, device=dev)
        self.h = symm.rendezvous(self.t, td.group.WORLD)
        self.ptrs = [int(q) for q in self.h.buffer_ptrs]
        self.itemsize = self.t.element_size()
        self.mc = 0
        try:  # NVSwitch multicast (NVLS) address of the same buffer on every rank, when supported
            if os.environ.get("LEGATE_SPARSE_MULTICAST", "0") not in ("0", "") and bool(self.h.has_multicast_support):
                self.mc = int(self.h.multicast_ptr)
        except Exception:
            self.mc = 0

    def peer_ptrs(self, row_offset: int):
        """destinations for a kernel's broadcast stores: ("mc", address) when NVSwitch multicast
        is available (one store, replicated by the switch), else the unicast peer pointers"""
        me = rank()
        off = int(row_offset) * self.itemsize
        if self.mc:
            return ("mc", self.mc + off)
        return [q + off for g, q in enumerate(self.ptrs) if g != me]

    def barrier(self):
        self.h.barrier(channel=0)


_symm_cache: dict = {}
_symm_broken = False


def symm_vector(n: int, dtype: torch.dtype, tag: str = "y"):
    """Cached symmetric vector (collective on first use: all ranks must call in the same order).
    Returns None when peer memory is unavailable → callers fall back to NCCL all-gather."""
    global _symm_broken
    if _symm_broken or world_size() == 1 or world_size() > 8 or not torch.cuda.is_available():
        return None
    if os.environ.get("LEGATE_SPARSE_NO_SYMM", "0") not in ("0", ""):
        return None
    key = (int(n), dtype, tag)
    v = _symm_cache.get(key)
    if v is None:
        ok = torch.ones(1, dtype=torch.int32, device="cuda")
        try:
            v = SymmVector(n, dtype)
        except Exception as e:  # pragma: no cover - depends on the box
            import warnings

            warnings.warn(f"symmetric memory unavailable ({e}); using NCCL all-gather")
            ok.zero_()
            v = None
        td.all_reduce(ok, op=td.ReduceOp.MIN)   # all ranks agree on the path
        if int(ok.item()) == 0:
            _symm_broken = True
            return None
        _symm_cache[key] = v
    return v


_symm_turn: dict = {}


def symm_vector_alternating(n: int, dtype: torch.dtype, tag: str):
    """Two symmetric vectors per (n, dtype, tag) handed out in turn (collective, same order on every
    rank).  A producer that closes every use with `barrier()` may then write the returned buffer
    without an opening barrier: before anyone writes buffer b again, every rank has passed the
    closing barrier of the call in between, which is stream-ordered after its reads of b."""
    key = (int(n), dtype, tag)
    turn = 1 - _symm_turn.get(key, 1)
    _symm_turn[key] = turn
    return symm_vector(n, dtype, f"{tag}{turn}")


class ScalarBoard:
    """Peer-mapped boards for in-kernel all-reduces of device scalars (b2s_allreduce_board): one
    small symmetric buffer per rank + local sequence counters.  Replaces NCCL all-reduce /
    symmetric-memory barriers inside the CG iteration (one one-warp kernel per exchange)."""

    def __init__(self):
        import ctypes

        import torch.distributed._symmetric_memory as symm

        from . import _native as N

        dev = torch.device("cuda", torch.cuda.current_device())
        nbytes = int(N.load().b2s_board_bytes())
        self.t = symm.empty(nbytes, dtype=torch.uint8, device=dev)
        self.t.zero_()
        self.h = symm.rendezvous(self.t, td.group.WORLD)
        self.ptrs = [int(q) for q in self.h.buffer_ptrs]
        self.arr = (ctypes.c_void_p * len(self.ptrs))(*[ctypes.c_void_p(q) for q in self.ptrs])
        self.seq = torch.zeros(8, dtype=torch.int64, device=dev)
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)
        self.rank, self.nranks = rank(), world_size()
        torch.cuda.synchronize()
        self.h.barrier(channel=0)        # every board is zeroed before anyone writes a slot
        torch.cuda.synchronize()

    def allreduce(self, scalar: torch.Tensor, channel: int, cur_out=None, prev_out=None):
        """scalar[0] <- sum over ranks (in rank order); optionally prev_out[0] <- cur_out[0],
        cur_out[0] <- sum.  Stream-ordered, capturable in a CUDA graph."""
        import ctypes

        from . import _native as N
        from ._device import np_dtype_of, ptr, stream_ptr, vt_enum

        N.check(
            N.load().b2s_allreduce_board(
                vt_enum(np_dtype_of(scalar)), ptr(scalar), ctypes.cast(self.arr, ctypes.c_void_p), rank(),
                world_size(), int(channel), ptr(self.seq), ptr(cur_out), ptr(prev_out), ptr(self.err), stream_ptr()),
            "allreduce_board")
        return scalar

    def check(self):
        if int(self.err.item()) != 0:
            raise RuntimeError("in-kernel all-reduce timed out waiting for a peer rank")


_board = None
_board_broken = False


def scalar_board():
    """Cached ScalarBoard (collective on first use), or None when peer memory is unavailable /
    LEGATE_SPARSE_NO_BOARD is set → callers fall back to NCCL all-reduce."""
    global _board, _board_broken
    if _board is not None:
        return _board
    if _board_broken or world_size() == 1 or world_size() > 8 or not torch.cuda.is_available():
        return None
    if os.environ.get("LEGATE_SPARSE_NO_BOARD", "0") not in ("0", "") or os.environ.get("LEGATE_SPARSE_NO_SYMM", "0") not in ("0", ""):
        return None
    ok = torch.ones(1, dtype=torch.int32, device="cuda")
    b = None
    try:
        b = ScalarBoard()
    except Exception as e:  # pragma: no cover - depends on the box
        import warnings

        warnings.warn(f"scalar board unavailable ({e}); using NCCL all-reduce")
        ok.zero_()
    td.all_reduce(ok, op=td.ReduceOp.MIN)
    if int(ok.item()) == 0:
        _board_broken = True
        return None
    _board = b
    return _board


_user_symm: dict = {}


def replicated_empty(n: int, dtype: torch.dtype):
    """A length-n device vector in SYMMETRIC memory (mapped into every rank) for use as the ``out=`` of
    ``A.dot(x, out=...)`` with several ranks: the SpMV kernel then stores its rows straight into
    every rank's copy of THIS buffer and no staging copy is made (collective: every rank must call
    it in the same order).  Falls back to a plain device tensor when peer memory is unavailable."""
    if world_size() == 1 or not torch.cuda.is_available() or _symm_broken:
        return torch.empty(int(n), dtype=dtype, device="cuda" if torch.cuda.is_available() else "cpu")
    key = ("user", len(_user_symm))
    sv = symm_vector(int(n), dtype, f"user{len(_user_symm)}")
    if sv is None:
        return torch.empty(int(n), dtype=dtype, device="cuda")
    _user_symm[sv.t.data_ptr()] = sv
    return sv.t


def symm_of(t):
    """The SymmVector behind a tensor handed out by replicated_empty (else None)."""
    if isinstance(t, torch.Tensor) and t.is_cuda:
        sv = _user_symm.get(t.data_ptr())
        if sv is not None and sv.t.numel() == t.numel() and sv.t.dtype == t.dtype:
            return sv
    return None
