"""Device-buffer plumbing: torch tensors as HBM buffers + typed wrappers over the C ABI.

PyTorch is used ONLY for device memory, streams and (in dist.py) torch.distributed;
all arithmetic on the hot path is done by libb200sparse kernels.
"""
from __future__ import annotations

import ctypes
from ctypes import c_int64, c_void_p, byref

import numpy as np
import torch

from . import _native as N

_NP2ENUM = {
    np.dtype(np.float32): N.B2S_F32,
    np.dtype(np.float64): N.B2S_F64,
    np.dtype(np.complex64): N.B2S_C64,
    np.dtype(np.complex128): N.B2S_C128,
}
_NP2TORCH = {
    np.dtype(np.float32): torch.float32,
    np.dtype(np.float64): torch.float64,
    np.dtype(np.complex64): torch.complex64,
    np.dtype(np.complex128): torch.complex128,
    np.dtype(np.int32): torch.int32,
    np.dtype(np.int64): torch.int64,
    np.dtype(np.bool_): torch.bool,
    np.dtype(np.uint8): torch.uint8,
    np.dtype(np.int8): torch.int8,
    np.dtype(np.int16): torch.int16,
    np.dtype(np.float16): torch.float16,
}
_TORCH2NP = {v: k for k, v in _NP2TORCH.items()}


def np_dtype_of(t) -> np.dtype:
    if isinstance(t, torch.Tensor):
        return _TORCH2NP[t.dtype]
    return np.dtype(t.dtype)


def torch_dtype(dt) -> torch.dtype:
    return _NP2TORCH[np.dtype(dt)]


def vt_enum(dt) -> int:
    try:
        return _NP2ENUM[np.dtype(dt)]
    except KeyError:
        raise NotImplementedError(f"dtype {dt} is not supported by the native kernels")


def real_dtype(dt) -> np.dtype:
    dt = np.dtype(dt)
    return np.dtype(np.float32) if dt in (np.dtype(np.float32), np.dtype(np.complex64)) else np.dtype(np.float64)


_checked = False


def require_cuda() -> torch.device:
    """Fail loudly when there is no GPU or no native library (never fall back to CPU)."""
    global _checked
    if not _checked:
        N.load()
        if not torch.cuda.is_available():
            raise RuntimeError(
                "legate_sparse (b200): no CUDA device is available; the sm_90a kernels are the "
                "only compute path (there is no CPU fallback)."
            )
        _checked = True
    return torch.device("cuda", torch.cuda.current_device())


def stream_ptr() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t) -> c_void_p:
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def is_device_tensor(x) -> bool:
    return isinstance(x, torch.Tensor) and x.is_cuda


def to_device(x, dtype=None, copy=False) -> torch.Tensor:
    """numpy / torch(cpu|cuda) → contiguous CUDA tensor (optionally cast)."""
    dev = require_cuda()
    if isinstance(x, torch.Tensor):
        t = x
        if not t.is_cuda:
            t = t.to(dev, non_blocking=True)
            copy = False
    else:
        a = np.ascontiguousarray(x)
        t = torch.from_numpy(a).to(dev, non_blocking=False)
        copy = False
    if dtype is not None and t.dtype != torch_dtype(dtype):
        t = t.to(torch_dtype(dtype))
        copy = False
    if not t.is_contiguous():
        t = t.contiguous()
        copy = False
    if copy:
        t = t.clone()
    return t


def to_host(t) -> np.ndarray:
    if isinstance(t, torch.Tensor):
        return t.detach().cpu().numpy()
    return np.asarray(t)


def empty(n, dtype) -> torch.Tensor:
    return torch.empty(int(n), dtype=torch_dtype(dtype), device=require_cuda())


def zeros(n, dtype) -> torch.Tensor:
    return torch.zeros(int(n), dtype=torch_dtype(dtype), device=require_cuda())


# ------------------------------------------------------------------ reductions workspace
_red_ws = {}


def new_reduce_ws() -> torch.Tensor:
    """A reduction workspace owned by the caller (e.g. one per captured CUDA graph)."""
    return torch.zeros(int(N.load().b2s_reduce_workspace_bytes()), dtype=torch.uint8, device=require_cuda())


def reduce_ws() -> torch.Tensor:
    dev = require_cuda()
    key = (dev.index, torch.cuda.current_stream().cuda_stream)
    ws = _red_ws.get(key)
    if ws is None:
        nbytes = int(N.load().b2s_reduce_workspace_bytes())
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        _red_ws[key] = ws
    return ws


# ------------------------------------------------------------------ SpMV plan
class SpmvPlan:
    """Owner of a native b2s_spmv_plan + its device workspace (cached per matrix)."""

    def __init__(self, itype, nrows, ncols, nnz, indptr, indices):
        lib = N.load()
        nbytes = int(lib.b2s_spmv_plan_workspace_bytes(nrows, nnz))
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=indptr.device)
        self.handle = c_void_p(0)
        N.check(
            lib.b2s_spmv_plan_create(
                itype, nrows, ncols, nnz, ptr(indptr), ptr(indices), ptr(self.ws), nbytes, stream_ptr(),
                byref(self.handle),
            ),
            "spmv_plan_create",
        )
        self._lib = lib

    def info(self):
        a, b, c = c_int64(0), c_int64(0), c_int64(0)
        N.check(self._lib.b2s_spmv_plan_info(self.handle, byref(a), byref(b), byref(c)), "spmv_plan_info")
        return {"ntiles": a.value, "tile_nnz": b.value, "window_tiles": c.value}

    def __del__(self):
        try:
            if self.handle:
                self._lib.b2s_spmv_plan_destroy(self.handle)
                self.handle = c_void_p(0)
        except Exception:
            pass


_side = {}


def _side_stream():
    """one extra stream per device for copies that overlap kernels"""
    d = torch.cuda.current_device()
    if d not in _side:
        _side[d] = torch.cuda.Stream(device=d)
    return _side[d]


class ColBlock:
    """Owner of a native b2s_colblock (column-blocked copy of a row block) + its workspace.

    Built when ``suggest`` says the gathers of x have no L2 locality (x much larger than ~20 MB and
    rows reaching across it); holds a copy of the values, so it is cached with the row block and
    dropped whenever the matrix data changes."""

    @staticmethod
    def suggest(vt, it, nrows, ncols, nnz, indptr, indices) -> int:
        nb = ctypes.c_int(1)
        N.check(N.load().b2s_csr_colblock_suggest(vt, it, nrows, ncols, nnz, ptr(indptr), ptr(indices),
                                                  stream_ptr(), byref(nb)), "csr_colblock_suggest")
        return int(nb.value)

    def __init__(self, vt, it, nrows, ncols, nnz, indptr, indices, data, nblocks):
        lib = N.load()
        nbytes = int(lib.b2s_csr_colblock_workspace_bytes(vt, it, nrows, nnz, nblocks))
        if nbytes < 0:
            raise ValueError("bad colblock arguments")
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=indptr.device)
        self.handle = c_void_p(0)
        self._lib = lib
        N.check(lib.b2s_csr_colblock_create(vt, it, nrows, ncols, nnz, ptr(indptr), ptr(indices), ptr(data),
                                            nblocks, ptr(self.ws), nbytes, stream_ptr(), byref(self.handle)),
                "csr_colblock_create")
        self.nblocks = nblocks

    def info(self):
        nb, bc = ctypes.c_int(0), c_int64(0)
        per = (c_int64 * 32)()
        N.check(self._lib.b2s_csr_colblock_info(self.handle, byref(nb), byref(bc), per), "csr_colblock_info")
        return {"nblocks": nb.value, "block_cols": bc.value, "blk_nnz": [int(per[i]) for i in range(nb.value)]}

    def spmv(self, x, y, w=None, dot_out=None, peer_ptrs=None):
        arr, npeers = None, 0
        if peer_ptrs is not None:
            peer_ptrs, npeers = _npeers(peer_ptrs)
            arr = _peer_array(peer_ptrs)
        N.check(self._lib.b2s_spmv_colblock(
            self.handle, ptr(x), ptr(y), ptr(w) if w is not None else c_void_p(0),
            ptr(dot_out) if dot_out is not None else c_void_p(0),
            ctypes.cast(arr, c_void_p) if arr is not None else c_void_p(0), npeers, stream_ptr()),
            "spmv_colblock")

    def spmv_from_host(self, x_host: torch.Tensor, y, ncols):
        """y = A x with x in host memory: slice b+1 of x is copied on a side stream while block b
        runs (block b only reads its own slice of x).  Returns the device copy of x."""
        info = self.info()
        bw, nb = info["block_cols"], info["nblocks"]
        x_dev = torch.empty(ncols, dtype=x_host.dtype, device=y.device)
        cur = torch.cuda.current_stream()
        side = _side_stream()
        side.wait_stream(cur)
        for b in range(nb):
            lo, hi = b * bw, min((b + 1) * bw, ncols)
            if hi > lo:
                with torch.cuda.stream(side):
                    x_dev[lo:hi].copy_(x_host[lo:hi], non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(side)
                cur.wait_event(ev)
            N.check(self._lib.b2s_spmv_colblock_part(self.handle, b, ptr(x_dev), ptr(y), stream_ptr()),
                    "spmv_colblock_part")
        x_dev.record_stream(side)
        return x_dev

    def spmv_part(self, b, x, y):
        """one column block of the sequence (block b only reads slice b of x)"""
        N.check(self._lib.b2s_spmv_colblock_part(self.handle, b, ptr(x), ptr(y), stream_ptr()), "spmv_colblock_part")

    def spmv_part_accumulate(self, b, x, y):
        """y += A_b x for block b, whatever its position (y already holds the earlier blocks)"""
        N.check(self._lib.b2s_spmv_colblock_part(self.handle, b | (1 << 30), ptr(x), ptr(y), stream_ptr()),
                "spmv_colblock_part")

    def __del__(self):
        try:
            if self.handle:
                self._lib.b2s_csr_colblock_destroy(self.handle)
                self.handle = c_void_p(0)
        except Exception:
            pass


class HostPipe:
    """y_host = A x_host for a column-blocked operand, pipelined over PCIe in both directions.

    The row block is cut into `nchunks` row chunks, each with its own column-blocked operand
    (2-D blocks: row chunk x column block).  Slice b of x is uploaded on a copy stream while earlier
    blocks run; the launches are ordered so that a row chunk is FINISHED (all its column blocks
    done) as early as possible, and its rows of y travel back on a second copy stream while the
    next chunks are still being computed.  Built once per matrix (holds a second column-blocked
    copy of the values, like ColBlock)."""

    def __init__(self, vt, it, nrows, ncols, indptr, indices, data, nblocks, nchunks, full=None):
        self.nrows, self.ncols, self.nblocks = nrows, ncols, nblocks
        self.full = full          # the un-chunked column-blocked operand (ColBlock) of the same rows
        nchunks = max(1, min(int(nchunks), nrows))
        step = -(-nrows // nchunks)
        step += step & 1                      # even chunk starts keep y slices 16-byte aligned
        self.bounds = [min(i * step, nrows) for i in range(nchunks + 1)]
        while len(self.bounds) > 2 and self.bounds[-2] == self.bounds[-1]:
            self.bounds.pop()
        self.chunks = []
        ip_host = None
        for c in range(len(self.bounds) - 1):
            c0, c1 = self.bounds[c], self.bounds[c + 1]
            lo, hi = int(indptr[c0].item()), int(indptr[c1].item())
            ip = (indptr[c0:c1 + 1] - lo).contiguous()
            cb = ColBlock(vt, it, c1 - c0, ncols, hi - lo, ip, indices[lo:hi], data[lo:hi], nblocks) if hi > lo else None
            self.chunks.append((c0, c1, ip, cb))
        info = next(cb.info() for (_, _, _, cb) in self.chunks if cb is not None)
        self.block_cols = info["block_cols"]
        dev = indptr.device
        self.x_dev = torch.empty(ncols, dtype=data.dtype, device=dev)
        self.y_dev = torch.empty(nrows, dtype=data.dtype, device=dev)
        self.h2d = torch.cuda.Stream(device=dev)
        self.d2h = torch.cuda.Stream(device=dev)
        nc = len(self.chunks)
        if full is not None:
            # only the LAST column block decides when a row of y is final: blocks 0..nb-2 run as single
            # launches over all rows (fewer launches, no per-chunk ramp), the last block chunk by chunk
            self.order = [(-1, b) for b in range(nblocks - 1)] + [(c, nblocks - 1) for c in range(nc)]
        else:
            # launch order: chunk c / block b at key c + b * lag; ties finish chunks first
            lag = max(1, nc // nblocks)
            self.order = sorted(((c, b) for c in range(nc) for b in range(nblocks)),
                                key=lambda cb_: (cb_[0] + cb_[1] * lag, -cb_[1]))

    def run(self, x_host, y_host: torch.Tensor, x_dev=None):
        """x_host: host vector uploaded slice by slice — or None with `x_dev` already complete on the
        device (several ranks: the slices were all-gathered over NVLink); y_host: host result."""
        cur = torch.cuda.current_stream()
        self.h2d.wait_stream(cur)          # earlier readers of x_dev / y_dev are done
        self.d2h.wait_stream(cur)
        bw, nb = self.block_cols, self.nblocks
        ev_x = []
        xd = self.x_dev if x_dev is None else x_dev
        if x_dev is None:
            with torch.cuda.stream(self.h2d):
                for b in range(nb):
                    lo, hi = b * bw, min((b + 1) * bw, self.ncols)
                    if hi > lo:
                        self.x_dev[lo:hi].copy_(x_host[lo:hi], non_blocking=True)
                    e = torch.cuda.Event()
                    e.record(self.h2d)
                    ev_x.append(e)
        waited = [x_dev is not None] * nb
        done_blocks = [0] * len(self.chunks)
        for (c, b) in self.order:
            if not waited[b]:
                cur.wait_event(ev_x[b])
                waited[b] = True
            if c < 0:                      # a whole-matrix launch of an early column block
                self.full.spmv_part(b, xd, self.y_dev)
                for i in range(len(done_blocks)):
                    done_blocks[i] += 1
                continue
            c0, c1, _, cb = self.chunks[c]
            y_c = self.y_dev[c0:c1]
            if cb is None:
                if b == 0:
                    y_c.zero_()
            elif self.full is not None:
                cb.spmv_part_accumulate(b, xd, y_c)
            else:
                cb.spmv_part(b, xd, y_c)
            done_blocks[c] += 1
            if done_blocks[c] == nb:       # chunk finished: its rows of y go home
                e = torch.cuda.Event()
                e.record(cur)
                self.d2h.wait_event(e)
                with torch.cuda.stream(self.d2h):
                    y_host[c0:c1].copy_(y_c, non_blocking=True)
        cur.wait_stream(self.d2h)          # the caller's stream order covers the copies
        return y_host


# ------------------------------------------------------------------ typed wrappers
def spmv(vt, it, nrows, ncols, nnz, indptr, indices, data, x, y, plan=None, variant=N.B2S_SPMV_AUTO):
    N.check(
        N.load().b2s_spmv_csr(
            vt, it, nrows, ncols, nnz, ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y),
            plan.handle if plan is not None else c_void_p(0), variant, stream_ptr(),
        ),
        "spmv_csr",
    )


def _peer_array(ptrs):
    arr = (c_void_p * max(len(ptrs), 1))(*[c_void_p(int(q)) for q in ptrs])
    return arr


def _npeers(peer_ptrs):
    """peer_ptrs is a list of unicast pointers, or ("mc", ptr) for an NVSwitch multicast address"""
    if isinstance(peer_ptrs, tuple):
        return [peer_ptrs[1]], -1
    return list(peer_ptrs), len(peer_ptrs)


def spmv_bcast(vt, it, nrows, ncols, nnz, indptr, indices, data, x, y_local, peer_ptrs, plan):
    """SpMV whose y stores also go to the peers' replicated buffers (fused all-gather)."""
    peer_ptrs, npeers = _npeers(peer_ptrs)
    arr = _peer_array(peer_ptrs)
    N.check(
        N.load().b2s_spmv_csr_bcast(
            vt, it, nrows, ncols, nnz, ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y_local),
            ctypes.cast(arr, c_void_p), npeers, plan.handle, stream_ptr(),
        ),
        "spmv_csr_bcast",
    )


def cg_pupdate_bcast(p, r, rho, rho1, peer_ptrs):
    dt = np_dtype_of(p)
    peer_ptrs, npeers = _npeers(peer_ptrs)
    arr = _peer_array(peer_ptrs)
    N.check(
        N.load().b2s_cg_pupdate_bcast(vt_enum(dt), p.numel(), ptr(p), ptr(r), ptr(rho), ptr(rho1),
                                      ctypes.cast(arr, c_void_p), npeers, stream_ptr()),
        "cg_pupdate_bcast",
    )


def cg_pupdate_halo(p, r, rho, rho1, peer_ptrs, lo, hi):
    """p update whose result is stored only into the slices the peers need (halo exchange)"""
    dt = np_dtype_of(p)
    arr = _peer_array(peer_ptrs)
    n = max(len(peer_ptrs), 1)
    lo_a = (c_int64 * n)(*[int(v) for v in lo])
    hi_a = (c_int64 * n)(*[int(v) for v in hi])
    N.check(
        N.load().b2s_cg_pupdate_halo(vt_enum(dt), p.numel(), ptr(p), ptr(r), ptr(rho), ptr(rho1),
                                     ctypes.cast(arr, c_void_p), len(peer_ptrs), ctypes.cast(lo_a, c_void_p),
                                     ctypes.cast(hi_a, c_void_p), stream_ptr()),
        "cg_pupdate_halo",
    )


def spmv_dot(vt, it, nrows, ncols, nnz, indptr, indices, data, x, y, w, plan, dot_out, board=None, channel=0):
    if board is not None:   # w.y summed over the ranks inside the final reduction kernel
        N.check(
            N.load().b2s_spmv_csr_dot_allreduce(
                vt, it, nrows, ncols, nnz, ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y), ptr(w),
                plan.handle, ptr(dot_out), ctypes.cast(board.arr, c_void_p), board.rank, board.nranks, int(channel),
                ptr(board.seq), ptr(board.err), stream_ptr()),
            "spmv_csr_dot_allreduce")
        return
    N.check(
        N.load().b2s_spmv_csr_dot(
            vt, it, nrows, ncols, nnz, ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y), ptr(w),
            plan.handle, ptr(dot_out), stream_ptr(),
        ),
        "spmv_csr_dot",
    )


def axpby(y, x, a, b, isalpha, negate):
    vt = vt_enum(np_dtype_of(y))
    N.check(
        N.load().b2s_axpby(vt, y.numel(), ptr(y), ptr(x), ptr(a), ptr(b), int(bool(isalpha)), int(bool(negate)),
                           stream_ptr()),
        "axpby",
    )


def dot(x, y, conj=False, out=None, ws=None):
    dt = np_dtype_of(x)
    if out is None:
        out = empty(1, dt)
    N.check(
        N.load().b2s_dot(vt_enum(dt), x.numel(), ptr(x), ptr(y), int(conj), ptr(out),
                         ptr(ws if ws is not None else reduce_ws()), stream_ptr()),
        "dot",
    )
    return out


def nrm2(x, out=None):
    dt = np_dtype_of(x)
    if out is None:
        out = empty(1, real_dtype(dt))
    N.check(N.load().b2s_nrm2(vt_enum(dt), x.numel(), ptr(x), ptr(out), ptr(reduce_ws()), stream_ptr()), "nrm2")
    return out


_cgs_ws = {}


def cgs_ws() -> torch.Tensor:
    dev = require_cuda()
    key = (dev.index, torch.cuda.current_stream().cuda_stream)
    ws = _cgs_ws.get(key)
    if ws is None:
        ws = torch.zeros(int(N.load().b2s_cgs_workspace_bytes()), dtype=torch.uint8, device=dev)
        _cgs_ws[key] = ws
    return ws


def cgs_project(basis, ldv, n, k, u, h):
    """h[:k] = basis[:k, :n]^H u   (GMRES Arnoldi projection; basis rows are the Krylov vectors)"""
    dt = np_dtype_of(u)
    N.check(N.load().b2s_cgs_project(vt_enum(dt), n, k, ptr(basis), ldv, ptr(u), ptr(h), ptr(cgs_ws()),
                                     stream_ptr()), "cgs_project")
    return h


def cgs_update(basis, ldv, n, k, h, u, negate=True, nrm_out=None):
    """u -= basis[:k]^T h (negate) or u += ... ; optional fused ||u|| into the device scalar nrm_out"""
    dt = np_dtype_of(u)
    N.check(N.load().b2s_cgs_update(vt_enum(dt), n, k, ptr(basis), ldv, ptr(h), int(bool(negate)), ptr(u),
                                    ptr(nrm_out) if nrm_out is not None else c_void_p(0), ptr(cgs_ws()),
                                    stream_ptr()), "cgs_update")
    return u


def vscale_inv(x, s, out):
    """out = x / s[0] with s a device real scalar"""
    dt = np_dtype_of(x)
    N.check(N.load().b2s_vscale_inv(vt_enum(dt), x.numel(), ptr(x), ptr(s), ptr(out), stream_ptr()), "vscale_inv")
    return out


def cg_update(x, r, p, q, rho, pq, rr_out, ws=None, board=None, channel=0, cur_out=None, prev_out=None):
    dt = np_dtype_of(x)
    if board is not None:   # r.r summed over the ranks inside the kernel's final reduction
        N.check(
            N.load().b2s_cg_update_allreduce(
                vt_enum(dt), x.numel(), ptr(x), ptr(r), ptr(p), ptr(q), ptr(rho), ptr(pq), ptr(rr_out),
                ptr(ws if ws is not None else reduce_ws()), ctypes.cast(board.arr, c_void_p), board.rank,
                board.nranks, int(channel), ptr(board.seq), ptr(cur_out), ptr(prev_out), ptr(board.err), stream_ptr()),
            "cg_update_allreduce")
        return
    N.check(
        N.load().b2s_cg_update(vt_enum(dt), x.numel(), ptr(x), ptr(r), ptr(p), ptr(q), ptr(rho), ptr(pq),
                               ptr(rr_out), ptr(ws if ws is not None else reduce_ws()), stream_ptr()),
        "cg_update",
    )


def cg_pupdate(p, r, rho, rho1):
    dt = np_dtype_of(p)
    N.check(N.load().b2s_cg_pupdate(vt_enum(dt), p.numel(), ptr(p), ptr(r), ptr(rho), ptr(rho1), stream_ptr()),
            "cg_pupdate")
