"""csr_array — the scipy.sparse-shaped CSR matrix of the reference
(reference legate_sparse/csr.py:88-558) on top of the native kernels.

Hot path (SURVEY §8a): ``dot``/``@`` → :func:`spmv` (csr.py:562-593 upstream) or
:func:`spgemm_csr_csr_csr` (csr.py:598-748 upstream) → C ABI → sm_90a kernels.

Storage differs from the reference on purpose: plain ``indptr`` (int64) instead of the
Rect<1> ``pos`` store, column indices narrowed to int32 on the device when
``ncols < 2**31`` (scipy does the same), values in the matrix dtype.  Construction logic
(dense→CSR, COO→CSR, DIA→CSR) runs on the host in numpy — the reference marks those paths
as single-task / not scalable (csr.py:134-138) and SURVEY §2 keeps them out of the GPU
scope; device-resident arrays (torch CUDA tensors) can be passed directly to skip the host.

Vectors may be numpy arrays (result returned as numpy; one H2D + one D2H copy) or CUDA
``torch.Tensor`` (result stays on the device).
"""
from __future__ import annotations

import warnings
from ctypes import byref, c_int64

import numpy
import scipy.sparse
import torch

from . import _native as N
from . import dist
from .base import CompressedBase
from .settings import settings
from .types import coord_ty, nnz_ty  # noqa: F401
from .utils import (
    SUPPORTED_DATATYPES,
    cast_to_common_type,
    is_dtype_supported,
)

_INT32_MAX = 2**31 - 1


def _is_dev(x) -> bool:
    return isinstance(x, torch.Tensor) and x.is_cuda


def _as_host(x, dtype=None, copy=False):
    """numpy / torch → numpy array on the host."""
    if isinstance(x, torch.Tensor):
        a = x.detach().cpu().numpy()
        copy = False if x.is_cuda else copy
    else:
        a = numpy.asarray(x)
    if dtype is not None and a.dtype != numpy.dtype(dtype):
        a = a.astype(dtype)
        copy = False
    return a.copy() if copy else a


class _RowBlock:
    """Device-resident rows [r0, r1) of a matrix: rebased indptr, (narrowed) indices, data."""

    __slots__ = ("r0", "r1", "nnz", "indptr", "indices", "data", "itype", "plan", "colblock", "hostpipe", "_colrange")

    def __init__(self, r0, r1, indptr, indices, data):
        self.r0, self.r1 = int(r0), int(r1)
        self.indptr, self.indices, self.data = indptr, indices, data
        self.nnz = int(data.numel())
        self.itype = N.B2S_I32 if indices.dtype == torch.int32 else N.B2S_I64
        self.plan = None
        self.colblock = None   # None: not decided yet, False: not worthwhile, else _device.ColBlock
        self.hostpipe = None   # _device.HostPipe of the host-vector path (built on first use)
        self._colrange = None

    @property
    def nrows(self):
        return self.r1 - self.r0

    def colrange(self):
        """[min col, max col] touched by this row block = the x window the block needs
        (the reference's image(crd→x, MIN_MAX), csr.py:591); (1, 0) for an empty block."""
        if self._colrange is None:
            if self.nnz == 0:
                self._colrange = (1, 0)
            else:
                mn, mx = torch.aminmax(self.indices)
                self._colrange = (int(mn.item()), int(mx.item()))
        return self._colrange


class csr_array(CompressedBase):
    format = "csr"
    __array_ufunc__ = None  # make numpy defer to __rmul__/__rmatmul__

    def __init__(self, arg, shape=None, dtype=None, copy=False):
        self.ndim = 2
        self.indices_sorted = False
        self.canonical_format = False
        self._h_data = self._h_indices = self._h_indptr = None
        self._g_data = self._g_indices = self._g_indptr = None
        self._blk = None
        self._bounds = None
        self._B_full = None  # replicated device copy used when this matrix is the B of A@B
        self._nnz_per_rank = None

        if dtype is not None:
            dtype = numpy.dtype(dtype)

        # dense CUDA tensor → CSR on the device (two-pass count / fill with a `!= 0` test:
        # reference dense_to_csr.cu:25-43,128-149); a dense CPU tensor goes the numpy way below
        if isinstance(arg, torch.Tensor) and arg.dim() == 2:
            if arg.is_cuda:
                shape = tuple(arg.shape)
                arg = _dense_to_csr_device(arg)
                copy = False
            else:
                arg = arg.detach().numpy()

        if isinstance(arg, (scipy.sparse.csr_array, scipy.sparse.csr_matrix)):
            shape = arg.shape
            arg = (arg.data, arg.indices, arg.indptr)

        if isinstance(arg, numpy.ndarray):
            # dense → CSR, two-pass count/fill with a `!= 0` test
            # (reference dense_to_csr.cc:32-40,55-64); keeps arg.dtype, ignores `dtype`
            assert arg.ndim == 2
            shape = arg.shape
            mask = arg != 0
            counts = mask.sum(axis=1, dtype=numpy.int64)
            indptr = numpy.zeros(shape[0] + 1, dtype=numpy.int64)
            numpy.cumsum(counts, out=indptr[1:])
            rows, cols = numpy.nonzero(mask)  # row-major → columns ascending within a row
            self._h_indptr = indptr
            self._h_indices = cols.astype(numpy.int64, copy=False)
            self._h_data = numpy.ascontiguousarray(arg[rows, cols])
            dtype = arg.dtype

        elif isinstance(arg, csr_array):
            shape = arg.shape
            if arg._h_data is not None:
                self._h_data = arg._h_data.copy()
                self._h_indices = arg._h_indices.copy()
                self._h_indptr = arg._h_indptr.copy()
            if arg._g_data is not None:
                self._g_data = arg._g_data.clone()
                self._g_indices = arg._g_indices.clone()
                self._g_indptr = arg._g_indptr.clone()
            if arg._h_data is None and arg._g_data is None and arg._blk is not None:
                b = arg._blk   # row-sharded matrix: deep copy of this rank's block
                self._blk = _RowBlock(b.r0, b.r1, b.indptr.clone(), b.indices.clone(), b.data.clone())
                self._nnz_per_rank = arg._nnz_per_rank
            self._bounds = arg._bounds
            self.indices_sorted = arg.indices_sorted
            self.canonical_format = arg.canonical_format
            if dtype is None:
                dtype = arg.dtype

        elif isinstance(arg, tuple):
            if len(arg) == 2:
                if not isinstance(arg[1], tuple):
                    # empty matrix ctor: csr_array((M, N), [dtype])
                    (M, Ncols) = arg
                    shape = arg
                    if dtype is None:
                        dtype = numpy.dtype(numpy.float64)
                    arg = (
                        numpy.zeros(0, dtype=dtype),
                        numpy.zeros(0, dtype=coord_ty),
                        numpy.zeros(int(M) + 1, dtype=coord_ty),
                    )
                else:
                    # COO: (data, (row, col)) — stable sort by row; duplicates are kept and
                    # columns keep their input order inside a row (reference csr.py:198-219)
                    if shape is None:
                        raise AssertionError("Cannot infer shape in this case.")
                    st_data, (st_row, st_col) = arg
                    if _is_dev(st_data) and _is_dev(st_row) and _is_dev(st_col):
                        row_sort = torch.argsort(st_row, stable=True)
                        new_data = st_data[row_sort]
                        new_col = st_col[row_sort].to(torch.int64)
                        counts = torch.bincount(st_row.to(torch.int64), minlength=int(shape[0]))
                        new_ptr = torch.zeros(int(shape[0]) + 1, dtype=torch.int64, device=st_row.device)
                        torch.cumsum(counts, 0, out=new_ptr[1:])
                        arg = (new_data, new_col, new_ptr)
                    else:
                        row_array = _as_host(st_row)
                        row_sort = numpy.argsort(row_array, kind="stable")
                        new_data = _as_host(st_data)[row_sort]
                        new_col = _as_host(st_col)[row_sort]
                        new_ptr = numpy.zeros(int(shape[0]) + 1, dtype=numpy.int64)
                        numpy.cumsum(
                            numpy.bincount(row_array.astype(numpy.int64, copy=False), minlength=int(shape[0])),
                            out=new_ptr[1:],
                        )
                        arg = (new_data, new_col, new_ptr)
                    copy = False

            if len(arg) == 3:
                if shape is None or len(shape) != 2:
                    raise AssertionError("Cannot infer shape in this case.")
                (data, indices, indptr) = arg
                nptr = indptr.shape[0]
                if nptr != int(shape[0]) + 1:
                    raise AssertionError("Can't understand tuple of inputs for csr_array constructor")
                if _is_dev(data) or _is_dev(indices) or _is_dev(indptr):
                    from ._device import to_device

                    self._g_data = to_device(data, copy=copy)
                    gi = to_device(indices, copy=copy)
                    if gi.dtype not in (torch.int32, torch.int64):
                        gi = gi.to(torch.int64)
                    self._g_indices = gi
                    self._g_indptr = to_device(indptr, dtype=numpy.int64, copy=copy)
                    if dtype is None:
                        from ._device import np_dtype_of

                        dtype = np_dtype_of(self._g_data)
                else:
                    self._h_data = _as_host(data, copy=copy)
                    self._h_indices = _as_host(indices, dtype=coord_ty, copy=copy)
                    self._h_indptr = _as_host(indptr, dtype=coord_ty, copy=copy)
                    if dtype is None:
                        dtype = self._h_data.dtype
        else:
            raise NotImplementedError("Can't convert to CSR from the input")

        assert shape is not None
        self.shape = tuple(int(i) for i in shape)

        stored = self._stored_dtype()
        if dtype is None:
            dtype = stored
        dtype = numpy.dtype(dtype)
        if stored != dtype:
            self._cast_data_inplace(dtype)
        self._dtype = dtype

    # ------------------------------------------------------------------ internals
    def _stored_dtype(self):
        if self._h_data is not None:
            return self._h_data.dtype
        from ._device import np_dtype_of

        return np_dtype_of(self._g_data if self._g_data is not None else self._blk.data)

    def _cast_data_inplace(self, dtype):
        if self._h_data is not None:
            self._h_data = self._h_data.astype(dtype)
        if self._g_data is not None:
            from ._device import torch_dtype

            self._g_data = self._g_data.to(torch_dtype(dtype))
        if self._h_data is None and self._g_data is None and self._blk is not None:
            from ._device import torch_dtype

            b = self._blk   # row-sharded: cast the block's values, keep its structure
            self._blk = _RowBlock(b.r0, b.r1, b.indptr, b.indices, b.data.to(torch_dtype(dtype)))
            return
        self._blk = None

    @classmethod
    def _from_parts(cls, shape, dtype, h=None, g=None, bounds=None, blk=None):
        self = cls.__new__(cls)
        self.ndim = 2
        self.indices_sorted = False
        self.canonical_format = False
        self._h_data, self._h_indices, self._h_indptr = h if h is not None else (None, None, None)
        self._g_data, self._g_indices, self._g_indptr = g if g is not None else (None, None, None)
        self._blk = blk
        self._bounds = bounds
        self._B_full = None
        self._nnz_per_rank = None
        self.shape = tuple(int(i) for i in shape)
        self._dtype = numpy.dtype(dtype)
        return self

    @classmethod
    def from_row_block(cls, data, indices, indptr_local, shape, row_start=0, bounds=None):
        """Build a (possibly distributed) matrix from THIS rank's row block only: rows
        [row_start, row_start+len(indptr_local)-1) with a 0-based local indptr.  Nothing is
        replicated — the layout a 1-D row-partitioned run keeps per GPU (reference
        csr.py:587-591).  Arrays are device tensors (or are uploaded)."""
        from ._device import np_dtype_of, to_device

        d = to_device(data)
        ip = to_device(indptr_local, dtype=numpy.int64)
        idx = to_device(indices)
        if idx.dtype not in (torch.int32, torch.int64):
            idx = idx.to(torch.int64)
        nloc = ip.numel() - 1
        if bounds is None:
            bounds = dist.row_block_bounds(shape[0], dist.world_size())
        blk = _RowBlock(row_start, row_start + nloc, ip, idx, d)
        return cls._from_parts(shape, np_dtype_of(d), bounds=numpy.asarray(bounds, dtype=numpy.int64), blk=blk)

    def _have_host(self):
        return self._h_data is not None

    def _ensure_host(self):
        if self._h_data is None:
            if self._g_data is None:
                # row-sharded matrix (from_row_block / distributed SpGEMM result): the global
                # arrays are gathered on request — a COLLECTIVE, every rank must get here
                self._gather_global()
            self._h_data = self._g_data.detach().cpu().numpy()
            self._h_indices = self._g_indices.detach().cpu().numpy().astype(numpy.int64, copy=False)
            self._h_indptr = self._g_indptr.detach().cpu().numpy()
        return self._h_data, self._h_indices, self._h_indptr

    def _gather_global(self):
        """Materialise the replicated global arrays of a row-sharded matrix on the device:
        all-gather(v) of the row blocks; the global indptr comes from the per-rank nnz offsets
        (the reference's ncclAllGather + scan of per-rank nnz, spgemm_csr_csr_csr.cu:43-62).
        Collective; a no-op when the global arrays already exist."""
        if self._g_data is not None or self._h_data is not None:
            return
        blk = self._blk
        if blk is None:
            raise RuntimeError("csr_array holds neither global arrays nor a row block")
        if dist.world_size() == 1:
            self._g_data, self._g_indices, self._g_indptr = blk.data, blk.indices, blk.indptr
            return
        all_idx, counts = dist.allgather_varlen(blk.indices)
        all_dat, _ = dist.allgather_varlen(blk.data)
        row_nnz = blk.indptr[1:] - blk.indptr[:-1]
        all_row_nnz, _ = dist.allgather_varlen(row_nnz)
        g_ptr = torch.zeros(self.shape[0] + 1, dtype=torch.int64, device=blk.data.device)
        torch.cumsum(all_row_nnz, 0, out=g_ptr[1:])
        self._g_data, self._g_indices, self._g_indptr = all_dat, all_idx, g_ptr
        self._nnz_per_rank = numpy.asarray(counts, dtype=numpy.int64)

    def gather(self):
        """Replicate a row-sharded matrix on every rank (collective); returns self."""
        self._gather_global()
        return self

    def nnz_offset(self):
        """Global position of this rank's first stored entry (row-sharded matrices): the exclusive
        scan of the per-rank nnz, what the reference adds to its local `pos`
        (spgemm_csr_csr_csr.cu:317-332)."""
        counts = self._rank_nnz()
        return int(counts[: dist.rank()].sum())

    def _rank_nnz(self):
        if getattr(self, "_nnz_per_rank", None) is None:
            blk = self._block()
            self._nnz_per_rank = dist.allgather_i64(blk.nnz, blk.data.device)
        return self._nnz_per_rank

    def row_bounds(self):
        if self._bounds is None:
            self._bounds = dist.row_block_bounds(self.shape[0], dist.world_size())
        return self._bounds

    def set_row_bounds(self, bounds):
        """Override the row partition (e.g. dist.nnz_balanced_bounds); drops the cached block."""
        self._bounds = numpy.asarray(bounds, dtype=numpy.int64)
        self._blk = None

    def _narrow_ok(self):
        return self.shape[1] <= _INT32_MAX and not settings.index64()

    def _block(self) -> _RowBlock:
        """Device row block of this rank (the whole matrix for a single process)."""
        if self._blk is not None:
            return self._blk
        from ._device import require_cuda, to_device

        dev = require_cuda()
        G, r = dist.world_size(), dist.rank()
        bounds = self.row_bounds()
        r0, r1 = int(bounds[r]), int(bounds[r + 1])
        narrow = self._narrow_ok()
        if self._g_data is not None:
            ip = self._g_indptr[r0 : r1 + 1]
            lo, hi = int(self._g_indptr[r0].item()), int(self._g_indptr[r1].item())
            idx = self._g_indices[lo:hi]
            dat = self._g_data[lo:hi]
            if G > 1 or r0 != 0:
                ip = ip - lo
                dat = dat.clone()  # fresh allocation → 16-byte aligned for the vector loads
                idx = idx.clone()
            if narrow and idx.dtype == torch.int64:
                idx32 = torch.empty(idx.numel(), dtype=torch.int32, device=dev)
                from ._device import ptr, stream_ptr

                N.check(N.load().b2s_cast_i64_to_i32(idx.numel(), ptr(idx), ptr(idx32), stream_ptr()), "cast")
                idx = idx32
        else:
            hd, hi_, hp = self._ensure_host()
            lo, hi = int(hp[r0]), int(hp[r1])
            ip = to_device(numpy.ascontiguousarray(hp[r0 : r1 + 1] - lo))
            idx_host = hi_[lo:hi]
            idx = to_device(numpy.ascontiguousarray(idx_host.astype(numpy.int32) if narrow else idx_host))
            dat = to_device(numpy.ascontiguousarray(hd[lo:hi]))
        self._blk = _RowBlock(r0, r1, ip, idx, dat)
        return self._blk

    def _plan(self, blk: _RowBlock):
        if blk.plan is None and blk.nnz > 0:
            from ._device import SpmvPlan

            blk.plan = SpmvPlan(blk.itype, blk.nrows, self.shape[1], blk.nnz, blk.indptr, blk.indices)
        return blk.plan

    def _colblock(self, blk: _RowBlock):
        """Column-blocked copy of the row block when x would not stay L2-resident (decided once by the
        native heuristic; see b2s_csr_colblock_suggest), else None."""
        if blk.colblock is None:
            blk.colblock = False
            if blk.nnz > 0 and settings.spmv_variant() == N.B2S_SPMV_AUTO:
                from ._device import ColBlock, vt_enum

                vt = vt_enum(self.dtype)
                nb = ColBlock.suggest(vt, blk.itype, blk.nrows, self.shape[1], blk.nnz, blk.indptr, blk.indices)
                if nb > 1:
                    blk.colblock = ColBlock(vt, blk.itype, blk.nrows, self.shape[1], blk.nnz, blk.indptr,
                                            blk.indices, blk.data, nb)
        return blk.colblock or None

    def _hostpipe(self, blk: _RowBlock):
        """2-D blocked operand + copy streams of the host-vector SpMV path (built on first use)."""
        hp = getattr(blk, "hostpipe", None)
        if hp is None:
            import os

            from ._device import HostPipe, vt_enum

            cb = self._colblock(blk)
            nchunks = int(os.environ.get("LEGATE_SPARSE_HOSTPIPE_CHUNKS", "8"))
            hp = HostPipe(vt_enum(self.dtype), blk.itype, blk.nrows, self.shape[1], blk.indptr, blk.indices,
                          blk.data, cb.nblocks, nchunks, full=cb)
            blk.hostpipe = hp
        return hp

    # ------------------------------------------------------------------ properties
    @property
    def dim(self):
        return self.ndim

    @property
    def nnz(self):
        if self._h_data is not None:
            return int(self._h_data.shape[0])
        if self._g_data is not None:
            return int(self._g_data.numel())
        # row-sharded matrix: global nnz = sum of the per-rank counts
        return int(self._rank_nnz().sum())

    @property
    def dtype(self):
        return self._dtype

    def get_data(self):
        return self._ensure_host()[0]

    def set_data(self, data):
        if _is_dev(data):
            from ._device import np_dtype_of

            self._g_data = data.contiguous()
            if self._g_indices is None:
                from ._device import to_device

                self._g_indices = to_device(self._h_indices)
                self._g_indptr = to_device(self._h_indptr)
            self._h_data = None
            self._dtype = np_dtype_of(data)
        else:
            data = numpy.ascontiguousarray(_as_host(data))
            self._ensure_host()
            self._h_data = data
            self._g_data = self._g_indices = self._g_indptr = None
            self._dtype = data.dtype
        self._blk = None
        self._B_full = None

    data = property(fget=get_data, fset=set_data)

    def get_indices(self):
        return self._ensure_host()[1]

    def set_indices(self, indices):
        self._ensure_host()
        self._h_indices = numpy.ascontiguousarray(_as_host(indices, dtype=coord_ty))
        self._g_data = self._g_indices = self._g_indptr = None
        self._blk = None
        self._B_full = None
        self.canonical_format = False
        self.indices_sorted = False

    indices = property(fget=get_indices, fset=set_indices)

    def get_indptr(self):
        return self._ensure_host()[2]

    # indptr is read-only (reference csr.py:336)
    indptr = property(fget=get_indptr)

    # reference-internal names, read by its tests (test_unary_operation.py:32)
    @property
    def vals(self):
        return self.data

    @property
    def crd(self):
        return self.indices

    @property
    def pos(self):
        ip = self.indptr
        return numpy.stack([ip[:-1], ip[1:] - 1], axis=1)  # inclusive {lo, hi} like Rect<1>

    def has_sorted_indices(self):
        return self.indices_sorted

    def has_canonical_format(self):
        return self.canonical_format

    # ------------------------------------------------------------------ conversions
    def _astype_data(self, dtype, casting="unsafe"):
        if self._h_data is not None:
            return self._h_data.astype(dtype, casting=casting, copy=True)
        from ._device import torch_dtype

        src = self._g_data if self._g_data is not None else self._blk.data
        return src.to(torch_dtype(dtype), copy=True)

    def _with_data(self, data, copy=True):
        """A different matrix with the same sparsity structure (reference base.py:177-199);
        structure arrays are shared unless ``copy``."""
        if _is_dev(data) and self._h_data is None and self._g_data is None and self._blk is not None:
            # row-sharded matrix: `data` are the values of this rank's block
            from ._device import np_dtype_of

            b = self._blk
            assert data.numel() == b.nnz
            ip, idx = (b.indptr.clone(), b.indices.clone()) if copy else (b.indptr, b.indices)
            out = csr_array._from_parts(self.shape, np_dtype_of(data), bounds=self._bounds,
                                        blk=_RowBlock(b.r0, b.r1, ip, idx, data.contiguous()))
            out._nnz_per_rank = self._nnz_per_rank
            if not copy:
                out._blk.plan = b.plan
            return out
        if _is_dev(data):
            from ._device import np_dtype_of, to_device

            if self._g_indices is None:
                self._g_indices = to_device(self._h_indices)
                self._g_indptr = to_device(self._h_indptr)
            gi, gp = self._g_indices, self._g_indptr
            if copy:
                gi, gp = gi.clone(), gp.clone()
            out = csr_array._from_parts(self.shape, np_dtype_of(data), g=(data, gi, gp), bounds=self._bounds)
        else:
            data = numpy.asarray(data)
            _, hi, hp = self._ensure_host()
            if copy:
                hi, hp = hi.copy(), hp.copy()
            out = csr_array._from_parts(self.shape, data.dtype, h=(data, hi, hp), bounds=self._bounds)
        # share the already-uploaded structure of the row block when only values change
        if not copy and self._blk is not None and self._blk.data.numel() == (
            data.numel() if _is_dev(data) else data.shape[0]
        ) and dist.world_size() == 1:
            from ._device import to_device

            b = self._blk
            nb = _RowBlock(b.r0, b.r1, b.indptr, b.indices, to_device(data))
            nb.plan = b.plan
            out._blk = nb
        return out

    def copy(self):
        return csr_array(self)

    def conj(self, copy=True):
        if copy:
            return self.copy().conj(copy=False)
        return self._with_data(self.data.conj(), copy=False)

    def diagonal(self, k=0):
        rows, cols = self.shape
        if k <= -rows or k >= cols:
            return numpy.empty(0, dtype=self.dtype)
        if k != 0:
            raise NotImplementedError
        from ._device import empty, ptr, stream_ptr, to_host, vt_enum

        blk = self._block()
        n_out = min(rows, cols)
        out = torch.zeros(blk.nrows, dtype=blk.data.dtype, device=blk.data.device)
        # global row id = local row + r0: shift the column ids by passing a shifted compare
        if blk.r0 == 0:
            N.check(
                N.load().b2s_csr_diagonal(vt_enum(self.dtype), blk.itype, blk.nrows, ptr(blk.indptr),
                                          ptr(blk.indices), ptr(blk.data), ptr(out), stream_ptr()),
                "csr_diagonal",
            )
        else:
            shifted = (blk.indices.to(torch.int64) - blk.r0)
            N.check(
                N.load().b2s_csr_diagonal(vt_enum(self.dtype), N.B2S_I64, blk.nrows, ptr(blk.indptr),
                                          ptr(shifted), ptr(blk.data), ptr(out), stream_ptr()),
                "csr_diagonal",
            )
        full = dist.allgather_rows(out, self.row_bounds()) if dist.world_size() > 1 else out
        return to_host(full[:n_out])

    def todense(self, order=None, out=None):
        """CSR → dense (reference csr.py:370-383 → CSRToDense task, csr_to_dense.cu:25-47).
        Duplicates: last one wins (csr_to_dense.cc loop).  Single process with a GPU: the
        b2s_csr_to_dense kernel fills a device matrix (returned as numpy like every host-facing
        result, or written into a CUDA tensor ``out``); several ranks / no GPU: assembled on the
        host from the gathered arrays."""
        if order is not None:
            raise NotImplementedError
        if out is not None:
            out_dtype = _torch_np_dtype(out) if isinstance(out, torch.Tensor) else numpy.asarray(out).dtype
            if out_dtype != self.dtype:
                raise ValueError(f"Output type {out_dtype} is not consistent with dtype {self.dtype}")
        if dist.world_size() == 1 and torch.cuda.is_available() and self.shape[0] * self.shape[1] > 0:
            from ._device import ptr, stream_ptr, to_host, torch_dtype, vt_enum

            blk = self._block()
            dense = out if (_is_dev(out) and out.is_contiguous()) else torch.empty(
                self.shape, dtype=torch_dtype(self.dtype), device=blk.data.device)
            N.check(N.load().b2s_csr_to_dense(vt_enum(self.dtype), blk.itype, self.shape[0], self.shape[1],
                                              ptr(blk.indptr), ptr(blk.indices), ptr(blk.data), ptr(dense),
                                              stream_ptr()), "csr_to_dense")
            if out is None:
                return to_host(dense)
            if dense is not out:
                if isinstance(out, torch.Tensor):
                    out.copy_(dense)
                else:
                    numpy.asarray(out)[...] = to_host(dense)
            return out
        hd, hi, hp = self._ensure_host()
        if out is not None:
            out = numpy.asarray(out)
            out[...] = 0
        else:
            out = numpy.zeros(self.shape, dtype=self.dtype)
        rows = numpy.repeat(numpy.arange(self.shape[0], dtype=numpy.int64), numpy.diff(hp))
        out[rows, hi] = hd
        return out

    def multiply(self, other):
        return self * other

    def __rmul__(self, other):
        return self * other

    def __mul__(self, other):
        if numpy.ndim(other) == 0:
            return self._with_data(self.data * other)
        raise NotImplementedError

    def __rmatmul__(self, other):
        raise NotImplementedError

    def __matmul__(self, other):
        return self.dot(other)

    # ------------------------------------------------------------------ the hot path
    def dot(self, other, out=None):
        """``A @ x`` (SpMV) for 1-D / (n,1) x, ``A @ B`` (SpGEMM) for csr_array B
        (reference csr.py:419-493, same checks in the same order)."""
        if out is not None:
            assert isinstance(out, (numpy.ndarray, torch.Tensor))

        other_dtype = other.dtype if not isinstance(other, torch.Tensor) else _torch_np_dtype(other)
        if not is_dtype_supported(self.dtype) or not is_dtype_supported(other_dtype):
            msg = "Only the following datatypes are currently supported:" f" {SUPPORTED_DATATYPES}."
            raise NotImplementedError(msg)

        if len(other.shape) == 1 or (len(other.shape) == 2 and other.shape[1] == 1):
            if not isinstance(other, (numpy.ndarray, torch.Tensor)):
                other = numpy.array(other)
            assert self.shape[1] == other.shape[0]
            other_originally_2d = False
            if len(other.shape) == 2 and other.shape[1] == 1:
                other = other.squeeze(1) if isinstance(other, torch.Tensor) else other.squeeze(1)
                other_originally_2d = True

            if isinstance(other, numpy.ndarray) and not other.flags.c_contiguous:
                # the reference warns and copies a transformed (strided) x (csr.py:444-452)
                warnings.warn(
                    "CSR SpMV creating an implicit copy due to transformed x vector.",
                    category=RuntimeWarning,
                    stacklevel=2,
                )
                other = numpy.ascontiguousarray(other)

            A, x = cast_to_common_type(self, other)
            if out is not None:
                out_dtype = out.dtype if isinstance(out, numpy.ndarray) else _torch_np_dtype(out)
                if out_dtype != A.dtype:
                    raise ValueError(
                        f"Output type {out_dtype} is not consistent " f"with resolved dtype {A.dtype}"
                    )
                if other_originally_2d:
                    assert tuple(out.shape) == (self.shape[0], 1)
                else:
                    assert tuple(out.shape) == (self.shape[0],)

            y_arg = out
            if out is not None and other_originally_2d:
                y_arg = out.reshape(-1)  # (n,1) → (n,) view of the caller's buffer
            output = spmv(A, x, y_arg)

            if other_originally_2d and out is None:
                output = output.reshape((-1, 1))
            elif out is not None:
                output = out
            return output
        elif isinstance(other, csr_array):
            if out is not None:
                raise ValueError("Cannot provide out for CSRxCSR matmul.")
            assert self.shape[1] == other.shape[0]
            return spgemm_csr_csr_csr(*cast_to_common_type(self, other))
        else:
            raise NotImplementedError

    def dot_local(self, x, out=None):
        """SpMV on this rank's row block only (y stays row-sharded) — what the reference's
        spmv_microbenchmark measures without --repartition.  Device tensors: no collective at all.
        Host x / host out: x is uploaded in 1/G slices + one NVLink all-gather, and only this rank's
        rows of y come back (out has blk.nrows entries)."""
        from ._device import empty

        blk = self._block()
        if not _is_dev(x):
            # host x (replicated on every rank's host) → host y block: upload 1/G of x, all-gather it
            # over NVLink, multiply, read back only this rank's rows
            if dist.world_size() == 1:
                return spmv(self, x, out)
            x_dev = _x_to_device_dist(self, x)
            if (self._colblock(blk) is not None and isinstance(out, torch.Tensor) and not out.is_cuda
                    and out.is_contiguous() and out.dim() == 1 and out.numel() == blk.nrows
                    and out.dtype == x_dev.dtype):
                # column-blocked operand + host result: the last column block runs row chunk by row
                # chunk and finished chunks of y travel home while the next ones are computed
                self._hostpipe(blk).run(None, out, x_dev=x_dev)
                torch.cuda.current_stream().synchronize()
                return out
            y_dev = empty(blk.nrows, self.dtype)
            _spmv_block(self, blk, x_dev, y_dev)
            if out is None:
                return y_dev.cpu().numpy()
            if isinstance(out, torch.Tensor):
                out.copy_(y_dev)
            else:
                out[...] = y_dev.cpu().numpy()
            return out
        y = out if out is not None else empty(blk.nrows, self.dtype)
        _spmv_block(self, blk, x, y)
        return y

    # ------------------------------------------------------------------ structure ops
    def transpose(self, axes=None, copy=False):
        """CSR → CSR transpose (reference csr.py:512-542: expand pos to row ids, stable argsort
        by column, rebuild through the COO constructor)."""
        if axes is not None:
            raise AssertionError("axes parameter should be None")
        if self._g_data is not None and self._h_data is None:
            from ._device import ptr, stream_ptr

            nnz = int(self._g_data.numel())
            rows = torch.empty(nnz, dtype=torch.int64, device=self._g_data.device)
            N.check(
                N.load().b2s_csr_expand_rows(self.shape[0], nnz, ptr(self._g_indptr), ptr(rows), stream_ptr()),
                "csr_expand_rows",
            )
            crd = self._g_indices.to(torch.int64)
            sort_mask = torch.argsort(crd, stable=True)
            return csr_array(
                (self._g_data[sort_mask], (crd[sort_mask], rows[sort_mask])),
                shape=(self.shape[1], self.shape[0]),
                dtype=self.dtype,
                copy=False,
            )
        hd, hi, hp = self._ensure_host()
        rows_expanded = numpy.repeat(numpy.arange(self.shape[0], dtype=numpy.int64), numpy.diff(hp))
        sort_mask = numpy.argsort(hi, kind="stable")
        return csr_array(
            (hd[sort_mask], (hi[sort_mask], rows_expanded[sort_mask])),
            shape=(self.shape[1], self.shape[0]),
            dtype=self.dtype,
            copy=False,
        )

    T = property(transpose)

    def asformat(self, format, copy=False):
        if format is None or format == "csr":
            return self.copy() if copy else self
        raise NotImplementedError("Only CSR format is supported right now")

    def tocsr(self, copy=False):
        if copy:
            return self.copy().tocsr(copy=False)
        return self

    def toscipy(self):
        hd, hi, hp = self._ensure_host()
        return scipy.sparse.csr_array((hd, hi, hp), shape=self.shape)

    def __repr__(self):
        return f"<{self.shape[0]}x{self.shape[1]} b200 csr_array, dtype={self.dtype}>"


csr_matrix = csr_array


def _torch_np_dtype(t):
    from ._device import np_dtype_of

    return np_dtype_of(t)


def _counts_to_csr(nrows, ncols, count_pass, fill_pass, val_dtype, dev):
    """Shared two-pass shape of the device constructors: count → native scan → (nnz) → fill.
    Returns device (data, indices, indptr)."""
    from ._device import ptr, stream_ptr

    lib = N.load()
    indptr = torch.empty(nrows + 1, dtype=torch.int64, device=dev)
    count_pass(indptr[1:])
    ws_bytes = int(lib.b2s_scan_workspace_bytes(nrows))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    N.check(lib.b2s_scan_i64(nrows, ptr(indptr), ptr(ws), ws_bytes, stream_ptr()), "scan_i64")
    nnz = int(indptr[-1].item())     # the one host sync (the reference blocks on int(nnz) too, csr.py:130)
    narrow = ncols <= _INT32_MAX and not settings.index64()
    idx = torch.empty(nnz, dtype=torch.int32 if narrow else torch.int64, device=dev)
    dat = torch.empty(nnz, dtype=val_dtype, device=dev)
    if nnz > 0:
        fill_pass(N.B2S_I32 if narrow else N.B2S_I64, indptr, idx, dat)
    return dat, idx, indptr


def _dense_to_csr_device(dense: torch.Tensor):
    """Dense CUDA matrix → device CSR arrays (b2s_dense_to_csr_count / _fill)."""
    from ._device import np_dtype_of, ptr, stream_ptr, vt_enum

    dense = dense.detach()
    if not dense.is_contiguous():
        dense = dense.contiguous()
    nrows, ncols = int(dense.shape[0]), int(dense.shape[1])
    vt = vt_enum(np_dtype_of(dense))
    lib = N.load()

    def count(row_nnz):
        N.check(lib.b2s_dense_to_csr_count(vt, nrows, ncols, ncols, ptr(dense), ptr(row_nnz), stream_ptr()),
                "dense_to_csr_count")

    def fill(it, indptr, idx, dat):
        N.check(lib.b2s_dense_to_csr_fill(vt, it, nrows, ncols, ncols, ptr(dense), ptr(indptr), ptr(idx), ptr(dat),
                                          stream_ptr()), "dense_to_csr_fill")

    return _counts_to_csr(nrows, ncols, count, fill, dense.dtype, dense.device)


# ---------------------------------------------------------------------------- SpMV
def _x_to_device_dist(A: csr_array, x):
    """Replicated device copy of a HOST x with several ranks: every rank uploads only its 1/G slice
    over PCIe and the slices are all-gathered over NVLink (one NCCL all-gather) instead of G full
    uploads of the same vector."""
    from ._device import empty, torch_dtype

    G, r = dist.world_size(), dist.rank()
    m = A.shape[1]
    xh = x if isinstance(x, torch.Tensor) else torch.from_numpy(numpy.ascontiguousarray(x))
    if xh.dtype != torch_dtype(A.dtype):
        xh = xh.to(torch_dtype(A.dtype))
    cb = dist.row_block_bounds(m, G)
    x_dev = empty(m, A.dtype)
    c0, c1 = int(cb[r]), int(cb[r + 1])
    if c1 > c0:
        x_dev[c0:c1].copy_(xh[c0:c1], non_blocking=True)
    dist.allgather_into(x_dev, cb)
    return x_dev


def _spmv_block(A: csr_array, blk: _RowBlock, x_dev, y_dev):
    """y_dev[0:blk.nrows] = A[blk.r0:blk.r1, :] @ x_dev   (one native launch sequence)."""
    from ._device import spmv as _spmv, vt_enum

    cb = A._colblock(blk)
    if cb is not None:
        cb.spmv(x_dev, y_dev)
        return
    plan = A._plan(blk)
    _spmv(vt_enum(A.dtype), blk.itype, blk.nrows, A.shape[1], blk.nnz, blk.indptr, blk.indices, blk.data,
          x_dev, y_dev, plan=plan, variant=settings.spmv_variant())


def _bcast_ok(blk: _RowBlock) -> bool:
    """the fused SpMV+all-gather needs the TMA pipe kernel: 16-byte aligned arrays"""
    return all(t.data_ptr() % 16 == 0 for t in (blk.indptr, blk.indices, blk.data))


def spmv(A: csr_array, x, y=None):
    """y = A @ x.  Replaces the reference's ``spmv`` task launch (csr.py:562-593): the row
    block of this rank is computed by the sm_90a kernel; with more than one rank the blocks
    are all-gathered so that y is replicated like x.

    numpy in → numpy out (H2D of x, D2H of y); CUDA tensor in → CUDA tensor out."""
    from ._device import empty, to_device, to_host

    blk = A._block()
    host_io = not _is_dev(x)
    G = dist.world_size()
    n = A.shape[0]
    if G == 1 and host_io and A._colblock(blk) is not None:
        # host x and y + column-blocked operand: 2-D (row chunk x column block) pipeline — slice b+1 of
        # x is uploaded while block b runs, finished row chunks of y travel back while later chunks are
        # still being computed (_device.HostPipe)
        from ._device import torch_dtype

        xh = x if isinstance(x, torch.Tensor) else torch.from_numpy(numpy.ascontiguousarray(x))
        y_t = None
        if y is None:
            y_t = torch.empty(n, dtype=torch_dtype(A.dtype))
        elif isinstance(y, torch.Tensor) and not y.is_cuda and y.is_contiguous() and y.dim() == 1:
            y_t = y
        elif isinstance(y, numpy.ndarray) and y.flags.c_contiguous and y.ndim == 1:
            y_t = torch.from_numpy(y)
        if (y_t is not None and xh.dtype == torch_dtype(A.dtype) and y_t.dtype == xh.dtype and xh.dim() == 1
                and xh.is_contiguous()):
            A._hostpipe(blk).run(xh, y_t)
            torch.cuda.current_stream().synchronize()      # host memory is handed back: copies must be complete
            if y is not None:
                return y
            return y_t.numpy()
    if G == 1:
        x_dev = to_device(x, dtype=A.dtype)
        if y is not None and _is_dev(y) and y.is_contiguous():
            y_dev = y
        else:
            y_dev = empty(n, A.dtype)
        _spmv_block(A, blk, x_dev, y_dev)
    else:
        x_dev = _x_to_device_dist(A, x) if host_io else to_device(x, dtype=A.dtype)
        bounds = A.row_bounds()
        from ._device import torch_dtype

        # collective decision (same on every rank): symmetric memory available or not.  Two buffers
        # are used in turn: the closing barrier of call k orders every peer's reads of buffer k%2
        # (call k-2's result) before anyone writes it again, so no opening barrier is needed.
        own = dist.symm_of(y) if y is not None else None
        if own is not None:
            # the caller's out= lives in symmetric memory (dist.replicated_empty): the kernel stores into
            # every rank's copy of it directly.  The caller may reuse it call after call, so an opening
            # barrier orders the peers' reads of the previous content before anyone overwrites it.
            sv = own
            sv.barrier()
        else:
            sv = dist.symm_vector_alternating(n, torch_dtype(A.dtype), "spmv_y")
        if sv is not None:
            # fused SpMV + all-gather: y stores go to every rank's replicated buffer over NVLink
            from ._device import spmv_bcast, vt_enum

            local = sv.t[blk.r0 : blk.r1]
            if blk.nnz > 0 and A._colblock(blk) is not None:
                A._colblock(blk).spmv(x_dev, local, peer_ptrs=sv.peer_ptrs(blk.r0))
            elif blk.nnz > 0 and _bcast_ok(blk):
                spmv_bcast(vt_enum(A.dtype), blk.itype, blk.nrows, A.shape[1], blk.nnz, blk.indptr,
                           blk.indices, blk.data, x_dev, local, sv.peer_ptrs(blk.r0), A._plan(blk))
            else:
                # rare: empty block or unaligned user slices → local kernel + explicit peer copies
                _spmv_block(A, blk, x_dev, local)
                for g in range(G):
                    if g != dist.rank() and blk.nrows > 0:
                        sv.h.get_buffer(g, (n,), sv.t.dtype)[blk.r0 : blk.r1].copy_(local)
            sv.barrier()   # every block has landed everywhere
            if own is not None:
                y_dev = y
            elif y is not None and _is_dev(y) and y.is_contiguous():
                y.copy_(sv.t)
                y_dev = y
            else:
                y_dev = sv.t if y is not None else sv.t.clone()
        else:
            if y is not None and _is_dev(y) and y.is_contiguous():
                y_dev = y
            else:
                y_dev = empty(n, A.dtype)
            _spmv_block(A, blk, x_dev, y_dev[blk.r0 : blk.r1])
            dist.allgather_into(y_dev, bounds)
    if y is not None:
        if _is_dev(y):
            if y_dev is not y:
                y.copy_(y_dev)
            return y
        if isinstance(y, torch.Tensor):
            y.copy_(y_dev)  # direct D2H (no staging copy when y is pinned)
            return y
        y[...] = to_host(y_dev)
        return y
    return to_host(y_dev) if host_io else y_dev


# ---------------------------------------------------------------------------- SpGEMM
def _full_device_csr(B: csr_array):
    """Whole matrix on this rank's device (B of A@B is replicated: SURVEY §8e)."""
    if B._B_full is not None:
        return B._B_full
    from ._device import ptr, stream_ptr, to_device

    if dist.world_size() == 1:
        blk = B._block()
        B._B_full = (blk.indptr, blk.indices, blk.data)
        return B._B_full
    narrow = B._narrow_ok()
    if B._g_data is None and B._h_data is None:
        B._gather_global()       # row-sharded B (e.g. the result of an earlier distributed SpGEMM)
    if B._g_data is not None:
        idx = B._g_indices
        if narrow and idx.dtype == torch.int64:
            idx32 = torch.empty(idx.numel(), dtype=torch.int32, device=idx.device)
            N.check(N.load().b2s_cast_i64_to_i32(idx.numel(), ptr(idx), ptr(idx32), stream_ptr()), "cast")
            idx = idx32
        B._B_full = (B._g_indptr, idx, B._g_data)
    else:
        hd, hi, hp = B._ensure_host()
        B._B_full = (to_device(hp), to_device(hi.astype(numpy.int32) if narrow else hi), to_device(hd))
    return B._B_full


def spgemm_csr_csr_csr(A: csr_array, B: csr_array) -> csr_array:
    """C = A @ B (reference csr.py:598-748).  Row block of A x replicated B → row block of C
    (symbolic → scan → numeric on the device); with several ranks the C blocks are
    all-gathered(v) into a replicated C."""
    from ._device import ptr, require_cuda, stream_ptr, vt_enum

    dev = require_cuda()
    lib = N.load()
    blk = A._block()
    b_ptr, b_idx, b_dat = _full_device_csr(B)
    a_idx = blk.indices
    # both operands must use the same index width
    if a_idx.dtype != b_idx.dtype:
        a_idx = a_idx.to(torch.int64)
        b_idx = b_idx.to(torch.int64)
    itype = N.B2S_I32 if a_idx.dtype == torch.int32 else N.B2S_I64
    nA, kA, nB = blk.nrows, A.shape[1], B.shape[1]
    nnzB = int(b_dat.numel())
    import os as _os
    import time as _time

    _timing = _os.environ.get("B2S_SPGEMM_TIMING") is not None   # phase timings (adds syncs)

    def _tick(label, t_prev):
        if not _timing:
            return t_prev
        torch.cuda.synchronize()
        now = _time.perf_counter()
        print(f"[spgemm] {label}: {(now - t_prev) * 1e3:.3f} ms")
        return now

    _t = _tick("start", _time.perf_counter())
    ws_bytes = int(lib.b2s_spgemm_workspace_bytes(nA, blk.nnz, nB))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    c_ptr = torch.empty(nA + 1, dtype=torch.int64, device=dev)
    nnzC, products = c_int64(0), c_int64(0)
    N.check(
        lib.b2s_spgemm_symbolic(itype, nA, kA, nB, ptr(blk.indptr), ptr(a_idx), blk.nnz, ptr(b_ptr), ptr(b_idx),
                                nnzB, ptr(c_ptr), ptr(ws), ws_bytes, byref(nnzC), byref(products), stream_ptr()),
        "spgemm_symbolic",
    )
    _t = _tick("alloc ws + symbolic", _t)
    c_idx = torch.empty(nnzC.value, dtype=a_idx.dtype, device=dev)
    c_dat = torch.empty(nnzC.value, dtype=blk.data.dtype, device=dev)
    _t = _tick("alloc C", _t)
    N.check(
        lib.b2s_spgemm_numeric(vt_enum(A.dtype), itype, nA, kA, nB, ptr(blk.indptr), ptr(a_idx), ptr(blk.data),
                               blk.nnz, ptr(b_ptr), ptr(b_idx), ptr(b_dat), nnzB, ptr(c_ptr), ptr(c_idx),
                               ptr(c_dat), ptr(ws), ws_bytes, stream_ptr()),
        "spgemm_numeric",
    )
    _t = _tick("numeric", _t)
    shape = (A.shape[0], B.shape[1])
    G = dist.world_size()
    if G == 1:
        C = csr_array._from_parts(shape, A.dtype, g=(c_dat, c_idx, c_ptr))
        C._blk = _RowBlock(0, shape[0], c_ptr, c_idx, c_dat)
    else:
        # row-sharded C, as upstream (spgemm_csr_csr_csr.cu:43-62,317-332): every rank keeps its row
        # block; only the per-rank nnz is exchanged (→ global offsets).  The replicated arrays are
        # gathered on request (C.gather(), C.indices / .data / .indptr, or C as the B of a later A@B).
        C = csr_array._from_parts(shape, A.dtype, bounds=A.row_bounds(),
                                  blk=_RowBlock(blk.r0, blk.r1, c_ptr, c_idx, c_dat))
        C._nnz_per_rank = dist.allgather_i64(int(nnzC.value), dev)
        prod_all = dist.allgather_i64(int(products.value), dev)
        products = c_int64(int(prod_all.sum()))
    C.indices_sorted = True
    C._last_products = int(products.value)
    return C
