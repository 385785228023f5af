"""Iterative solvers and the LinearOperator family
(reference legate_sparse/linalg.py:85-668).

The solver loops keep every vector in HBM as a CUDA tensor and every scalar (rho, pq, …) as
a 1-element device array, exactly like the reference keeps them as Legate futures
(linalg.py:440-445): the host only synchronises at the convergence test every
``conv_test_iters`` iterations (linalg.py:529-533).

Array convention: if ``b`` is a numpy array the result, the callback argument and the
vectors handed to user-defined ``matvec`` callables are numpy arrays (drop-in for scipy
code); if ``b`` is a CUDA ``torch.Tensor`` everything stays on the device.

Fast path: ``cg`` with a ``csr_array`` A and no preconditioner runs three fused kernels per
iteration (SpMV+p·q, x/r update + r·r, p update) instead of the reference's
1 SpMV + 2 dots + 3 axpby + 1 copy; the recurrence and its floating-point operations are the
same.  Set ``LEGATE_SPARSE_CG_UNFUSED=1`` to run the op-for-op reference sequence.
"""
from __future__ import annotations

import inspect
import os
import warnings

import numpy as np
import torch

from . import dist
from . import _native as N


def _is_dev(x):
    return isinstance(x, torch.Tensor) and x.is_cuda


def _np_dtype(x):
    from ._device import np_dtype_of

    return np_dtype_of(x) if isinstance(x, torch.Tensor) else np.dtype(x.dtype)


# ======================================================================= LinearOperator
class LinearOperator:
    """Common interface for matrix-vector products (scipy.sparse.linalg.LinearOperator
    shape; reference linalg.py:85-302).  Subclasses implement ``_matvec(x, out=None)``."""

    ndim = 2

    def __new__(cls, *args, **kwargs):
        if cls is LinearOperator:
            # Operate as _CustomLinearOperator factory.
            return super(LinearOperator, cls).__new__(_CustomLinearOperator)
        obj = super(LinearOperator, cls).__new__(cls)
        if type(obj)._matvec == LinearOperator._matvec and type(obj)._matmat == LinearOperator._matmat:
            warnings.warn(
                "LinearOperator subclass should implement at least one of _matvec and _matmat.",
                category=RuntimeWarning,
                stacklevel=2,
            )
        return obj

    def __init__(self, dtype, shape):
        if dtype is not None:
            dtype = np.dtype(dtype)
        self.dtype = dtype
        self.shape = tuple(shape)

    def _init_dtype(self):
        """Called from subclasses at the end of __init__: infer dtype from matvec(zeros)."""
        if self.dtype is None:
            v = np.zeros(self.shape[-1])
            self.dtype = _np_dtype(self.matvec(v))

    def _matmat(self, X):
        raise NotImplementedError

    def _matvec(self, x, out=None):
        raise NotImplementedError

    def matvec(self, x, out=None):
        M, Ncols = self.shape
        if tuple(x.shape) != (Ncols,) and tuple(x.shape) != (Ncols, 1):
            raise ValueError("dimension mismatch")
        y = self._matvec(x, out=out)
        if not isinstance(y, torch.Tensor):
            y = np.asarray(y)
        if x.ndim == 1:
            y = y.reshape((M,))
        elif x.ndim == 2:
            y = y.reshape(M, 1)
        else:
            raise ValueError("invalid shape returned by user-defined matvec()")
        return y

    def _rmatvec(self, x, out=None):
        raise NotImplementedError

    def rmatvec(self, x, out=None):
        M, Ncols = self.shape
        if tuple(x.shape) != (M,) and tuple(x.shape) != (M, 1):
            raise ValueError("dimension mismatch")
        y = self._rmatvec(x, out=out)
        if not isinstance(y, torch.Tensor):
            y = np.asarray(y)
        if x.ndim == 1:
            y = y.reshape(Ncols)
        elif x.ndim == 2:
            y = y.reshape(Ncols, 1)
        else:
            raise ValueError("invalid shape returned by user-defined rmatvec()")
        return y


class _CustomLinearOperator(LinearOperator):
    """Linear operator defined by user callables (reference linalg.py:307-363): the ``out=``
    keyword is forwarded only when the callable's signature has it."""

    def __init__(self, shape, matvec, rmatvec=None, matmat=None, dtype=None, rmatmat=None):
        super().__init__(dtype, shape)
        self.args = ()
        self.__matvec_impl = matvec
        self.__rmatvec_impl = rmatvec
        self._matvec_has_out = self._has_out(self.__matvec_impl)
        self._rmatvec_has_out = self._has_out(self.__rmatvec_impl)
        self._init_dtype()

    def _matvec(self, x, out=None):
        if self._matvec_has_out:
            return self.__matvec_impl(x, out=out)
        if out is None:
            return self.__matvec_impl(x)
        res = self.__matvec_impl(x)
        _assign(out, res)
        return out

    def _rmatvec(self, x, out=None):
        func = self.__rmatvec_impl
        if func is None:
            raise NotImplementedError("rmatvec is not defined")
        if self._rmatvec_has_out:
            return func(x, out=out)
        if out is None:
            return func(x)
        _assign(out, func(x))
        return out

    def _has_out(self, o):
        if o is None:
            return False
        return "out" in inspect.signature(o).parameters


def _assign(out, res):
    """out[:] = res across numpy / torch combinations."""
    if isinstance(out, torch.Tensor):
        if not isinstance(res, torch.Tensor):
            res = torch.from_numpy(np.ascontiguousarray(res))
        out.copy_(res.reshape(out.shape))
    else:
        if isinstance(res, torch.Tensor):
            res = res.detach().cpu().numpy()
        out[:] = np.asarray(res).reshape(out.shape)


class _SparseMatrixLinearOperator(LinearOperator):
    """Wraps a sparse matrix; caches the conjugate transpose (reference linalg.py:369-387)."""

    def __init__(self, A):
        self.A = A
        self.AH = None
        super().__init__(A.dtype, A.shape)

    def _matvec(self, x, out=None):
        return self.A.dot(x, out=out)

    def _rmatvec(self, x, out=None):
        if self.AH is None:
            self.AH = self.A.T.conj(copy=False)
        return self.AH.dot(x, out=out)


class IdentityOperator(LinearOperator):
    def __init__(self, shape, dtype=None):
        super().__init__(dtype, shape)

    def _matvec(self, x, out=None):
        if out is not None:
            _assign(out, x)
            return out
        return x.clone() if isinstance(x, torch.Tensor) else x.copy()

    def _rmatvec(self, x, out=None):
        return self._matvec(x, out=out)


def make_linear_operator(A):
    if isinstance(A, LinearOperator):
        return A
    return _SparseMatrixLinearOperator(A)


# ======================================================================= cg_axpby
def _scalar_dev(a, dtype):
    """0-d / 1-element array or python scalar → 1-element device tensor of `dtype`."""
    from ._device import to_device, torch_dtype

    if _is_dev(a):
        a = a.reshape(-1)[:1]
        return a if a.dtype == torch_dtype(dtype) else a.to(torch_dtype(dtype))
    return to_device(np.asarray(a, dtype=dtype).reshape(-1)[:1])


def cg_axpby(y, x, a, b, isalpha=True, negate=False):
    """y = alpha*x + beta*y with alpha or beta = (+/-) a/b computed ON THE DEVICE from the
    1-element arrays a, b (reference linalg.py:433-451, AXPBY task axpby.cu:25-47):
    isalpha → y = (a/b)*x + y, else y = x + (a/b)*y.  Updates y in place and returns it."""
    from ._device import axpby as _axpby
    from ._device import to_device, to_host

    dt = _np_dtype(y)
    if _is_dev(y):
        _axpby(y, to_device(x, dtype=dt), _scalar_dev(a, dt), _scalar_dev(b, dt), isalpha, negate)
        return y
    yd = to_device(y)
    _axpby(yd, to_device(x, dtype=dt), _scalar_dev(a, dt), _scalar_dev(b, dt), isalpha, negate)
    y[...] = to_host(yd).reshape(y.shape)
    return y


def _get_atol_rtol(b_norm, tol=None, atol=0.0, rtol=1e-5):
    rtol = float(tol) if tol is not None else rtol
    if atol is None:
        atol = rtol
    atol = max(float(atol), float(rtol) * float(b_norm))
    return atol, rtol


# ======================================================================= device-side operators
class _DevOp:
    """Uniform device-side view ``apply(x_dev, out_dev) -> y_dev`` of a LinearOperator."""

    def __init__(self, op, numpy_mode):
        self.op = op
        self.numpy_mode = numpy_mode
        self.is_identity = isinstance(op, IdentityOperator)
        self.csr = op.A if isinstance(op, _SparseMatrixLinearOperator) else None

    def apply(self, x, out=None):
        from ._device import to_device, to_host

        if self.is_identity:
            if out is None:
                return x.clone()
            out.copy_(x)
            return out
        if self.csr is not None:
            from .csr import spmv

            A = self.csr
            if _np_dtype(x) != A.dtype:
                A = A.astype(np.result_type(A.dtype, _np_dtype(x)), copy=False)
                self.csr = A
            return spmv(A, x, out)
        if self.numpy_mode:
            y = self.op.matvec(to_host(x))
            y = to_device(y, dtype=_np_dtype(x))
            if out is None:
                return y
            out.copy_(y)
            return out
        y = self.op.matvec(x, out=out)
        if out is not None and y is not out:
            out.copy_(y)
            return out
        return y


def _vec_in(v, dtype):
    """user vector → contiguous 1-D device tensor of dtype (copy)."""
    from ._device import to_device

    return to_device(v, dtype=dtype).reshape(-1)


def _vec_out(t, like):
    from ._device import to_host

    if _is_dev(like):
        return t.reshape(like.shape) if like.ndim == 2 else t
    h = to_host(t)
    if isinstance(like, torch.Tensor):
        return torch.from_numpy(h).reshape(like.shape)
    return h.reshape(like.shape) if like.ndim == 2 else h


# ======================================================================= CG
def cg(
    A,
    b,
    x0=None,
    tol=None,
    maxiter=None,
    M=None,
    callback=None,
    atol=0.0,
    rtol=1e-5,
    conv_test_iters=25,
):
    """Preconditioned conjugate gradient (reference linalg.py:465-535; returns ``(x, iters)``
    — NOT scipy's ``(x, info)`` — and tests convergence only every ``conv_test_iters``
    iterations and at ``maxiter-1``)."""
    from . import _device as D

    assert len(b.shape) == 1 or (len(b.shape) == 2 and b.shape[1] == 1)
    assert len(A.shape) == 2 and A.shape[0] == A.shape[1]

    numpy_mode = not _is_dev(b)
    A_op = make_linear_operator(A)
    dtype = np.result_type(A_op.dtype if A_op.dtype is not None else np.float64, _np_dtype(b))
    if dtype not in (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.complex64), np.dtype(np.complex128)):
        dtype = np.dtype(np.float64)

    n = b.shape[0]
    b_dev = D.to_device(b, dtype=dtype).reshape(-1)
    bnrm2 = float(D.nrm2(b_dev).item())
    atol, _ = _get_atol_rtol(bnrm2, tol, atol, rtol)
    if maxiter is None:
        maxiter = n * 10

    M_op = IdentityOperator(A_op.shape, dtype=A_op.dtype) if M is None else make_linear_operator(M)
    Ad, Md = _DevOp(A_op, numpy_mode), _DevOp(M_op, numpy_mode)

    x = D.zeros(n, dtype) if x0 is None else _vec_in(x0, dtype).clone()

    fused_ok = (
        Ad.csr is not None
        and Md.is_identity
        and os.environ.get("LEGATE_SPARSE_CG_UNFUSED", "0") in ("0", "")
        and Ad.csr.dtype == dtype
    )
    if fused_ok:
        x, iters = _cg_fused(Ad.csr, b_dev, x, dtype, atol, maxiter, callback, conv_test_iters, numpy_mode)
        return _vec_out(x, b), iters

    # ---- op-for-op reference sequence (any operator / preconditioner) ----
    p = D.zeros(n, dtype)
    r = b_dev - Ad.apply(x)  # b - A x0
    iters = 0
    rho = D.zeros(1, dtype)
    rho1 = D.zeros(1, dtype)
    pq = D.zeros(1, dtype)
    z = None
    q = None
    while iters < maxiter:
        z = Md.apply(r, out=z)
        rho1, rho = rho, rho1
        D.dot(r, z, out=rho)
        if iters == 0:
            p.copy_(z)
        else:
            # p = z + (rho/rho1) p
            D.axpby(p, z, rho, rho1, False, False)
        q = Ad.apply(p, out=q)
        D.dot(p, q, out=pq)
        D.axpby(x, p, rho, pq, True, False)   # x += (rho/pq) p
        D.axpby(r, q, rho, pq, True, True)    # r -= (rho/pq) q
        iters += 1
        if callback is not None:
            callback(D.to_host(x) if numpy_mode else x)
        if (iters % conv_test_iters == 0 or iters == (maxiter - 1)) and float(D.nrm2(r).item()) < atol:
            break
    return _vec_out(x, b), iters


_cg_profile: list = []   # (iterations, device ms) per graph replay of the last solve (LEGATE_SPARSE_CG_PROFILE=1)


def _prof_begin(prof):
    if prof is None:
        return None
    e0 = torch.cuda.Event(enable_timing=True)
    e0.record()
    return e0


def _prof_end(prof, e0, n):
    if prof is None:
        return
    e1 = torch.cuda.Event(enable_timing=True)
    e1.record()
    prof.append((n, e0, e1))


def cg_profile():
    """[(iterations, device milliseconds)] per CUDA-graph replay of the last fused CG solve that ran
    with LEGATE_SPARSE_CG_PROFILE=1 (CUDA events on the launching stream)."""
    torch.cuda.synchronize()
    return [(n, e0.elapsed_time(e1)) for (n, e0, e1) in _cg_profile]


def _halo_ranges(blk, device):
    """Per peer (rank order, self skipped): the slice [lo, hi) of MY row block that the peer's rows
    touch — the [min col, max col] image of ITS rows (the reference's image(crd→x, MIN_MAX),
    csr.py:591), clipped to my rows.  Collective (one all-gather of 2 integers).  None when every
    peer needs (almost) everything."""
    G = dist.world_size()
    r0, r1 = blk.r0, blk.r1
    cr = torch.tensor(list(blk.colrange()), dtype=torch.int64, device=device)
    allcr = torch.empty(2 * G, dtype=torch.int64, device=device)
    torch.distributed.all_gather_into_tensor(allcr, cr)
    allcr = allcr.cpu().numpy().reshape(G, 2)
    lo, hi = [], []
    for g in range(G):
        if g == dist.rank():
            continue
        a, b = max(int(allcr[g, 0]), r0), min(int(allcr[g, 1]) + 1, r1)
        lo.append(max(a - r0, 0))
        hi.append(max(b - r0, 0) if b > a else 0)
        if b <= a:
            lo[-1], hi[-1] = 1, 0          # empty: this peer never reads my block
    sent = sum(max(h - l, 0) for l, h in zip(lo, hi))
    if sent < (G - 1) * (r1 - r0):          # otherwise every peer needs everything
        return (lo, hi)
    return None


class _CgState:
    """Buffers, halo ranges, exchange boards and CUDA graphs of the fused CG iteration for one
    (matrix block, dtype, world size, graph length).  Cached on the matrix (`A._cg_state`): a second
    solve with the same operator replays the captured graphs from its first iteration on and pays no
    set-up (time-stepping codes solve with one matrix many times; the bench's wall clock then
    measures iterations, not graph capture)."""

    def __init__(self, A, dtype, nper):
        from . import _device as D

        self.G = G = dist.world_size()
        self.n = n = A.shape[0]
        self.blk = blk = A._block()
        self.bounds = A.row_bounds()
        self.dtype, self.nper = dtype, nper
        self.key = (id(blk), np.dtype(dtype), G, nper)
        r0, r1 = blk.r0, blk.r1
        self.plan = A._plan(blk)
        self.ncols = A.shape[1]
        self.vt = D.vt_enum(dtype)
        self.pv = dist.symm_vector(n, D.torch_dtype(dtype), "cg_p") if G > 1 else None
        self.halo, self.peer_ptrs = None, None
        if self.pv is not None:
            self.p_full = self.pv.t      # replicated p lives in symmetric memory: peers store into it
            self.p_full.zero_()
            self.pv.barrier()
            self.peer_ptrs = self.pv.peer_ptrs(r0)
            # halo exchange: peer g only needs the part of my p block inside the [min col, max col]
            # image of ITS rows (banded / stencil matrices: a few boundary rows instead of the block)
            if not isinstance(self.peer_ptrs, tuple) and os.environ.get("LEGATE_SPARSE_NO_HALO", "0") in ("0", ""):
                self.halo = _halo_ranges(blk, self.p_full.device)
        else:
            self.p_full = D.zeros(n, dtype)
        self.p_loc = self.p_full[r0:r1]
        self.q = D.empty(r1 - r0, dtype)
        self.x_loc = D.empty(r1 - r0, dtype)
        self.r = D.empty(r1 - r0, dtype)
        self.rho, self.rho1 = D.zeros(1, dtype), D.zeros(1, dtype)
        self.pq, self.rr = D.zeros(1, dtype), D.zeros(1, dtype)
        # cross-GPU scalar sums: in-kernel exchange through peer-mapped boards (one one-warp kernel
        # each, summed in rank order) instead of NCCL all-reduces; channel 0 doubles as the "every p
        # block has landed" barrier.  One sync point per dependency, no NCCL node in the graph.
        self.board = dist.scalar_board() if (G > 1 and self.pv is not None) else None
        self.token = D.zeros(1, dtype) if self.board is not None else None
        self.red_ws = D.new_reduce_ws()   # owned by this state: never allocated inside a graph capture
        self.graph1 = self.graphN = None
        self.graph_failed = False

    def body(self):
        """one CG iteration on fixed buffers (capturable in a CUDA graph)"""
        from . import _device as D

        blk, G = self.blk, self.G
        if self.pv is not None:
            # no barrier needed before overwriting p_full: the reduction of rr at the end of the
            # previous iteration already orders every rank's SpMV (the reader of p_full) before this point
            if self.halo is not None:
                D.cg_pupdate_halo(self.p_loc, self.r, self.rho, self.rho1, self.peer_ptrs, self.halo[0], self.halo[1])
            else:
                D.cg_pupdate_bcast(self.p_loc, self.r, self.rho, self.rho1, self.peer_ptrs)   # p block → every rank
            if self.board is not None:
                self.board.allreduce(self.token, 0)               # all blocks have landed (flag exchange)
            else:
                self.pv.barrier()
        else:
            D.cg_pupdate(self.p_loc, self.r, self.rho, self.rho1)
            if G > 1:
                dist.allgather_into(self.p_full, self.bounds)
        fuse = self.board is not None and os.environ.get("LEGATE_SPARSE_CG_NO_FUSED_EXCHANGE", "0") in ("0", "")
        if self.plan is not None:
            # several ranks: the p.q partials are exchanged inside the dot's final reduction kernel
            D.spmv_dot(self.vt, blk.itype, blk.nrows, self.ncols, blk.nnz, blk.indptr, blk.indices, blk.data,
                       self.p_full, self.q, self.p_loc, self.plan, self.pq,
                       board=self.board if fuse else None, channel=1)
        else:  # empty block
            self.q.zero_()
            self.pq.zero_()
        if self.board is not None and (not fuse or self.plan is None):
            self.board.allreduce(self.pq, 1)
        elif self.board is None:
            dist.allreduce_sum_(self.pq)
        if fuse:
            # ... and the r.r partials inside cg_update's last CTA (rho1 <- rho ; rho <- sum(rr) there too)
            D.cg_update(self.x_loc, self.r, self.p_loc, self.q, self.rho, self.pq, self.rr, ws=self.red_ws,
                        board=self.board, channel=2, cur_out=self.rho, prev_out=self.rho1)
            return
        D.cg_update(self.x_loc, self.r, self.p_loc, self.q, self.rho, self.pq, self.rr, ws=self.red_ws)
        if self.board is not None:
            self.board.allreduce(self.rr, 2, cur_out=self.rho, prev_out=self.rho1)   # rho1 <- rho ; rho <- sum(rr)
        else:
            dist.allreduce_sum_(self.rr)
            self.rho1.copy_(self.rho)   # old rho → rho1 ; new rho = rr  (z == r)
            self.rho.copy_(self.rr)

    def capture(self, want_n):
        """CUDA graphs of the body: one iteration, and `nper` iterations back to back (between two
        convergence tests the host has nothing to say, so one replay = 25 iterations and the loop is
        insensitive to host-side jitter).  The collectives of the body are captured with it."""
        if self.graph_failed:
            return
        try:
            if self.graph1 is None:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self.body()
                self.graph1 = g
            if want_n and self.graphN is None and self.nper > 1:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for _ in range(self.nper):
                        self.body()
                self.graphN = g
        except Exception as e:  # pragma: no cover - depends on driver / NCCL capture support
            warnings.warn(f"CUDA graph capture of the CG iteration failed ({e}); running eagerly")
            self.graph1 = self.graphN = None
            self.graph_failed = True
            torch.cuda.synchronize()


def _cg_fused(A, b_dev, x, dtype, atol, maxiter, callback, conv_test_iters, numpy_mode):
    """Identity-preconditioned CG on row-block-local vectors with fused kernels.

    Per iteration (G = number of ranks):
      p_loc  = r_loc + (rho/rho1) p_loc            cg_pupdate        (+ halo stores to the peers if G>1)
      q_loc  = A_blk p_full ; pq = <p_loc, q_loc>   spmv_csr_dot      (+ board exchange if G>1)
      x_loc += a p_loc ; r_loc -= a q_loc ; rr=<r,r> cg_update         (+ board exchange if G>1)
    The next rho is rr (z == r for the identity preconditioner)."""
    from . import _device as D
    from .csr import _spmv_block

    G = dist.world_size()
    nper = max(int(conv_test_iters), 1)
    blk = A._block()
    st = getattr(A, "_cg_state", None)
    fresh = st is None or st.key != (id(blk), np.dtype(dtype), G, nper) or st.blk is not blk
    if fresh:
        st = _CgState(A, dtype, nper)
        A._cg_state = st
    bounds = st.bounds
    r0, r1 = blk.r0, blk.r1
    cplx = dtype.kind == "c"

    # r = b - A x0 ; the solve starts from rho1 = 0 (⇒ the first p update is p = r)
    st.x_loc.copy_(x[r0:r1] if G > 1 else x)
    if bool(torch.any(x != 0).item()) if x.numel() else False:
        _spmv_block(A, blk, x, st.q)
        torch.sub(b_dev[r0:r1], st.q, out=st.r)
    else:
        st.r.copy_(b_dev[r0:r1])
    st.rho1.zero_()
    D.dot(st.r, st.r, out=st.rho)
    dist.allreduce_sum_(st.rho)
    rho, r = st.rho, st.r

    # LEGATE_SPARSE_CG_GRAPH=0 disables the CUDA graphs
    mode = os.environ.get("LEGATE_SPARSE_CG_GRAPH", "1")
    want_graph = callback is None and mode != "0"
    prof = _cg_profile if os.environ.get("LEGATE_SPARSE_CG_PROFILE", "0") not in ("0", "") else None
    if prof is not None:
        prof.clear()
    iters = 0

    def run(k):
        """advance k iterations with as few launches as possible"""
        done = 0
        while done < k:
            if want_graph and (st.graph1 is None or (st.graphN is None and maxiter - iters >= 2 * nper)) \
                    and (not fresh or iters + done >= 1) and not st.graph_failed:
                # a fresh state runs iteration 0 eagerly (lazy allocations, NCCL warm-up) and captures then
                st.capture(want_n=maxiter - iters >= 2 * nper)
            if want_graph and st.graphN is not None and k - done >= nper:
                ev = _prof_begin(prof)
                st.graphN.replay()
                _prof_end(prof, ev, nper)
                done += nper
            elif want_graph and st.graph1 is not None:
                ev = _prof_begin(prof)
                st.graph1.replay()
                _prof_end(prof, ev, 1)
                done += 1
            else:
                st.body()
                done += 1

    while iters < maxiter:
        if callback is not None:
            step = 1
        else:
            # iterations until the next convergence test (every conv_test_iters and at maxiter-1)
            step = nper - iters % nper
            if iters < maxiter - 1:
                step = min(step, maxiter - 1 - iters)
            step = max(1, min(step, maxiter - iters))
        run(step)
        iters += step
        if callback is not None:
            xf = dist.allgather_rows(st.x_loc, bounds) if G > 1 else st.x_loc
            callback(D.to_host(xf) if numpy_mode else xf.clone())
        if iters % conv_test_iters == 0 or iters == (maxiter - 1):
            if cplx:
                nr2 = D.nrm2(r) ** 2
                dist.allreduce_sum_(nr2)
                rnorm = float(torch.sqrt(nr2).item())
            else:
                rnorm = float(torch.sqrt(rho.abs()).item())
            if rnorm < atol:
                break
    if st.board is not None:
        st.board.check()
    # the iterate lives in the cached state: hand out a copy
    x_out = dist.allgather_rows(st.x_loc, bounds) if G > 1 else st.x_loc.clone()
    return x_out, iters


# ======================================================================= GMRES
def _gmres_sharded(A, b_dev, x, dtype, atol, restart, maxiter, callback, callback_type, b_norm, numpy_mode):
    """Restarted GMRES on ROW-SHARDED vectors (identity preconditioner, several ranks): every rank
    keeps rows [r0, r1) of the Krylov basis, of u and of x — the partition the reference gets from
    Legate for ``V[:, :j+1].conj().T @ u`` (linalg.py:628-631).  Per Arnoldi step: one SpMV on the
    local rows (needs the replicated v_j: one all-gather of n values), local CGS kernels, and two
    small all-reduces (the j+1 projections, the norm).  Same arithmetic as the replicated path except
    for the order of the cross-rank sums."""
    from . import _device as D
    from .csr import _spmv_block

    G = dist.world_size()
    n = A.shape[0]
    blk = A._block()
    bounds = A.row_bounds()
    r0, r1 = blk.r0, blk.r1
    nl = r1 - r0
    tdt = D.torch_dtype(dtype)
    rdt = D.torch_dtype(D.real_dtype(dtype))
    dev = b_dev.device
    ldv = (max(nl, 1) + 31) // 32 * 32
    V = torch.empty((restart, ldv), dtype=tdt, device=dev)        # local rows of the basis vectors
    H = torch.zeros((restart + 1, restart), dtype=tdt, device=dev)
    hcol = torch.empty(restart, dtype=tdt, device=dev)
    hn = torch.empty(1, dtype=rdt, device=dev)
    e = np.zeros((restart + 1,), dtype=dtype)
    # replicated operand of the SpMV.  With peer memory: a symmetric buffer into which every rank
    # copies only the slices its peers' rows touch (halo exchange over NVLink, like CG's p) + one
    # barrier; otherwise (or when every peer needs everything) an NCCL all-gather of v_j.
    zv = dist.symm_vector(n, tdt, "gmres_z")
    halo = _halo_ranges(blk, dev) if (zv is not None and os.environ.get("LEGATE_SPARSE_NO_HALO", "0") in ("0", "")) else None
    z_full = zv.t if zv is not None else torch.empty(n, dtype=tdt, device=dev)
    peers = [g for g in range(G) if g != dist.rank()]
    peer_bufs = [zv.h.get_buffer(g, (n,), tdt) for g in peers] if halo is not None else None
    u = torch.empty(nl, dtype=tdt, device=dev)
    x_loc = x[r0:r1].clone()
    b_loc = b_dev[r0:r1]

    def gather(v_loc):
        z_full[r0:r1].copy_(v_loc)
        if halo is not None:
            # the all-reduces of the previous step order every rank's SpMV (the reader of z_full)
            # before these stores
            for k, buf in enumerate(peer_bufs):
                lo, hi = halo[0][k], halo[1][k]
                if hi > lo:
                    buf[r0 + lo : r0 + hi].copy_(v_loc[lo:hi])
            zv.barrier()
        else:
            dist.allgather_into(z_full, bounds)
        return z_full

    def norm_all(sq_holder):
        """global 2-norm from the local one in sq_holder (device real scalar), in place"""
        sq_holder.mul_(sq_holder)
        dist.allreduce_sum_(sq_holder)
        sq_holder.sqrt_()

    iters = 0
    while True:
        _spmv_block(A, blk, gather(x_loc), u)                      # u = (A x)_loc
        r = b_loc - u
        D.nrm2(r, out=hn)
        norm_all(hn)
        r_norm = float(hn.item())
        if callback_type == "x":
            xf = dist.allgather_rows(x_loc, bounds)
            callback(D.to_host(xf) if numpy_mode else xf)
        elif callback_type == "pr_norm" and iters > 0:
            callback(r_norm / b_norm)
        if r_norm <= atol or iters >= maxiter:
            break
        if nl > 0:
            D.vscale_inv(r, hn, V[0, :nl])
        e[:] = 0
        e[0] = r_norm
        for j in range(restart):
            _spmv_block(A, blk, gather(V[j, :nl]), u)              # u = (A v_j)_loc
            if nl > 0:
                D.cgs_project(V, ldv, nl, j + 1, u, hcol)          # local part of V_j^H u
            else:
                hcol.zero_()
            dist.allreduce_sum_(hcol[: j + 1])
            if nl > 0:
                D.cgs_update(V, ldv, nl, j + 1, hcol, u, negate=True, nrm_out=hn)   # u -= V_j h ; hn = ||u_loc||
            else:
                hn.zero_()
            norm_all(hn)
            H[: j + 1, j] = hcol[: j + 1]
            H[j + 1, j] = hn[0]
            if j + 1 < restart and nl > 0:
                D.vscale_inv(u, hn, V[j + 1, :nl])
        y = np.linalg.lstsq(D.to_host(H), e, rcond=None)[0]       # identical on every rank
        y_dev = D.to_device(np.ascontiguousarray(y), dtype=dtype)
        if nl > 0:
            D.cgs_update(V, ldv, nl, restart, y_dev, x_loc, negate=False)   # x += V y
        iters += restart
    info = 0
    if iters == maxiter and not (r_norm <= atol):
        info = iters
    return dist.allgather_rows(x_loc, bounds), info


def gmres(
    A,
    b,
    x0=None,
    tol=None,
    restart=None,
    maxiter=None,
    M=None,
    callback=None,
    restrt=None,
    atol=0.0,
    callback_type=None,
    rtol=1e-5,
):
    """Restarted GMRES with classical Gram-Schmidt (reference linalg.py:540-668, itself the
    CuPy algorithm).  Returns ``(x, info)``.  SpMV, norms and the tall-skinny
    ``V^H u`` / ``u -= V h`` / ``x += V y`` products run on the native kernels (b2s_cgs_project /
    b2s_cgs_update / b2s_vscale_inv; the basis is stored basis-vector-major); the
    (restart+1) x restart least-squares problem is solved on the host, as upstream."""
    from . import _device as D

    assert len(b.shape) == 1 or (len(b.shape) == 2 and b.shape[1] == 1)
    assert len(A.shape) == 2 and A.shape[0] == A.shape[1]
    assert restrt is None or not restart
    if restrt is not None:
        restart = restrt

    numpy_mode = not _is_dev(b)
    A_op = make_linear_operator(A)
    n = A_op.shape[0]
    M_op = IdentityOperator(A_op.shape, dtype=A_op.dtype) if M is None else make_linear_operator(M)
    dtype = np.result_type(A_op.dtype if A_op.dtype is not None else np.float64, _np_dtype(b))
    if dtype.kind not in "fc":
        dtype = np.dtype(np.float64)
    Ad, Md = _DevOp(A_op, numpy_mode), _DevOp(M_op, numpy_mode)
    tdt = D.torch_dtype(dtype)

    b_dev = D.to_device(b, dtype=dtype).reshape(-1)
    x = D.zeros(n, dtype) if x0 is None else _vec_in(x0, dtype).clone()

    bnrm2 = float(D.nrm2(b_dev).item())
    atol, _ = _get_atol_rtol(bnrm2, tol, atol, rtol)
    b_norm = bnrm2

    if maxiter is None:
        maxiter = n * 10
    if restart is None:
        restart = 20
    restart = min(restart, n)
    if callback_type is None:
        callback_type = "pr_norm"
    if callback_type not in ("x", "pr_norm"):
        raise ValueError("Unknown callback_type: {}".format(callback_type))
    if callback is None:
        callback_type = None

    if dist.world_size() > 1 and Ad.csr is not None and Md.is_identity and Ad.csr.dtype == dtype and \
            os.environ.get("LEGATE_SPARSE_GMRES_REPLICATED", "0") in ("0", ""):
        mx, info = _gmres_sharded(Ad.csr, b_dev, x, dtype, atol, restart, maxiter, callback, callback_type, b_norm,
                                  numpy_mode)
        return _vec_out(mx, b), info

    dev = b_dev.device
    # Krylov basis, basis-vector-major (row c = v_c): every kernel streams unit-stride rows.
    # The leading dimension is padded so that each row starts 16-byte aligned (128-bit loads).
    ldv = (n + 31) // 32 * 32
    V = torch.empty((restart, ldv), dtype=tdt, device=dev)
    H = torch.zeros((restart + 1, restart), dtype=tdt, device=dev)
    hcol = torch.empty(restart, dtype=tdt, device=dev)
    hn = torch.empty(1, dtype=D.torch_dtype(D.real_dtype(dtype)), device=dev)
    e = np.zeros((restart + 1,), dtype=dtype)

    iters = 0
    while True:
        mx = Md.apply(x)
        r = b_dev - Ad.apply(mx)
        D.nrm2(r, out=hn)
        r_norm = float(hn.item())
        if callback_type == "x":
            callback(D.to_host(mx) if numpy_mode else mx)
        elif callback_type == "pr_norm" and iters > 0:
            callback(r_norm / b_norm)
        if r_norm <= atol or iters >= maxiter:
            break
        D.vscale_inv(r, hn, V[0, :n])          # v_0 = r / ||r||
        e[0] = r_norm

        # Arnoldi iteration (classical Gram-Schmidt, reference linalg.py:627-657)
        for j in range(restart):
            vj = V[j, :n]
            z = vj if Md.is_identity else Md.apply(vj)     # operators never write their input
            u = Ad.apply(z)
            if u.dtype != tdt:
                u = u.to(tdt)
            if u.data_ptr() == vj.data_ptr() or not u.is_contiguous():
                u = u.contiguous().clone()      # never update a basis row in place
            D.cgs_project(V, ldv, n, j + 1, u, hcol)        # h = V_j^H u
            D.cgs_update(V, ldv, n, j + 1, hcol, u, negate=True, nrm_out=hn)   # u -= V_j h ; hn = ||u||
            H[: j + 1, j] = hcol[: j + 1]
            H[j + 1, j] = hn[0]
            if j + 1 < restart:
                D.vscale_inv(u, hn, V[j + 1, :n])          # v_{j+1} = u / ||u||

        # least squares H y = e on the host (small), as upstream (linalg.py:658-661)
        y = np.linalg.lstsq(D.to_host(H), e, rcond=None)[0]
        y_dev = D.to_device(np.ascontiguousarray(y), dtype=dtype)
        D.cgs_update(V, ldv, n, restart, y_dev, x, negate=False)   # x += V y
        iters += restart

    info = 0
    if iters == maxiter and not (r_norm <= atol):
        info = iters
    return _vec_out(mx, b), info
