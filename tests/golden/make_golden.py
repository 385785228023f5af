#!/usr/bin/env python
"""Generate the golden fixtures under tests/golden/.  Needs a checkout of the reference
(nv-legate/legate-sparse), named by LEGATE_SPARSE_REFERENCE; the fixtures it writes are committed
and are what the tests read — nothing under tests/ touches the reference at test time.

    LEGATE_SPARSE_REFERENCE=<reference checkout> python tests/golden/make_golden.py

What it produces
  reference_known_answers.json  known-answer vectors transcribed from the reference's own
                                tests / README (file:line recorded per entry)
  refrun_diags.npz              outputs of the reference's OWN gallery.diags + dia_array.tocsr
  refrun_cg.npz / refrun_gmres.npz
                                outputs of the reference's OWN linalg.cg / linalg.gmres loops
  mtx/*.mtx + mtx_expected.npz  the reference's 5 MatrixMarket test inputs re-emitted through
                                scipy.io.mmwrite (data, not source) + scipy.io.mmread results
  spmv_spgemm_scipy.npz         seeded inputs + scipy.sparse results (the BASELINE.json oracle)

How the reference's Python runs here: `legate` and `cupynumeric` are not installable
(SURVEY F13), so this script registers SHIMS before importing the reference modules
*unmodified* from the reference's legate_sparse/: cupynumeric → numpy, legate.core → a stub
namespace, legate_sparse.{config,runtime,utils,csr} → minimal stand-ins (stores are plain
numpy arrays; csr_array just records the arrays it is given).  The Legate TASK launched by
linalg.cg_axpby is replaced by the C restatement of its body (oracle.axpby,
axpby.cc:34-44).  Everything else — diags(), dia_array.transpose/_tocsr_transposed, the
LinearOperator classes, the cg and gmres loops — is the reference's code executing as is.
"""
import importlib
import json
import os
import sys
import types

import numpy as np
import scipy.io
import scipy.sparse as sp
import scipy.stats as stats

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, "..", ".."))
REF = os.environ.get("LEGATE_SPARSE_REFERENCE", "")
sys.path.insert(0, ROOT)
from oracle import oracle  # noqa: E402


# ------------------------------------------------------------------ shims
def install_shims():
    sys.modules["cupynumeric"] = np

    legate = types.ModuleType("legate")
    core = types.ModuleType("legate.core")

    def track_provenance(*a, **k):
        def deco(f):
            return f
        return deco

    core.track_provenance = track_provenance
    core.types = types.SimpleNamespace(bool_=bool, uint64=np.uint64, string_type=str)
    core.LogicalStore = np.ndarray
    for name in ("align", "broadcast", "image", "Shape", "ImageComputationHint"):
        setattr(core, name, lambda *a, **k: None)
    legate.core = core
    sys.modules["legate"] = legate
    sys.modules["legate.core"] = core

    pkg = types.ModuleType("legate_sparse")
    pkg.__path__ = [os.path.join(REF, "legate_sparse")]
    sys.modules["legate_sparse"] = pkg

    config = types.ModuleType("legate_sparse.config")
    config.SparseOpCode = types.SimpleNamespace(AXPBY=0, ZIP_TO_RECT1=1, UNZIP_RECT1=2)
    config.rect1 = None
    sys.modules["legate_sparse.config"] = config

    runtime = types.ModuleType("legate_sparse.runtime")
    runtime.runtime = types.SimpleNamespace(sparse_library=None)
    sys.modules["legate_sparse.runtime"] = runtime

    utils = types.ModuleType("legate_sparse.utils")
    utils.get_store_from_cupynumeric_array = lambda arr, copy=False: (np.array(arr) if copy else arr)
    utils.store_to_cupynumeric_array = lambda s: s
    utils.copy_store = lambda s: np.array(s)
    utils.get_storage_type = lambda s: s.dtype

    def cast_arr(arr, dtype=None):
        arr = np.array(arr) if not isinstance(arr, np.ndarray) else arr
        return arr.astype(dtype) if dtype is not None else arr

    utils.cast_arr = cast_arr
    sys.modules["legate_sparse.utils"] = utils

    csr = types.ModuleType("legate_sparse.csr")

    class csr_array:  # records what the reference hands to its CSR constructor
        def __init__(self, arg, shape=None, dtype=None, copy=False):
            if isinstance(arg, tuple) and len(arg) == 3:
                self.data, self.indices, self.indptr = (np.asarray(a) for a in arg)
                self.shape = tuple(shape)
            else:  # empty ctor
                self.shape = tuple(arg)
                self.data = np.zeros(0, dtype=shape if shape is not None else np.float64)
                self.indices = np.zeros(0, dtype=np.int64)
                self.indptr = np.zeros(self.shape[0] + 1, dtype=np.int64)
            self.dtype = dtype

    csr.csr_array = csr_array
    sys.modules["legate_sparse.csr"] = csr


def ref_modules():
    if not os.path.isdir(os.path.join(REF, "legate_sparse")):
        sys.exit("set LEGATE_SPARSE_REFERENCE to a checkout of nv-legate/legate-sparse")
    install_shims()
    gallery = importlib.import_module("legate_sparse.gallery")
    linalg = importlib.import_module("legate_sparse.linalg")

    def cg_axpby(y, x, a, b, isalpha=True, negate=False):
        # body of the AXPBY task (axpby.cc:34-44) in place of the Legate task launch
        out = oracle.axpby(y, x, np.asarray(a, dtype=np.float64).reshape(-1),
                           np.asarray(b, dtype=np.float64).reshape(-1), isalpha, negate)
        y[...] = out
        return y

    linalg.cg_axpby = cg_axpby
    return gallery, linalg


# ------------------------------------------------------------------ inputs
class Normal(stats.rv_continuous):  # same generator as tests/integration/utils/sample.py:21-37
    def _rvs(self, *args, size=None, random_state=None):
        return random_state.standard_normal(size)


def sample(N, D, density, seed):
    return sp.random(N, D, density=density, format="csr", dtype=np.float64, random_state=seed,
                     data_rvs=Normal(seed=seed)().rvs)


def spd_system(N, seed=471014, density=0.1):
    # test_cg_solve.py:24-35
    A = np.asarray(sample(N, N, density, seed).todense())
    A = 0.5 * (A + A.T)
    A = A + N * np.eye(N)
    x = np.asarray(sample(N, 1, density, seed).todense()).squeeze()
    return sp.csr_array(A), x


def poisson2d_diagonals(N):
    # examples/common.py:313-327
    diag_size = N * N - 1
    first = np.full((N - 1), -1.0)
    chunks = np.concatenate([np.zeros(1), first])
    diag_a = np.concatenate([first, np.tile(chunks, (diag_size - (N - 1)) // N)])
    diag_g = -1.0 * np.ones(N * (N - 1))
    diag_c = 4.0 * np.ones(N * N)
    return [diag_g, diag_a, diag_c, diag_a, diag_g], [-N, -1, 0, 1, N]


def main():
    gallery, linalg = ref_modules()
    out = {}

    # ---------------- known answers transcribed from the reference's tests
    known = {
        "csr_6x6": {
            "source": "tests/integration/test_csr_to_dense.py:24-42, test_unary_operation.py:24-43",
            "indptr": [0, 2, 5, 7, 9, 11, 14],
            "data": [2, 1, 5, 8, 2, 3, 4, 6, 1, 9, 4, 7, 2, 1],
            "indices": [0, 4, 0, 1, 5, 2, 3, 1, 3, 0, 4, 0, 4, 5],
            "dense": [[2, 0, 0, 0, 1, 0], [5, 8, 0, 0, 0, 2], [0, 0, 3, 4, 0, 0],
                      [0, 6, 0, 1, 0, 0], [9, 0, 0, 0, 4, 0], [7, 0, 0, 0, 2, 1]],
            "times2": [4, 2, 10, 16, 4, 6, 8, 12, 2, 18, 8, 14, 4, 2],
            "times3": [6, 3, 15, 24, 6, 9, 12, 18, 3, 27, 12, 21, 6, 3],
        },
        "readme_tridiagonal": {
            "source": "README.md:78-124 (5x5 tridiagonal A of ones, B of threes; A@B and A@ones)",
            "n": 5,
            "AB_dense": [[6, 6, 3, 0, 0], [6, 9, 6, 3, 0], [3, 6, 9, 6, 3], [0, 3, 6, 9, 6], [0, 0, 3, 6, 6]],
            "A_ones": [2, 3, 3, 3, 2],
        },
        "cg_axpby": {
            "source": "tests/integration/test_cg_axpby.py:21-42",
            "y": [2.0, 3.0], "x": [0.0, 1.0], "a": [2.0], "b": [3.0],
            "expected": {  # key = "isalpha,negate"
                "1,0": [2.0, 3.0 + 2.0 / 3.0],
                "1,1": [2.0, 3.0 - 2.0 / 3.0],
                "0,0": [0.0 + (2.0 / 3.0) * 2.0, 1.0 + (2.0 / 3.0) * 3.0],
                "0,1": [0.0 - (2.0 / 3.0) * 2.0, 1.0 - (2.0 / 3.0) * 3.0],
            },
        },
    }
    with open(os.path.join(HERE, "reference_known_answers.json"), "w") as f:
        json.dump(known, f, indent=1)

    # ---------------- reference diags / DIA→CSR
    cases = {}
    idx = 0
    for N in (12, 34):
        for nd in (3, 5):
            for dt in (np.float32, np.float64, np.complex64, np.complex128):
                offs = [x - (nd // 2) for x in range(nd)]
                A = gallery.diags([1] * nd, offs, shape=(N, N), format="csr", dtype=dt)
                cases[f"c{idx}"] = dict(kind="banded", N=N, nd=nd, dtype=np.dtype(dt).name, data=A.data,
                                        indices=A.indices, indptr=A.indptr)
                idx += 1
    for N in (6, 17):
        d, o = poisson2d_diagonals(N)
        A = gallery.diags(d, o, dtype=np.float64).tocsr()
        cases[f"c{idx}"] = dict(kind="poisson2d", N=N, nd=5, dtype="float64", data=A.data, indices=A.indices,
                                indptr=A.indptr)
        idx += 1
    # rectangular + explicit zeros inside a diagonal (dropped by dia.py:171)
    A = gallery.diags([np.array([1.0, 0.0, 3.0, 4.0]), np.array([5.0, 6.0, 0.0, 7.0])], [0, 2], shape=(4, 7),
                      format="csr", dtype=np.float64)
    cases[f"c{idx}"] = dict(kind="rect_zeros", N=4, nd=2, dtype="float64", data=A.data, indices=A.indices,
                            indptr=A.indptr)
    flat = {}
    for k, v in cases.items():
        for kk, vv in v.items():
            flat[f"{k}__{kk}"] = np.asarray(vv)
    np.savez_compressed(os.path.join(HERE, "refrun_diags.npz"), **flat)

    # ---------------- reference CG / GMRES loops
    A_sp, x_true = spd_system(200)
    b = A_sp @ x_true
    op = linalg.LinearOperator(A_sp.shape, matvec=lambda v: A_sp @ v)
    x_cg, it_cg = linalg.cg(op, b, tol=1e-8)
    x_cg1, it_cg1 = linalg.cg(op, b, tol=1e-8, conv_test_iters=1)
    # Poisson 16x16, rtol 1e-10
    d, o = poisson2d_diagonals(16)
    P = sp.diags(d, o, dtype=np.float64).tocsr()
    bp = np.random.default_rng(2).random(P.shape[0])
    opP = linalg.LinearOperator(P.shape, matvec=lambda v: P @ v)
    x_p, it_p = linalg.cg(opP, bp, rtol=1e-10)
    np.savez_compressed(
        os.path.join(HERE, "refrun_cg.npz"),
        A_data=A_sp.data, A_indices=A_sp.indices.astype(np.int64), A_indptr=A_sp.indptr.astype(np.int64),
        n=A_sp.shape[0], b=b, x_true=x_true, x_cg=x_cg, it_cg=it_cg, x_cg1=x_cg1, it_cg1=it_cg1,
        P_data=P.data, P_indices=P.indices.astype(np.int64), P_indptr=P.indptr.astype(np.int64),
        nP=P.shape[0], bp=bp, x_p=x_p, it_p=it_p,
    )
    x_g, info_g = linalg.gmres(op, b, atol=1e-5, tol=1e-5, maxiter=300)
    x_g2, info_g2 = linalg.gmres(opP, bp, rtol=1e-8, restart=30, maxiter=3000)
    np.savez_compressed(os.path.join(HERE, "refrun_gmres.npz"), x_g=x_g, info_g=info_g, x_g2=x_g2,
                        info_g2=info_g2)
    print("reference cg iters", it_cg, it_cg1, it_p, "gmres info", info_g, info_g2)

    # ---------------- MatrixMarket inputs (re-emitted data) + scipy.io.mmread results
    os.makedirs(os.path.join(HERE, "mtx"), exist_ok=True)
    exp = {}
    for name in ("test.mtx", "GlossGT.mtx", "Ragusa18.mtx", "cage4.mtx", "karate.mtx"):
        src = os.path.join(REF, "testdata", name)
        m = scipy.io.mmread(src)
        field = None
        with open(src) as f:
            hdr = f.readline().split()
        field, symmetry = hdr[3], hdr[4]
        dst = os.path.join(HERE, "mtx", name)
        mm = m
        if symmetry == "symmetric":
            mm = sp.tril(m).tocoo()
        scipy.io.mmwrite(dst, mm, field=field if field != "pattern" else "pattern", symmetry=symmetry,
                         comment="re-emitted by tests/golden/make_golden.py from the reference testdata")
        # mmwrite appends .mtx when missing; normalise
        if not os.path.exists(dst) and os.path.exists(dst + ".mtx"):
            os.rename(dst + ".mtx", dst)
        exp[name.replace(".", "_")] = np.asarray(scipy.io.mmread(dst).todense(), dtype=np.float64)
        assert np.array_equal(exp[name.replace(".", "_")], np.asarray(m.todense(), dtype=np.float64)), name
    np.savez_compressed(os.path.join(HERE, "mtx_expected.npz"), **exp)

    # ---------------- seeded SpMV / SpGEMM inputs + scipy results
    rng = np.random.default_rng(20260921)
    A = sp.random(61, 47, density=0.2, format="csr", dtype=np.float64, random_state=7,
                  data_rvs=rng.standard_normal)
    x = rng.standard_normal(47)
    S = sp.random(40, 40, density=0.15, format="csr", dtype=np.float64, random_state=8,
                  data_rvs=rng.standard_normal)
    C = (S @ S).tocsr()
    C.sort_indices()
    np.savez_compressed(
        os.path.join(HERE, "spmv_spgemm_scipy.npz"),
        A_data=A.data, A_indices=A.indices.astype(np.int64), A_indptr=A.indptr.astype(np.int64), A_shape=A.shape,
        x=x, y=A @ x, y_dense=np.asarray(A.todense()) @ x,
        S_data=S.data, S_indices=S.indices.astype(np.int64), S_indptr=S.indptr.astype(np.int64), S_shape=S.shape,
        C_data=C.data, C_indices=C.indices.astype(np.int64), C_indptr=C.indptr.astype(np.int64),
    )
    print("golden fixtures written to", HERE)


if __name__ == "__main__":
    main()
