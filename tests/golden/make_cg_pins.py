#!/usr/bin/env python
"""Pins for BASELINE config 3 (CG on the 5-point Laplacian, rtol 1e-10): run
``scipy.sparse.linalg.cg`` — the oracle north_star names — AND the reference's own ``linalg.cg``
(reference legate_sparse/linalg.py:465-535, imported unmodified behind the shims of
make_golden.py) on Poisson N x N grids, and record what a GPU run can be held to without
shipping the 8-33 MB iterates: iteration counts, TRUE relative residuals ||b - A x|| / ||b||,
||x||, and a strided sample of x.

    LEGATE_SPARSE_REFERENCE=<reference checkout> python tests/golden/make_cg_pins.py [1024 2048]
                                                         → tests/golden/scipy_cg_poisson.npz

Both solvers stop on the RECURRENCE residual; after thousands of iterations the true residual
has drifted above it (1024^2: 4.7e-10 for a 1e-10 request, for scipy and the reference alike) —
the pins record the true figures of both so that the GPU solve is compared like for like.
Run time on 8 host cores: 1024^2 ~2.5 min, 2048^2 ~20 min.
"""
import os
import sys
import time

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)


def poisson(N):
    n = N * N
    main = np.full(n, 4.0)
    off1 = np.full(n - 1, -1.0)
    off1[np.arange(1, n) % N == 0] = 0
    offn = np.full(n - N, -1.0)
    S = sp.diags([offn, off1, main, off1, offn], [-N, -1, 0, 1, N], format="csr")
    S.eliminate_zeros()
    return S


def main():
    grids = [int(a) for a in sys.argv[1:]] or [1024, 2048]
    out = {}
    path = os.path.join(HERE, "scipy_cg_poisson.npz")
    if os.path.exists(path):
        out = dict(np.load(path))
    import make_golden

    _, ref_linalg = make_golden.ref_modules()
    for N in grids:
        S = poisson(N)
        n = N * N
        b = np.random.default_rng(2).random(n)
        its = [0]

        def cb(_):
            its[0] += 1

        t = time.time()
        xs, info = spl.cg(S, b, rtol=1e-10, atol=0.0, maxiter=10 * n, callback=cb)
        t_scipy = time.time() - t
        assert info == 0
        res_s = np.linalg.norm(b - S @ xs) / np.linalg.norm(b)
        t = time.time()
        op = ref_linalg.LinearOperator(S.shape, matvec=lambda v: S @ v)
        xr, it_ref = ref_linalg.cg(op, b, rtol=1e-10)
        t_ref = time.time() - t
        xr = np.asarray(xr)
        res_r = np.linalg.norm(b - S @ xr) / np.linalg.norm(b)
        idx = np.arange(0, n, max(1, n // 4096), dtype=np.int64)
        pre = f"n{N}_"
        out.update({pre + "scipy_iters": its[0], pre + "scipy_true_relres": res_s, pre + "ref_iters": int(it_ref),
                    pre + "ref_true_relres": res_r, pre + "xnorm_scipy": np.linalg.norm(xs),
                    pre + "xnorm_ref": np.linalg.norm(xr), pre + "sample_idx": idx, pre + "x_scipy": xs[idx],
                    pre + "x_ref": xr[idx], pre + "rel_diff_scipy_vs_ref": np.linalg.norm(xs - xr) / np.linalg.norm(xs)})
        print(N, "scipy", its[0], res_s, f"{t_scipy:.0f}s", "reference", it_ref, res_r, f"{t_ref:.0f}s",
              "iterate rel diff", out[pre + "rel_diff_scipy_vs_ref"], flush=True)
        np.savez_compressed(path, **out)


if __name__ == "__main__":
    main()
