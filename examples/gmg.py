#!/usr/bin/env python
"""Geometric-multigrid-preconditioned CG for the 2-D Poisson problem — the workload of the
reference's examples/gmg.py (BASELINE config 3), written against this repo's legate_sparse:

  * Galerkin coarse operators  A_c = R A P  (two CSR x CSR SpGEMMs per level), P = R^T
    (csr_array.transpose), R = full-weighting restriction assembled through the COO constructor;
  * weighted-Jacobi smoother from A.diagonal();
  * one V-cycle per CG iteration, handed to linalg.cg as a LinearOperator preconditioner.

All vectors are CUDA tensors, so every A @ x inside the cycle is the sm_90a SpMV and the
element-wise smoother arithmetic stays on the device.

    python examples/gmg.py -n 512 -l 4
"""
import argparse
import time

from _common import poisson2d

import numpy as np
import torch

import legate_sparse as sparse
import legate_sparse.linalg as linalg


def full_weighting(nf: int):
    """Restriction from an nf x nf grid to the (nf//2) x (nf//2) grid: coarse point (I,J) sits on
    fine point (2I,2J) and averages its 3x3 neighbourhood with weights 1/4, 1/8, 1/16."""
    nc = nf // 2
    I, J = np.meshgrid(np.arange(nc), np.arange(nc), indexing="ij")
    rows, cols, vals = [], [], []
    for di, dj, w in [(0, 0, 0.25)] + [(a, b, 0.125) for a, b in ((1, 0), (-1, 0), (0, 1), (0, -1))] + \
                     [(a, b, 0.0625) for a in (-1, 1) for b in (-1, 1)]:
        fi, fj = 2 * I + di, 2 * J + dj
        ok = (fi >= 0) & (fi < nf) & (fj >= 0) & (fj < nf)
        rows.append((I * nc + J)[ok]); cols.append((fi * nf + fj)[ok]); vals.append(np.full(ok.sum(), w))
    rows, cols, vals = (np.concatenate(a) for a in (rows, cols, vals))
    return sparse.csr_array((vals, (rows.astype(np.int64), cols.astype(np.int64))), shape=(nc * nc, nf * nf)), nc


class VCycle:
    def __init__(self, A, n, levels, omega=2.0 / 3.0):
        self.levels = []
        for _ in range(levels - 1):
            if n < 4:
                break
            R, nc = full_weighting(n)
            P = (R.T * 4.0)                        # bilinear interpolation = 4 R^T
            Ac = R @ A @ P                          # Galerkin triple product: 2 SpGEMMs
            self.levels.append((A, R, P, self._dinv(A, omega)))
            A, n = Ac, nc
        self.coarse = (A, self._dinv(A, omega))

    @staticmethod
    def _dinv(A, omega):
        return torch.from_numpy(omega / A.diagonal()).cuda()

    def apply(self, r, out=None):
        z = self._cycle(0, r)
        if out is not None:
            out.copy_(z)
            return out
        return z

    def _cycle(self, k, r):
        if k == len(self.levels):
            A, dinv = self.coarse
            x = dinv * r
            for _ in range(8):                      # a few Jacobi sweeps on the coarsest grid
                x = x + dinv * (r - A @ x)
            return x
        A, R, P, dinv = self.levels[k]
        x = dinv * r                                # pre-smoothing from a zero guess
        coarse_r = R @ (r - A @ x)
        x = x + P @ self._cycle(k + 1, coarse_r)
        return x + dinv * (r - A @ x)               # post-smoothing


def solve(n, levels, rtol=1e-10, maxiter=200, verbose=True):
    A = poisson2d(sparse, n)
    b = torch.from_numpy(np.random.default_rng(0).random(n * n)).cuda()
    t0 = time.perf_counter()
    mg = VCycle(A, n, levels)
    torch.cuda.synchronize()
    t_setup = time.perf_counter() - t0
    M = linalg.LinearOperator(A.shape, matvec=mg.apply, dtype=np.float64)
    t0 = time.perf_counter()
    x, iters = linalg.cg(A, b, rtol=rtol, maxiter=maxiter, M=M, conv_test_iters=1)
    torch.cuda.synchronize()
    t_solve = time.perf_counter() - t0
    rel = float((b - A @ x).norm() / b.norm())
    if verbose:
        print(f"GMG-PCG {n}x{n}, {len(mg.levels) + 1} levels: setup {t_setup * 1e3:.1f} ms, {iters} iterations, "
              f"solve {t_solve * 1e3:.1f} ms ({t_solve / max(iters, 1) * 1e3:.3f} ms/iter), rel. residual {rel:.2e}")
    return iters, rel


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("-n", "--grid", type=int, default=256)
    ap.add_argument("-l", "--levels", type=int, default=4)
    ap.add_argument("--rtol", type=float, default=1e-10)
    ap.add_argument("-m", "--maxiter", type=int, default=200)
    a = ap.parse_args()
    solve(a.grid, a.levels, a.rtol, a.maxiter)
