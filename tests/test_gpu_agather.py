"""GPU parity of the async-gather SpMV kernel (csrc/b2s_spmv_agather.cuh; written for BASELINE
config 5, reference: cusparseSpMV in src/sparse/array/csr/spmv.cu:117-152) vs scipy / the oracle.
The kernel runs on request; B2S_SPMV_AGATHER=1 selects it here so the
edge cases of its segmented sum are covered on purpose-built matrices:
rows inside one thread / one warp / several warps / several tiles, empty rows (start, middle, end,
runs longer than a tile's row-pointer stage), a partial last tile, a matrix smaller than a tile,
y += A_b x (column blocks), f32 / c64 values, int64 column ids.
Tolerance: fp64 1e-10 relative (BASELINE.json north_star); f32 3e-5."""
import numpy as np
import pytest
import scipy.sparse as sp

import legate_sparse as sparse
from oracle import oracle
from tests import gen

pytestmark = pytest.mark.gpu


def relerr(a, b):
    a, b = np.asarray(a), np.asarray(b)
    d = np.linalg.norm((a - b).ravel())
    n = np.linalg.norm(b.ravel())
    return d / n if n > 0 else d


def force(monkeypatch, on="1"):
    monkeypatch.setenv("B2S_SPMV_VARIANT", "pipe")
    monkeypatch.setenv("B2S_SPMV_AGATHER", on)
    monkeypatch.setenv("B2S_SPMV_TILE_NNZ", "1024")
    monkeypatch.setenv("B2S_SPMV_NO_WINDOW", "1")


def csr_from_deg(deg, m, rng, dtype=np.float64):
    n = len(deg)
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=indptr[1:])
    cols = rng.integers(0, m, size=int(indptr[-1])).astype(np.int64)
    data = rng.standard_normal(int(indptr[-1])).astype(dtype)
    if np.dtype(dtype).kind == "c":
        data = data + 1j * rng.standard_normal(data.shape[0]).astype(data.real.dtype)
    return sp.csr_array((data, cols, indptr), shape=(n, m))


def xvec(m, rng, dtype):
    x = rng.standard_normal(m).astype(dtype)
    if np.dtype(dtype).kind == "c":
        x = x + 1j * rng.standard_normal(m).astype(x.real.dtype)
    return x


@pytest.mark.parametrize("index64", ["0", "1"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex64])
def test_agather_irregular_rows_types(monkeypatch, dtype, index64):
    force(monkeypatch)
    monkeypatch.setenv("B2S_INDEX64", index64)
    rng = np.random.default_rng(21)
    n, m = 5000, 4100
    deg = rng.integers(0, 12, size=n)
    deg[:30] = 0            # empty rows at the start
    deg[2000:2100] = 0      # ... in the middle
    deg[-7:] = 0            # ... at the end
    deg[1234] = 3000        # spans 3-4 tiles
    deg[77] = 128           # exactly one warp's elements
    deg[78] = 1024          # exactly one tile's worth, not tile aligned
    deg[300:340] = 1        # rows that start and end inside one thread
    deg[400:420] = 4
    S = csr_from_deg(deg, m, rng, dtype)
    x = xvec(m, rng, dtype)
    A = sparse.csr_array(S)
    y = A @ x
    tol = 1e-10 if np.dtype(dtype) == np.float64 else 3e-5
    assert relerr(y, S @ x) < tol
    assert A._block().plan.info()["tile_nnz"] == 1024
    # bit-reproducible: no floating-point atomics, fixed summation order
    assert np.array_equal(y, A @ x)
    if np.dtype(dtype) == np.float64:
        assert relerr(y, oracle.spmv(S.indptr, S.indices, S.data, x)) < 1e-10
        # rows without entries are exactly zero, also when y held something before
        import torch
        out = torch.full((n,), 7.0, dtype=torch.float64, device="cuda")
        A.dot(torch.from_numpy(x).cuda(), out=out)
        assert np.all(out.cpu().numpy()[deg == 0] == 0.0)


def test_agather_matches_products_consumer(monkeypatch):
    """same matrix through the async-gather kernel and through the products consumer's long-row pass"""
    d, c, p = gen.powerlaw_csr(60000, 60000, max_row=5000, seed=11)
    S = sp.csr_array((d, c, p), shape=(60000, 60000))
    x = np.random.default_rng(4).standard_normal(60000)
    want = S @ x
    ys = {}
    for on in ("1", "0"):
        force(monkeypatch, on)
        A = sparse.csr_array(S)
        ys[on] = A @ x
        assert np.allclose(ys[on], want, rtol=1e-11, atol=1e-11), on
    assert relerr(ys["1"], ys["0"]) < 1e-13
    # default selection (no env): skewed rows take the products consumer's long-row pass (faster on H100)
    for k in ("B2S_SPMV_AGATHER", "B2S_SPMV_TILE_NNZ", "B2S_SPMV_NO_WINDOW", "B2S_SPMV_VARIANT"):
        monkeypatch.delenv(k, raising=False)
    A = sparse.csr_array(S)
    assert np.array_equal(A @ x, ys["0"])


@pytest.mark.parametrize("nnz_target", [1, 5, 1023, 1024, 1025, 3 * 1024, 3 * 1024 + 517])
def test_agather_small_and_partial_tiles(monkeypatch, nnz_target):
    force(monkeypatch)
    rng = np.random.default_rng(nnz_target)
    m = 300
    deg = []
    left = nnz_target
    while left > 0:
        k = int(min(left, rng.integers(0, 9)))
        deg.append(k)
        left -= k
    deg += [0, 0, 0]
    S = csr_from_deg(np.array(deg, dtype=np.int64), m, rng)
    assert S.nnz == nnz_target
    x = rng.standard_normal(m)
    A = sparse.csr_array(S)
    y = A @ x
    assert relerr(y, S @ x) < 1e-10
    assert np.all(y[np.array(deg) == 0] == 0.0)


def test_agather_many_rows_per_tile(monkeypatch):
    """tiles that touch more rows than the staged row-pointer window (260 entries): single-entry rows
    and long runs of empty rows (several thousand inside one tile) — the marks come from global memory"""
    force(monkeypatch)
    rng = np.random.default_rng(3)
    deg = np.ones(9000, dtype=np.int64)
    deg[1000:7000] = 0          # 6000 empty rows inside one tile
    deg[7100] = 2500
    deg = np.concatenate([deg, rng.integers(0, 3, size=4000)])
    S = csr_from_deg(deg, 5000, rng)
    x = rng.standard_normal(5000)
    A = sparse.csr_array(S)
    y = A @ x
    assert relerr(y, S @ x) < 1e-10
    assert np.all(y[deg == 0] == 0.0)


def test_agather_falls_back_when_a_tile_touches_too_many_rows(monkeypatch):
    """more than 65535 rows inside one tile cannot be marked with 16 bits: the products consumer runs"""
    force(monkeypatch)
    rng = np.random.default_rng(5)
    deg = np.zeros(200000, dtype=np.int64)
    deg[::400] = 7
    S = csr_from_deg(deg, 1000, rng)
    x = rng.standard_normal(1000)
    y = sparse.csr_array(S) @ x
    assert relerr(y, S @ x) < 1e-10


def test_agather_accumulate_column_blocks(monkeypatch):
    """y = A_0 x; y += A_1 x; ... : the accumulate flag of the kernel (forced column blocks)"""
    force(monkeypatch)
    monkeypatch.delenv("B2S_SPMV_VARIANT")          # column blocks are an AUTO-variant feature
    monkeypatch.setenv("B2S_SPMV_COLBLOCK", "3")
    d, c, p = gen.powerlaw_csr(30000, 30000, max_row=4000, seed=2)
    S = sp.csr_array((d, c, p), shape=(30000, 30000))
    S.sort_indices()
    x = np.random.default_rng(8).standard_normal(30000)
    A = sparse.csr_array((S.data, S.indices, S.indptr), shape=S.shape)
    y = A @ x
    assert A._block().colblock not in (None, False)
    assert np.allclose(y, S @ x, rtol=1e-11, atol=1e-11)


def test_agather_many_tiles_per_cta(monkeypatch):
    """one CTA per SM and ~20 tiles per CTA: the software pipeline in steady state and the flow control of the
    warp-summary buffers (a warp may run at most 8 tiles ahead of the warps that read its summaries)"""
    force(monkeypatch)
    monkeypatch.setenv("B2S_SPMV_CTAS", "1")
    d, c, p = gen.powerlaw_csr(400000, 400000, max_row=20000, seed=5)
    S = sp.csr_array((d, c, p), shape=(400000, 400000))
    import torch

    assert S.nnz > torch.cuda.get_device_properties(0).multi_processor_count * 1024 * 12
    x = np.random.default_rng(6).standard_normal(400000)
    A = sparse.csr_array(S)
    y = A @ x
    assert np.allclose(y, S @ x, rtol=1e-10, atol=1e-10)
    assert np.array_equal(y, A @ x)
