"""world_size-2 gloo tests (CPU) of the N>1 host-side logic: row partitions, ragged all-gather,
the distributed SpMV assembly and the all-gather(v) of SpGEMM blocks.  The per-rank block
product is computed with the ORACLE here (the sm_90a kernel needs a GPU) — what is under
test is the partition + collective plumbing of legate_sparse.dist."""
import os
import socket

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp

from legate_sparse import dist
from tests import gen


def test_row_block_bounds_and_nnz_balance():
    assert list(dist.row_block_bounds(10, 4)) == [0, 3, 6, 9, 10]
    assert list(dist.row_block_bounds(8, 2)) == [0, 4, 8]
    assert list(dist.row_block_bounds(0, 3)) == [0, 0, 0, 0]
    assert list(dist.row_block_bounds(2, 4)) == [0, 1, 2, 2, 2]
    d, c, p = gen.powerlaw_csr(5000, 5000, max_row=2000, seed=3)
    b = dist.nnz_balanced_bounds(p, 4)
    assert b[0] == 0 and b[-1] == 5000 and np.all(np.diff(b) >= 0)
    per = np.diff(p[b])
    assert per.max() <= p[-1] / 4 + 2000 + 1  # within one (max) row of the ideal share
    eq = np.diff(p[dist.row_block_bounds(5000, 4)])
    assert per.max() <= eq.max()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, n, seed, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as td

    td.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import oracle

        assert dist.world_size() == world and dist.rank() == rank
        S = sp.random(n, n, density=0.05, format="csr", random_state=seed, dtype=np.float64)
        x = np.random.default_rng(seed).standard_normal(n)
        for bounds in (dist.row_block_bounds(n, world), dist.nnz_balanced_bounds(S.indptr, world)):
            r0, r1 = int(bounds[rank]), int(bounds[rank + 1])
            blk = S[r0:r1]
            y_loc = torch.from_numpy(oracle.spmv(blk.indptr, blk.indices, blk.data, x))
            # (a) ragged all-gather of row blocks
            y = dist.allgather_rows(y_loc, bounds)
            assert np.allclose(y.numpy(), S @ x, rtol=1e-13)
            # (b) in-place variant
            full = torch.zeros(n, dtype=torch.float64)
            full[r0:r1] = y_loc
            dist.allgather_into(full, bounds)
            assert np.allclose(full.numpy(), S @ x, rtol=1e-13)
        # (c) all-reduce of a local dot
        t = torch.tensor([float(np.dot(x[r0:r1], x[r0:r1]))], dtype=torch.float64)
        dist.allreduce_sum_(t)
        assert abs(t.item() - float(x @ x)) < 1e-9
        # (d) all-gather(v) of SpGEMM C blocks → replicated C
        cp, ci, cv = oracle.spgemm(blk.indptr, blk.indices, blk.data, S.indptr, S.indices, S.data, n)
        all_idx, counts = dist.allgather_varlen(torch.from_numpy(ci))
        all_val, _ = dist.allgather_varlen(torch.from_numpy(cv))
        all_rnz, _ = dist.allgather_varlen(torch.from_numpy(np.diff(cp)))
        gp = np.concatenate([[0], np.cumsum(all_rnz.numpy())])
        C = sp.csr_array((all_val.numpy(), all_idx.numpy(), gp), shape=(n, n))
        assert int(counts.sum()) == C.nnz
        assert np.allclose(np.asarray(C.todense()), np.asarray((S @ S).todense()), rtol=1e-12, atol=1e-13)
        # (e) the product's row-sharded result object: per-rank nnz exchange (reference
        # spgemm_csr_csr_csr.cu:43-62), global offset of the block, gather on request
        from legate_sparse.csr import _RowBlock, csr_array

        blkC = _RowBlock(r0, r1, torch.from_numpy(cp.astype(np.int64)), torch.from_numpy(ci.astype(np.int64)),
                         torch.from_numpy(cv))
        Cs = csr_array._from_parts((n, n), np.float64, bounds=np.asarray(bounds, dtype=np.int64), blk=blkC)
        assert Cs._g_data is None and Cs._h_data is None      # nothing replicated yet
        assert Cs.nnz == C.nnz
        assert Cs.nnz_offset() == int(counts[:rank].sum())
        Cc = Cs.copy()                                        # deep copy of a row-sharded matrix
        assert Cc._blk is not Cs._blk and Cc.dtype == Cs.dtype
        assert np.array_equal(Cs.indptr, gp) and np.array_equal(Cs.indices, all_idx.numpy())
        assert np.array_equal(Cs.data, all_val.numpy())
        q.put((rank, "ok"))
    except Exception as e:  # surface the failure to the parent
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        td.destroy_process_group()


@pytest.mark.parametrize("n", [101, 64])
def test_two_rank_gloo_spmv_and_spgemm_assembly(n):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, n, 5, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, msg in res:
        assert msg == "ok", f"rank {rank}: {msg}"
