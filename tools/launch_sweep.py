#!/usr/bin/env python
"""SpMV launch-setting sweep on one GPU: resident CTAs per SM and shared-memory carve-out of the
products consumer, the L1 policy of its gathers, and the async-gather kernel against the long-row
pass, on the three gathered-x matrices of bench.py — random 10M x 10M / 50 per row (column-blocked),
the 4096^2 Laplacian and the 8M-row power-law matrix.  The library reads B2S_SPMV_CTAS /
_CARVEOUT / _L1_ALLOC / _AGATHER at every launch, so one process sweeps them all.

    python tools/launch_sweep.py [--steps 30] [--warmup 5]

Prints one JSON line per (matrix, setting): ms per SpMV (CUDA events, mean over --steps calls);
every matrix's default setting is timed first and last to show the drift.
"""
import argparse
import json
import os
import sys

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
for p in (ROOT, os.path.join(ROOT, "legate-sparse_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import legate_sparse as sparse  # noqa: E402

KNOBS = ("B2S_SPMV_CTAS", "B2S_SPMV_CARVEOUT", "B2S_SPMV_L1_ALLOC", "B2S_SPMV_AGATHER")

SETTINGS = {
    "random": [{}, {"B2S_SPMV_CTAS": "2"}, {"B2S_SPMV_CARVEOUT": "80"}, {"B2S_SPMV_CTAS": "4", "B2S_SPMV_CARVEOUT": "80"},
               {"B2S_SPMV_CTAS": "4", "B2S_SPMV_CARVEOUT": "100"}, {"B2S_SPMV_L1_ALLOC": "1"}],
    "laplacian": [{}, {"B2S_SPMV_CTAS": "4", "B2S_SPMV_CARVEOUT": "80"}, {"B2S_SPMV_CARVEOUT": "100"},
                  {"B2S_SPMV_L1_ALLOC": "0"}],
    "powerlaw": [{}, {"B2S_SPMV_CTAS": "2"}, {"B2S_SPMV_CARVEOUT": "80"}, {"B2S_SPMV_AGATHER": "1"},
                 {"B2S_SPMV_AGATHER": "1", "B2S_SPMV_CTAS": "3"}],
}


def time_spmv(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def matrices(dev):
    import bench
    from side_bench import poisson2d_block

    A = sparse.random(10_000_000, 10_000_000, density=50 / 10_000_000, rng=bench.SEED, dtype=np.float64)
    yield "random", A, torch.rand(A.shape[1], dtype=torch.float64, device=dev)
    del A
    N = 4096
    d, i, p = poisson2d_block(N, 0, N * N, dev)
    yield "laplacian", sparse.csr_array.from_row_block(d, i, p, (N * N, N * N)), torch.rand(N * N, dtype=torch.float64, device=dev)
    vals, cols, ptr, x, _ = bench.powerlaw_matrix(8_000_000, dev)
    yield "powerlaw", sparse.csr_array((vals, cols, ptr), shape=(8_000_000, 8_000_000)), x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda")
    props = torch.cuda.get_device_properties(dev)
    for name, A, x in matrices(dev):
        y = A.dot_local(x)
        ref = y.clone()
        for k, setting in enumerate(SETTINGS[name] + [{}]):
            for key in KNOBS:
                os.environ.pop(key, None)
            os.environ.update(setting)
            ms = time_spmv(lambda: A.dot_local(x, out=y), args.steps, args.warmup)
            diff = float(((y - ref).abs().max() / ref.abs().max()).item())
            print(json.dumps({"device": props.name, "matrix": name, "setting": setting or "default",
                              "repeat": k > 0 and not setting, "ms": ms, "max_rel_diff_vs_default": diff}), flush=True)
        for key in KNOBS:
            os.environ.pop(key, None)
        del A, x, y, ref
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
