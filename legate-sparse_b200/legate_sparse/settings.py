"""Environment flags (reference legate_sparse/settings.py:22-48 keeps two env settings;
only kernel-selection switches survive here — the Legate settings machinery is out of scope).

  LEGATE_SPARSE_FAST_SPGEMM   accepted for compatibility (reference csr.py:674); the hash SpGEMM
                              has a single algorithm, so the flag is read and ignored.
  B2S_INDEX64=1               keep 64-bit column indices on the device (default: 32-bit when
                              ncols < 2**31, like scipy).
  B2S_SPMV_VARIANT=auto|rowvec|tile|pipe   (auto = pipe when a plan exists and the arrays are 16-byte
                              aligned, else tile, else rowvec)
  B2S_SPMV_TILE_NNZ=1024|2048|4096   (read by the native library)
  B2S_SPMV_LONGROWS=0|1              (read by the native library) force the long-row pass off / on
  B2S_SPMV_AGATHER=0|1               (read by the native library) 1 runs the async-gather kernel for every
                                     gathered matrix on 1024-nnz tiles; default 0: the products consumer
                                     (+ long-row pass for skewed row lengths)
  B2S_SPMV_CTAS=N, B2S_SPMV_CARVEOUT=P   (read by the native library) resident CTAs per SM / shared-memory
                                     carve-out of the pipe and async-gather kernels (sweeps)
  B2S_SPMV_NO_WINDOW=1               (read by the native library) disable TMA x-window staging
"""
import os


class _Settings:
    def fast_spgemm(self) -> bool:
        return os.environ.get("LEGATE_SPARSE_FAST_SPGEMM", "0") not in ("0", "", "false", "False")

    def index64(self) -> bool:
        return os.environ.get("B2S_INDEX64", "0") not in ("0", "", "false", "False")

    def spmv_variant(self) -> int:
        v = os.environ.get("B2S_SPMV_VARIANT", "auto").lower()
        return {"auto": 0, "rowvec": 1, "tile": 2, "pipe": 3}.get(v, 0)


settings = _Settings()
