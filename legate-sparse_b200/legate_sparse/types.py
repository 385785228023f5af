"""Index / count dtypes of the public surface.

The reference fixes column coordinates to int64 and non-zero counts to uint64
(reference legate_sparse/types.py:20-25); user-visible index arrays keep those types here
(the device kernels may narrow columns to int32, see csr.py)."""
import numpy as _np

_names = {"coord_ty": "int64", "nnz_ty": "uint64", "float64": "float64", "int32": "int32", "int64": "int64",
          "uint64": "uint64"}
globals().update({alias: _np.dtype(name) for alias, name in _names.items()})
__all__ = list(_names)
