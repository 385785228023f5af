"""legate_sparse — the H100-native drop-in for the nv-legate/legate-sparse Python surface.

Same names as the reference package (reference legate_sparse/__init__.py:22-29):
``csr_array``/``csr_matrix``, ``dia_array``, ``diags``, ``random``, ``mmread``, ``linalg`` …, but every
SpMV / SpGEMM / CG vector operation is a hand-written sm_90a CUDA kernel in
``libb200sparse.so`` reached through a plain C ABI (include/b200sparse.h).  No Legate,
no cuSPARSE, no CPU fallback.
"""
from .csr import csr_array, csr_matrix  # noqa: F401
from .dia import dia_array, dia_matrix  # noqa: F401
from .module import *  # noqa: F401,F403
from .module import is_sparse_matrix, issparse, isspmatrix, isspmatrix_csr  # noqa: F401
from . import linalg  # noqa: F401
from . import dist  # noqa: F401

__version__ = "0.1.0"
