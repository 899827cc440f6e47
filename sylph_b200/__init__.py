"""sylph_b200 — H100-native (sm_90a) FracMinHash sketching + containment for sylph.

The product is the CUDA shared library behind include/sylph_b200.h; this package is the thin
host-side mirror used by the tests, bench.py and Python callers.  Importing it never touches
oracle/ (the CPU restatement is test infrastructure only) and there is no CPU fallback.
"""
from ._lib import SEM_AVX2, SEM_SCALAR, SylphError  # noqa: F401
from .api import Context  # noqa: F401

__all__ = ["Context", "SEM_AVX2", "SEM_SCALAR", "SylphError"]
