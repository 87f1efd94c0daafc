"""ctypes binding of tests/bucket_pct_twin.c: hs_percentile.h (the kernels' bucket p50 / p99) compiled for the host.
Test infrastructure.

The library is built by oracle_lib.build (the repository tree stays as it is), with the oracle's floating-point flags
(oracle/Makefile)."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = O.build("tests/bucket_pct_twin.c")
        L.hs_cpu_bucket_percentiles.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        L.hs_cpu_bucket_percentiles.restype = None
        _lib = L
    return _lib


def percentiles(multisets):
    """[(p50, p99)] of every list of values in ``multisets`` (each non-empty), as the kernels select them."""
    sizes = [len(v) for v in multisets]
    off = np.zeros(len(sizes) + 1, np.uint64)
    off[1:] = np.cumsum(sizes)
    v = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float64) for x in multisets]) if multisets else
                             np.zeros(0), np.float64)
    out = np.zeros((len(sizes), 2), np.float64)
    lib().hs_cpu_bucket_percentiles(v.ctypes.data, off.ctypes.data, len(sizes), out.ctypes.data)
    return out
