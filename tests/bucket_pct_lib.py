"""ctypes binding of tests/bucket_pct_twin.c: hs_percentile.h (the kernels' bucket p50 / p99) compiled for the host.
Test infrastructure.

The library is compiled on first use into a temporary directory (the repository tree stays as it is), with the
oracle's floating-point flags (oracle/Makefile)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "bucket_pct_twin.c")] + \
        [os.path.join(_ROOT, "happy-simulator_b200", "csrc", f) for f in ("hs_percentile.h", "hs_sampler.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _SRCS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"hs_bucket_pct_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libhs_bucket_pct_{h}.so")
        if not os.path.exists(so):
            fma = ["-mfma"] if " fma " in open("/proc/cpuinfo").read() else []
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", *fma,
                                   "-Wall", "-Wextra", "-Wno-unused-function", "-shared", "-o", tmp,
                                   _SRCS[0], "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
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
