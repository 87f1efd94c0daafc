"""ctypes binding of tests/fault_oracle.c: the CPU oracle with node faults.  Test infrastructure.

The library is compiled on first use into a temporary directory (the repository tree stays as it is), with the
oracle's own flags (oracle/Makefile)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import oracle_lib as O
from happysim_b200 import _abi as A

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "fault_oracle.c"), os.path.join(_ROOT, "oracle", "hs_oracle.c"),
         os.path.join(_ROOT, "include", "hs_b200.h")] + \
        [os.path.join(_ROOT, "happy-simulator_b200", "csrc", f) for f in ("hs_sampler.h", "hs_profile.h", "hs_sketch.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _SRCS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"hs_fault_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libhs_fault_oracle_{h}.so")
        if not os.path.exists(so):
            fma = ["-mfma"] if " fma " in open("/proc/cpuinfo").read() else []
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", *fma,
                                   "-pthread", "-shared", "-o", tmp, _SRCS[0], "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.hs_fault_oracle_run_range.argtypes = [C.POINTER(A.ModelDesc), C.POINTER(A.RunParams), C.POINTER(A.Outputs),
                                                C.c_uint32, C.c_uint32]
        L.hs_fault_oracle_run_range.restype = C.c_int
        _lib = L
    return _lib


def run(model, p: A.RunParams, chunk: int = 256):
    """All replicas of ``p`` on the fault oracle (a thread pool over slices of ``chunk`` replicas)."""
    d = model.desc()
    bufs, o = O.alloc_outputs(model.n_entities, p, model.sketch_layout()[2])
    n = p.n_replicas
    lib()

    def part(r0):
        assert lib().hs_fault_oracle_run_range(C.byref(d), C.byref(p), C.byref(o), r0, min(n, r0 + chunk)) == 0

    O._pool_map(part, range(0, n, chunk))
    return bufs
