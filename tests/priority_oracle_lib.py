"""ctypes binding of tests/priority_oracle.c: the CPU oracle with PriorityQueue servers.  Test infrastructure.

The library is compiled on first use into a temporary directory (the repository tree stays as it is), with the
oracle's own flags (oracle/Makefile)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib as O
from happysim_b200 import _abi as A

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "priority_oracle.c"), os.path.join(_ROOT, "oracle", "hs_oracle.c"),
         os.path.join(_ROOT, "include", "hs_b200.h")] + \
        [os.path.join(_ROOT, "happy-simulator_b200", "csrc", f) for f in ("hs_sampler.h", "hs_profile.h", "hs_sketch.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _SRCS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"hs_priority_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libhs_priority_oracle_{h}.so")
        if not os.path.exists(so):
            fma = ["-mfma"] if " fma " in open("/proc/cpuinfo").read() else []
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", *fma,
                                   "-pthread", "-shared", "-o", tmp, _SRCS[0], "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.hs_priority_oracle_run_range.argtypes = [C.POINTER(A.ModelDesc), C.POINTER(A.RunParams), C.POINTER(A.Outputs),
                                                   C.c_uint32, C.c_uint32]
        L.hs_priority_oracle_run_range.restype = C.c_int
        L.hs_priority_oracle_run_linked.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.POINTER(C.c_int64), C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64,
                                                    C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.hs_priority_oracle_run_linked.restype = C.c_int
        _lib = L
    return _lib


def run(model, p: A.RunParams, chunk: int = 256):
    """All replicas of ``p`` on the priority oracle (a thread pool over slices of ``chunk`` replicas); the buffers
    oracle_lib.alloc_outputs lays out."""
    d = model.desc()
    bufs, o = O.alloc_outputs(model.n_entities, p, model.sketch_layout()[2])
    n = p.n_replicas
    lib()

    def part(r0):
        assert lib().hs_priority_oracle_run_range(C.byref(d), C.byref(p), C.byref(o), r0, min(n, r0 + chunk)) == 0

    O._pool_map(part, range(0, n, chunk))
    return bufs


def run_linked(lm, params: list, *, end_ns, cseed):
    """A linked run (happysim_b200.linked.LinkedModel) on the priority oracle: oracle_lib.oracle_run_linked's interface
    and replica words (partition q: ``params[q]``, the coordinator: replica word P + g * (P + 1))."""
    nP = lm.n_partitions
    descs = [m.desc() for m in lm.models]
    outs = [O.alloc_outputs(m.n_entities, p, m.sketch_layout()[2]) for m, p in zip(lm.models, params)]
    ends = np.array(lm.window_ends(end_ns), dtype=np.int64)
    link_arrs, dst_arrs = [], []
    for q in range(nP):
        arr, dst = lm.link_descs(q)
        link_arrs.append(arr)
        dst_arrs.append((C.c_uint32 * max(1, len(dst)))(*dst))
    PP = lambda T, xs: (C.POINTER(T) * nP)(*[C.cast(C.pointer(x) if not isinstance(x, C.Array) else x, C.POINTER(T)) for x in xs])
    n = params[0].n_replicas
    delivered, lost = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    rc = lib().hs_priority_oracle_run_linked(nP, PP(A.ModelDesc, descs), PP(A.RunParams, params),
                                             PP(A.Outputs, [o for _, o in outs]), PP(A.LinkDesc, link_arrs),
                                             PP(C.c_uint32, dst_arrs), ends.ctypes.data_as(C.POINTER(C.c_int64)), len(ends),
                                             lm.n_streams, cseed, 0, nP, nP + 1,
                                             delivered.ctypes.data_as(C.POINTER(C.c_uint64)),
                                             lost.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert rc == 0, rc
    return [b for b, _ in outs], delivered, lost, ends
