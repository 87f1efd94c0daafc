"""ctypes binding of the CPU oracle built with -DHS_ORACLE_HIGH_WATER: the same runs, plus per replica the high-water
marks of the structures the device bounds (hs_oracle.c, HS_HW_*).  Test infrastructure.

The library is compiled on first use into a temporary directory (the repository tree stays as it is), with the
oracle's own flags (oracle/Makefile); the default build that oracle_lib loads compiles none of the counters."""
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
_SRCS = [os.path.join(_ROOT, "oracle", "hs_oracle.c"), os.path.join(_ROOT, "include", "hs_b200.h")] + \
        [os.path.join(_ROOT, "happy-simulator_b200", "csrc", f) for f in ("hs_sampler.h", "hs_profile.h", "hs_sketch.h")]
FIELDS = ("now", "now_pop", "future", "outbox", "inbox")     # HS_HW_NOW .. HS_HW_INBOX, then one queue per entity
HS_W_NCAP = 24               # csrc/hs_warp_engine.cuh: now-tier entries of a general-engine replica
HS_T_KS = 4                  # csrc/hs_thread_engine.cuh: of those, the thread engine keeps this many in shared memory
HS_NOW_CAP = 8               # csrc/hs_lane_engine.cuh: the lane engine's same-timestamp queue
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _SRCS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"hs_high_water_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libhs_oracle_hw_{h}.so")
        if not os.path.exists(so):
            fma = ["-mfma"] if " fma " in open("/proc/cpuinfo").read() else []
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", *fma,
                                   "-DHS_ORACLE_HIGH_WATER", "-pthread", "-shared", "-o", tmp, _SRCS[0], "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.hs_oracle_high_water_range.argtypes = [C.POINTER(A.ModelDesc), C.POINTER(A.RunParams), C.POINTER(A.Outputs),
                                                 C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
        L.hs_oracle_high_water_range.restype = C.c_int
        L.hs_oracle_high_water_linked.argtypes = [C.c_uint32] + [C.c_void_p] * 5 + [
            C.POINTER(C.c_int64), C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32,
            C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_void_p]
        L.hs_oracle_high_water_linked.restype = C.c_int
        _lib = L
    return _lib


def _marks(rows: np.ndarray) -> dict:
    """{field: uint32[n]} and "queue": uint32[n, n_entities] from the raw rows"""
    out = {f: rows[:, k].copy() for k, f in enumerate(FIELDS)}
    out["queue"] = rows[:, len(FIELDS):].copy()
    return out


def run(model, p: A.RunParams, chunk: int = 256):
    """Every replica of ``p`` on the instrumented oracle (a thread pool over slices of ``chunk`` replicas): the output
    buffers of oracle_lib.oracle_run and the high-water marks."""
    d = model.desc()
    bufs, o = O.alloc_outputs(model.n_entities, p, model.sketch_layout()[2])
    n = p.n_replicas
    rows = np.zeros((n, len(FIELDS) + model.n_entities), np.uint32)
    lib()

    def part(r0):
        assert lib().hs_oracle_high_water_range(C.byref(d), C.byref(p), C.byref(o), r0, min(n, r0 + chunk),
                                                rows.ctypes.data_as(C.POINTER(C.c_uint32))) == 0

    O._pool_map(part, range(0, n, chunk))
    return bufs, _marks(rows)


def _linked_slice(lm, params, *, end_ns, cseed):
    nP = lm.n_partitions
    descs = [m.desc() for m in lm.models]
    outs = [O.alloc_outputs(m.n_entities, p, m.sketch_layout()[2]) for m, p in zip(lm.models, params)]
    ends = np.array(lm.window_ends(end_ns), dtype=np.int64)
    link_arrs, dst_arrs = [], []
    for q in range(nP):
        arr, dst = lm.link_descs(q)
        link_arrs.append(arr)
        dst_arrs.append((C.c_uint32 * max(1, len(dst)))(*dst))
    n = params[0].n_replicas
    rows = [np.zeros((n, len(FIELDS) + m.n_entities), np.uint32) for m in lm.models]
    PP = lambda T, xs: (C.POINTER(T) * nP)(*[C.cast(C.pointer(x) if not isinstance(x, C.Array) else x, C.POINTER(T)) for x in xs])  # noqa: E731
    delivered, lost = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    rc = lib().hs_oracle_high_water_linked(
        nP, PP(A.ModelDesc, descs), PP(A.RunParams, params), PP(A.Outputs, [o for _, o in outs]),
        PP(A.LinkDesc, link_arrs), PP(C.c_uint32, dst_arrs), ends.ctypes.data_as(C.POINTER(C.c_int64)), len(ends),
        lm.n_streams, cseed, 0, nP, nP + 1, delivered.ctypes.data_as(C.POINTER(C.c_uint64)),
        lost.ctypes.data_as(C.POINTER(C.c_uint64)),
        (C.POINTER(C.c_uint32) * nP)(*[r.ctypes.data_as(C.POINTER(C.c_uint32)) for r in rows]))
    assert rc == 0, rc
    return [b for b, _ in outs], delivered, lost, rows


def run_linked(lm, params: list, *, end_ns, cseed, chunk: int = 64):
    """oracle_lib.oracle_run_linked_parallel on the instrumented oracle (the replica words of LinkedRun): per partition
    the output buffers, delivered / lost per replica, and per partition the high-water marks."""
    n = params[0].n_replicas
    lib()

    def part(r0):
        ps = []
        for p in params:
            q = A.RunParams.from_buffer_copy(p)
            q.n_replicas, q.replica_index_base = min(n, r0 + chunk) - r0, p.replica_index_base + r0
            ps.append(q)
        return _linked_slice(lm, ps, end_ns=end_ns, cseed=cseed)

    parts = O._pool_map(part, range(0, n, chunk))
    cat = lambda xs: None if xs[0] is None else np.concatenate(xs)  # noqa: E731
    outs = [{k: cat([pt[0][q][k] for pt in parts]) for k in parts[0][0][q]} for q in range(lm.n_partitions)]
    marks = [_marks(np.concatenate([pt[3][q] for pt in parts])) for q in range(lm.n_partitions)]
    return outs, np.concatenate([pt[1] for pt in parts]), np.concatenate([pt[2] for pt in parts]), marks


def fel_slots(model, inbox_cap: int = 0) -> int:
    """S, the future-event slots of a general-engine replica: general_setup's sizing rule (csrc/hs_engine.cu) --
    24, plus 2 per Source row (a Probe's ticks come from a Source row), (c + 1) per Server with c its largest
    concurrency over the sweep cells, 64 per CachingServer, 1 per FAULT row, and the inbox -- rounded up to 32."""
    e = model.entities
    live = 24 + inbox_cap
    for i in range(model.n_entities):
        k = int(e["kind"][i])
        if k == A.HS_ENT_SOURCE:
            live += 2
        elif k == A.HS_ENT_SERVER:
            c = int(e["i0"][i])
            if model.cell_i0 is not None:
                c = max(c, int(np.asarray(model.cell_i0)[:, i].max()))
            live += c + 1
        elif k == A.HS_ENT_CACHE_SERVER:
            live += 64
        elif k == A.HS_ENT_FAULT:
            live += 1
    return (live + 31) // 32 * 32
