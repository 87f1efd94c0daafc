"""ctypes binding of the CPU oracle built with -DHS_ORACLE_HIGH_WATER: the same runs, plus per replica the high-water
marks of the structures the device bounds (hs_oracle.c, HS_HW_*).  Test infrastructure.

The library is built by oracle_lib.build (the repository tree stays as it is); the default build that oracle_lib loads
compiles none of the counters."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O
from happysim_b200 import _abi as A

FIELDS = ("now", "now_pop", "future", "outbox", "inbox")     # HS_HW_NOW .. HS_HW_INBOX, then one queue per entity
HS_W_NCAP = 24               # csrc/hs_warp_engine.cuh: now-tier entries of a general-engine replica
HS_T_KS = 4                  # csrc/hs_thread_engine.cuh: of those, the thread engine keeps this many in shared memory
HS_NOW_CAP = 8               # csrc/hs_lane_engine.cuh: the lane engine's same-timestamp queue
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = O.build("oracle/hs_oracle.c", ("HS_ORACLE_HIGH_WATER",))
        L.hs_oracle_high_water_range.argtypes = [C.POINTER(A.ModelDesc), C.POINTER(A.RunParams), C.POINTER(A.Outputs),
                                                 C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
        L.hs_oracle_high_water_range.restype = C.c_int
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
    rows = np.zeros((p.n_replicas, len(FIELDS) + model.n_entities), np.uint32)
    bufs = O.run_range_parallel(lib().hs_oracle_high_water_range, model, p, chunk, rows.ctypes.data_as(C.POINTER(C.c_uint32)))
    return bufs, _marks(rows)


def _linked_slice(lm, params, *, end_ns, cseed):
    rows = [np.zeros((params[0].n_replicas, len(FIELDS) + m.n_entities), np.uint32) for m in lm.models]
    outs, delivered, lost, _ = O.run_linked_on(lib().hs_oracle_high_water_linked, lm, params, end_ns=end_ns, cseed=cseed,
                                               hw_rows=rows)
    return outs, delivered, lost, rows


def run_linked(lm, params: list, *, end_ns, cseed, chunk: int = 64):
    """oracle_lib.oracle_run_linked_parallel on the instrumented oracle (the replica words of LinkedRun): per partition
    the output buffers, delivered / lost per replica, and per partition the high-water marks."""
    lib()
    outs, delivered, lost, rows = O.run_slices(lambda ps: _linked_slice(lm, ps, end_ns=end_ns, cseed=cseed), params, chunk)
    return outs, delivered, lost, [_marks(r) for r in rows]


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
