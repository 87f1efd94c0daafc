"""ctypes binding of tests/layered_oracle.c: the CPU oracle with node faults, PriorityQueue servers and linked runs
whose replicas are sweep cells, and a LinkedRun stand-in on it.  Test infrastructure.

The library is built by oracle_lib.build (the repository tree stays as it is)."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O
from happysim_b200 import _abi as A
from happysim_b200.engine import make_params

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = O.build("tests/layered_oracle.c")
        L.hs_layered_oracle_run_range.argtypes = [C.POINTER(A.ModelDesc), C.POINTER(A.RunParams), C.POINTER(A.Outputs),
                                                  C.c_uint32, C.c_uint32]
        L.hs_layered_oracle_run_range.restype = C.c_int
        _lib = L
    return _lib


def run(model, p: A.RunParams, chunk: int = 256):
    """All replicas of ``p`` on the layered oracle (a thread pool over slices of ``chunk`` replicas); the buffers
    oracle_lib.alloc_outputs lays out."""
    return O.run_range_parallel(lib().hs_layered_oracle_run_range, model, p, chunk)


def run_linked(lm, params: list, *, end_ns, cseed, cseed_stride=0, crid_base=None, crid_stride=None, replicas_per_cell=1):
    """A linked run of ``lm`` (a LinkedModel with or without cells, FAULT rows and priority servers allowed) on the
    layered oracle: per partition the usual output buffers, per replica delivered / lost, and the window ends.
    Partition q runs ``params[q]``; the coordinator draws with key ``cseed + g * cseed_stride`` and replica word
    ``crid_base + g * crid_stride`` (default P and P + 1, LinkedRun's)."""
    return O.run_linked_on(lib().hs_layered_oracle_run_linked, lm, params, end_ns=end_ns, cseed=cseed,
                           cseed_stride=cseed_stride, crid_base=crid_base, crid_stride=crid_stride,
                           replicas_per_cell=replicas_per_cell)


def run_linked_parallel(lm, params: list, *, end_ns, chunk: int = 32, **kw):
    """run_linked on a thread pool over slices of ``chunk`` replicas (each keeps its global index, hence its cell and
    its draws), concatenated in replica order."""
    lib()
    outs, delivered, lost = O.run_slices(lambda ps: run_linked(lm, ps, end_ns=end_ns, **kw)[:3], params, chunk)
    return outs, delivered, lost, np.array(lm.window_ends(end_ns), dtype=np.int64)


class OracleCellsLinkedRun(O.OracleLinkedRun):
    """``happysim_b200.linked.LinkedRun`` on the layered oracle, same interface (cells, strides and replicas_per_cell
    included): install it with ``monkeypatch.setattr(linked, "LinkedRun", OracleCellsLinkedRun)`` and
    ParallelSimulation's host path runs without a GPU, faults and priority servers included.  Like
    oracle_lib.OracleLinkedRun its queues are unbounded and ``overflowed`` is all zeros; ``calls`` keeps the keyword
    arguments of every ``run``, the class's ``runs`` every instance made."""
    runs: list = []

    def __init__(self, lm, *, device=0):
        super().__init__(lm, device=device)
        OracleCellsLinkedRun.runs.append(self)

    def run(self, *, seed, end_ns, n_replicas=1, replica_index_base=0, caps=None, flags=A.HS_RUN_ORDER_HASH, queue_ring=0,
            replicas_per_cell=1, seed_stride=0, rid_stride=None):
        nP = self.lm.n_partitions
        caps = caps or {}
        per = [dict(caps[q] if isinstance(caps, (list, tuple)) else caps) for q in range(nP)]
        self.calls.append(dict(seed=seed, end_ns=end_ns, n_replicas=n_replicas, replica_index_base=replica_index_base,
                               caps=[dict(c) for c in per], flags=flags, queue_ring=queue_ring,
                               replicas_per_cell=replicas_per_cell, seed_stride=seed_stride, rid_stride=rid_stride))
        rs = nP + 1 if rid_stride is None else rid_stride
        ps = [make_params(seed=seed, seed_stride=seed_stride, end_ns=end_ns, n_replicas=n_replicas, rid_base=q, rid_stride=rs,
                          replica_index_base=replica_index_base, replicas_per_cell=replicas_per_cell, queue_ring=queue_ring,
                          flags=flags, **per[q]) for q in range(nP)]
        outs, delivered, lost, ends = run_linked(self.lm, ps, end_ns=end_ns, cseed=seed, cseed_stride=seed_stride,
                                                 crid_stride=rs, replicas_per_cell=replicas_per_cell)
        self.windows = len(ends)
        return outs, (delivered, lost, np.zeros(n_replicas, np.uint64))
