"""Linked runs whose replicas are sweep cells, on the CPU: a ctypes binding of tests/linked_sweep_oracle.c, a LinkedRun
stand-in on it, and the models the linked sweep tests share.  Test infrastructure.

The library is compiled on first use into a temporary directory (the repository tree stays as it is), with the
oracle's own flags (oracle/Makefile), as tests/linked_fault_oracle_lib.py compiles the oracle it includes."""
from __future__ import annotations

import ctypes as C
import dataclasses
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib as O
from happysim_b200 import _abi as A
from happysim_b200.engine import make_params
from happysim_b200.linked import LinkedModel

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "linked_sweep_oracle.c"), os.path.join(_HERE, "linked_fault_oracle.c"),
         os.path.join(_HERE, "fault_oracle.c"), os.path.join(_ROOT, "oracle", "hs_oracle.c"),
         os.path.join(_ROOT, "include", "hs_b200.h")] + \
        [os.path.join(_ROOT, "happy-simulator_b200", "csrc", f) for f in ("hs_sampler.h", "hs_profile.h", "hs_sketch.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _SRCS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"hs_fault_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libhs_linked_sweep_oracle_{h}.so")
        if not os.path.exists(so):
            fma = ["-mfma"] if " fma " in open("/proc/cpuinfo").read() else []
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", *fma,
                                   "-pthread", "-shared", "-o", tmp, _SRCS[0], "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.hs_cells_oracle_run_linked.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32,
                                                 C.POINTER(C.c_int64), C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64,
                                                 C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.hs_cells_oracle_run_linked.restype = C.c_int
        _lib = L
    return _lib


def run_cells(lm, params: list, *, end_ns, cseed, cseed_stride=0, crid_base=None, crid_stride=None, replicas_per_cell=1):
    """A linked run of ``lm`` (a LinkedModel with or without cells; FAULT rows allowed) on the cell oracle: per
    partition the usual output buffers, per replica delivered / lost.  Partition q runs ``params[q]``; the coordinator
    draws with key ``cseed + g * cseed_stride`` and replica word ``crid_base + g * crid_stride`` (default P and P + 1)."""
    nP = lm.n_partitions
    descs = [m.desc() for m in lm.models]
    outs = [O.alloc_outputs(m.n_entities, p, m.sketch_layout()[2]) for m, p in zip(lm.models, params)]
    ends = np.array(lm.window_ends(end_ns), dtype=np.int64)
    link_arrs, dst_arrs = [], []
    for q in range(nP):
        arr, dst = lm.link_descs(q)
        link_arrs.append(arr)
        dst_arrs.append((C.c_uint32 * max(1, len(dst)))(*dst))
    n_links = (C.c_uint32 * nP)(*[len(ls) for ls in lm.links])
    PP = lambda T, xs: (C.POINTER(T) * nP)(*[C.cast(C.pointer(x) if not isinstance(x, C.Array) else x, C.POINTER(T)) for x in xs])
    n = params[0].n_replicas
    delivered, lost = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    rc = lib().hs_cells_oracle_run_linked(nP, PP(A.ModelDesc, descs), PP(A.RunParams, params), PP(A.Outputs, [o for _, o in outs]),
                                          PP(A.LinkDesc, link_arrs), PP(C.c_uint32, dst_arrs), n_links,
                                          max(1, lm.n_cells), max(1, int(replicas_per_cell)),
                                          ends.ctypes.data_as(C.POINTER(C.c_int64)), len(ends), lm.n_streams,
                                          cseed, cseed_stride, nP if crid_base is None else crid_base,
                                          nP + 1 if crid_stride is None else crid_stride,
                                          delivered.ctypes.data_as(C.POINTER(C.c_uint64)), lost.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert rc == 0, rc
    return [b for b, _ in outs], delivered, lost, ends


def run_cells_parallel(lm, params: list, *, chunk: int = 32, **kw):
    """run_cells on a thread pool over slices of ``chunk`` replicas (each keeps its global index, hence its cell and
    its draws), concatenated in replica order."""
    n = params[0].n_replicas
    lib()

    def part(r0):
        ps = []
        for p in params:
            q = A.RunParams.from_buffer_copy(p)
            q.n_replicas, q.replica_index_base = min(n, r0 + chunk) - r0, p.replica_index_base + r0
            ps.append(q)
        return run_cells(lm, ps, **kw)

    parts = O._pool_map(part, range(0, n, chunk))
    outs = [{k: (None if v is None else np.concatenate([pt[0][q][k] for pt in parts])) for k, v in parts[0][0][q].items()}
            for q in range(lm.n_partitions)]
    return outs, np.concatenate([pt[1] for pt in parts]), np.concatenate([pt[2] for pt in parts]), parts[0][3]


def partition_params(lm, *, seed, end_ns, n, caps, seed_stride=0, rid_stride=None, replica_index_base=0, replicas_per_cell=1,
                     flags=A.HS_RUN_ORDER_HASH):
    """The hs_run_params of every partition of a linked run, as LinkedRun.run makes them (partition q: word q + g * rid_stride)."""
    nP = lm.n_partitions
    rs = nP + 1 if rid_stride is None else rid_stride
    return [make_params(seed=seed, seed_stride=seed_stride, end_ns=end_ns, n_replicas=n, rid_base=q, rid_stride=rs,
                        replica_index_base=replica_index_base, replicas_per_cell=replicas_per_cell, flags=flags,
                        **(caps[q] if isinstance(caps, (list, tuple)) else caps)) for q in range(nP)]


def cell_of(n, replica_index_base=0, replicas_per_cell=1, n_cells=1):
    return ((replica_index_base + np.arange(n)) // replicas_per_cell) % n_cells


class OracleCellsLinkedRun:
    """``happysim_b200.linked.LinkedRun`` on the cell oracle, same interface (cells, strides and replicas_per_cell
    included): install it with ``monkeypatch.setattr(linked, "LinkedRun", OracleCellsLinkedRun)`` and
    ParallelSimulation's host path runs without a GPU.  Like oracle_lib.OracleLinkedRun its queues are unbounded and
    ``overflowed`` is all zeros; ``calls`` keeps the keyword arguments of every ``run``, the class's ``runs`` every
    instance made."""
    runs: list = []

    def __init__(self, lm, *, device=0):
        lm.validate()
        self.lm, self.device = lm, device
        self.windows = 0
        self.calls = []
        OracleCellsLinkedRun.runs.append(self)

    def close(self):
        pass

    def run(self, *, seed, end_ns, n_replicas=1, replica_index_base=0, caps=None, flags=A.HS_RUN_ORDER_HASH, queue_ring=0,
            replicas_per_cell=1, seed_stride=0, rid_stride=None):
        nP = self.lm.n_partitions
        caps = caps or {}
        per = [dict(caps[q] if isinstance(caps, (list, tuple)) else caps) for q in range(nP)]
        self.calls.append(dict(seed=seed, end_ns=end_ns, n_replicas=n_replicas, replica_index_base=replica_index_base,
                               caps=[dict(c) for c in per], flags=flags, queue_ring=queue_ring,
                               replicas_per_cell=replicas_per_cell, seed_stride=seed_stride, rid_stride=rid_stride))
        ps = partition_params(self.lm, seed=seed, end_ns=end_ns, n=n_replicas, caps=per, seed_stride=seed_stride,
                              rid_stride=rid_stride, replica_index_base=replica_index_base,
                              replicas_per_cell=replicas_per_cell, flags=flags)
        for p in ps:
            p.queue_ring = queue_ring
        rs = nP + 1 if rid_stride is None else rid_stride
        outs, delivered, lost, ends = run_cells(self.lm, ps, end_ns=end_ns, cseed=seed, cseed_stride=seed_stride,
                                                crid_base=nP, crid_stride=rs, replicas_per_cell=replicas_per_cell)
        self.windows = len(ends)
        return outs, (delivered, lost, np.zeros(n_replicas, np.uint64))


# ---- models ---------------------------------------------------------------------------------------------------------------

def with_link_cells(lm, rng, n_cells: int, zero_loss_cell: bool = True):
    """``lm`` (partitions possibly with model cells already) with a per-cell link table: cell 0 keeps the links'
    own values, every other cell scales each latency mean by 0.5 to 2 and draws a loss from {0, 0.05, 0.2}; with
    ``zero_loss_cell`` cell 1 loses nothing and cell 2 (if any) loses on every link, so lossless and lossy cells sit
    side by side."""
    tab = []
    for q, ls in enumerate(lm.links):
        t = np.zeros((n_cells, len(ls), 2), np.float64)
        for k, l in enumerate(ls):
            t[0, k] = (l.latency_mean_s, l.packet_loss)
            for c in range(1, n_cells):
                loss = float(rng.choice([0.0, 0.05, 0.2]))
                if zero_loss_cell and c == 1:
                    loss = 0.0
                elif zero_loss_cell and c == 2:
                    loss = 0.2
                t[c, k] = (l.latency_mean_s * float(rng.uniform(0.5, 2.0)), loss)
        tab.append(t)
    return dataclasses.replace(lm, models=list(lm.models), links=[list(ls) for ls in lm.links], cell_links=tab)


def with_model_cells(lm, rng, n_cells: int):
    """``lm`` whose every partition has ``n_cells`` model cells (tests/sweep_models.with_cells, REMOTE rows untouched)."""
    import sweep_models as SM
    return dataclasses.replace(lm, models=[SM.with_cells(m, rng, n_cells, "any") for m in lm.models])


def celled(lm, seed: int, n_cells: int):
    """A LinkedModel with ``n_cells`` cells in the partitions and on the links."""
    rng = np.random.RandomState(31_000 + seed)
    return with_link_cells(with_model_cells(lm, rng, n_cells), rng, n_cells)


KEYS = ("summaries", "entity_stats", "records", "sink_samples", "service_samples", "sketches")


def assert_replica_equal(got, want, r_got: int, r_want: int, what=""):
    """Replica r_got of one linked run's outputs against replica r_want of another's, partition by partition, byte
    for byte.  Recorder rings of different capacities (runs sized for different rates) are compared over the slots
    both have, which must hold everything the replica recorded."""
    rings = {"records": "events_processed", "sink_samples": "n_sink_samples", "service_samples": "n_service_samples"}
    for q, (g, w) in enumerate(zip(got, want)):
        for k in KEYS:
            a, b = g.get(k), w.get(k)
            if a is None and b is None:
                continue
            x, y = a[r_got], b[r_want]
            if k in rings and x.shape != y.shape:
                m = min(len(x), len(y))
                if k != "records":
                    assert int(g["summaries"][rings[k]][r_got]) <= m, f"{what}: partition {q}, {k} wrapped"
                x, y = x[:m], y[:m]
            assert x.tobytes() == y.tobytes(), f"{what}: partition {q}, {k} of replica {r_got} differs"
