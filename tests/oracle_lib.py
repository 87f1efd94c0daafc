"""ctypes binding of the CPU oracle (oracle/libhs_oracle.so).  Test infrastructure."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import happysim_b200
from happysim_b200 import _abi as A
from happysim_b200.engine import make_params

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(_ROOT, "oracle", "libhs_oracle.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-C", os.path.join(_ROOT, "oracle")], stdout=subprocess.DEVNULL)
        L = C.CDLL(_SO)
        L.hs_oracle_run.argtypes = [C.POINTER(A.ModelDesc), C.POINTER(A.RunParams), C.POINTER(A.Outputs)]
        L.hs_oracle_run.restype = C.c_int
        L.hs_oracle_run_range.argtypes = [C.POINTER(A.ModelDesc), C.POINTER(A.RunParams), C.POINTER(A.Outputs),
                                          C.c_uint32, C.c_uint32]
        L.hs_oracle_run_range.restype = C.c_int
        L.hs_oracle_run_trace.argtypes = [C.POINTER(A.ModelDesc), C.POINTER(A.RunParams), C.POINTER(A.Outputs),
                                          C.POINTER(C.c_double), C.c_uint64, C.POINTER(C.c_double), C.c_uint64]
        L.hs_oracle_run_trace.restype = C.c_int
        L.hs_cpu_uniform.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint64]
        L.hs_cpu_uniform.restype = C.c_double
        for n in ("hs_cpu_log", "hs_cpu_exp1"):
            getattr(L, n).argtypes = [C.c_double]; getattr(L, n).restype = C.c_double
        L.hs_cpu_seconds_to_ns.argtypes = [C.c_double]; L.hs_cpu_seconds_to_ns.restype = C.c_int64
        L.hs_cpu_ns_to_seconds.argtypes = [C.c_int64]; L.hs_cpu_ns_to_seconds.restype = C.c_double
        L.hs_cpu_next_arrival_ns.argtypes = [C.c_int64, C.c_double, C.c_double]
        L.hs_cpu_next_arrival_ns.restype = C.c_int64
        L.hs_cpu_exp_latency_ns.argtypes = [C.c_double, C.c_double]; L.hs_cpu_exp_latency_ns.restype = C.c_int64
        L.hs_cpu_latency_bin.argtypes = [C.c_int64]; L.hs_cpu_latency_bin.restype = C.c_uint32
        L.hs_cpu_hash_step.argtypes = [C.c_uint64, C.c_int64, C.c_uint64, C.c_uint32, C.c_uint32]
        L.hs_cpu_hash_step.restype = C.c_uint64
        L.hs_cpu_next_arrival_profile_ns.argtypes = [C.c_int32] + [C.c_double] * 4 + [C.c_int64, C.c_double]
        L.hs_cpu_next_arrival_profile_ns.restype = C.c_int64
        L.hs_cpu_integrate_rate.argtypes = [C.c_int32] + [C.c_double] * 6
        L.hs_cpu_integrate_rate.restype = C.c_double
        L.hs_cpu_philox.argtypes = [C.c_uint32] * 6 + [C.POINTER(C.c_uint32)]
        L.hs_cpu_philox.restype = None
        L.hs_cpu_routing_key.argtypes = [C.c_double, C.c_int32, C.POINTER(C.c_double)]
        L.hs_cpu_routing_key.restype = C.c_int32
        L.hs_cpu_sketch_add.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_int32]
        L.hs_cpu_sketch_add.restype = None
        L.hs_cpu_hll_hash.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        L.hs_cpu_hll_hash.restype = None
        L.hs_cpu_cms_row_seed.argtypes = [C.c_uint64, C.c_int32]; L.hs_cpu_cms_row_seed.restype = C.c_uint64
        L.hs_cpu_cms_col.argtypes = [C.c_uint64, C.c_int32, C.c_int32]; L.hs_cpu_cms_col.restype = C.c_int32
        L.hs_cpu_bloom_bit.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.c_int32]; L.hs_cpu_bloom_bit.restype = C.c_int32
        L.hs_cpu_tdigest_add.argtypes = [C.c_void_p, C.c_double, C.c_uint32, C.c_uint32, C.c_double]
        L.hs_cpu_tdigest_add.restype = C.c_int
        L.hs_sketch_layout.argtypes = [C.POINTER(A.ModelDesc)] + [C.POINTER(C.c_uint64)] * 4
        L.hs_sketch_layout.restype = C.c_int
        _lib = L
    return _lib


def alloc_outputs(n_entities: int, p: A.RunParams, sketch_bytes: int = 0):
    """Host buffers (numpy) + the hs_outputs struct pointing at them."""
    n = p.n_replicas
    bufs = {
        "summaries": np.zeros(n, A.SUMMARY_DTYPE),
        "entity_stats": np.zeros((n, n_entities), A.STATS_DTYPE),
        "records": np.zeros((n, p.record_cap), A.RECORD_DTYPE) if p.record_cap else None,
        "sink_samples": np.zeros((n, p.sample_cap), A.SAMPLE_DTYPE) if p.sample_cap else None,
        "service_samples": np.zeros((n, p.service_cap), np.float64) if p.service_cap else None,
        "histograms": np.zeros((n, A.HS_HISTOGRAM_BINS), np.uint32) if (p.flags & A.HS_RUN_HISTOGRAM) else None,
        "sketches": np.zeros((n, sketch_bytes), np.uint8) if sketch_bytes else None,
    }
    o = A.Outputs()
    o.summaries = bufs["summaries"].ctypes.data_as(C.POINTER(A.ReplicaSummary))
    o.entity_stats = bufs["entity_stats"].ctypes.data_as(C.POINTER(A.EntityStats))
    if p.record_cap:
        o.records = bufs["records"].ctypes.data_as(C.POINTER(A.EventRecord))
    if p.sample_cap:
        o.sink_samples = bufs["sink_samples"].ctypes.data_as(C.POINTER(A.SinkSample))
    if p.service_cap:
        o.service_samples = bufs["service_samples"].ctypes.data_as(C.POINTER(C.c_double))
    if bufs["histograms"] is not None:
        o.histograms = bufs["histograms"].ctypes.data_as(C.POINTER(C.c_uint32))
    if bufs["sketches"] is not None:
        o.sketches = bufs["sketches"].ctypes.data_as(C.POINTER(C.c_uint8))
    return bufs, o


def oracle_run(model: happysim_b200.FlatModel, p: A.RunParams, r0=None, r1=None):
    d = model.desc()
    bufs, o = alloc_outputs(model.n_entities, p, model.sketch_layout()[2])
    if r0 is None:
        rc = lib().hs_oracle_run(C.byref(d), C.byref(p), C.byref(o))
    else:
        rc = lib().hs_oracle_run_range(C.byref(d), C.byref(p), C.byref(o), r0, r1)
    assert rc == 0, rc
    return bufs


def oracle_run_linked(lm, params: list, *, end_ns, cseed, cseed_stride=0, crid_base=None, crid_stride=None):
    """A linked run (happysim_b200.linked.LinkedModel) on the oracle: per partition the usual output buffers,
    plus per-replica counts of delivered / lost cross-partition events."""
    L = lib()
    nP = lm.n_partitions
    descs = [m.desc() for m in lm.models]
    outs = [alloc_outputs(m.n_entities, p, m.sketch_layout()[2]) for m, p in zip(lm.models, params)]
    ends = np.array(lm.window_ends(end_ns), dtype=np.int64)
    link_arrs, dst_arrs = [], []
    for q in range(nP):
        arr, dst = lm.link_descs(q)
        link_arrs.append(arr)
        dst_arrs.append((C.c_uint32 * max(1, len(dst)))(*dst))
    PP = lambda T, xs: (C.POINTER(T) * nP)(*[C.cast(C.pointer(x) if not isinstance(x, C.Array) else x, C.POINTER(T)) for x in xs])
    n = params[0].n_replicas
    delivered, lost = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    L.hs_oracle_run_linked.restype = C.c_int
    L.hs_oracle_run_linked.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.POINTER(C.c_int64), C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32,
                                       C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    rc = L.hs_oracle_run_linked(nP, PP(A.ModelDesc, descs), PP(A.RunParams, params), PP(A.Outputs, [o for _, o in outs]),
                                PP(A.LinkDesc, link_arrs), PP(C.c_uint32, dst_arrs),
                                ends.ctypes.data_as(C.POINTER(C.c_int64)), len(ends), lm.n_streams,
                                cseed, cseed_stride, nP if crid_base is None else crid_base,
                                nP + 1 if crid_stride is None else crid_stride,
                                delivered.ctypes.data_as(C.POINTER(C.c_uint64)), lost.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert rc == 0, rc
    return [b for b, _ in outs], delivered, lost, ends


class OracleLinkedRun:
    """``happysim_b200.linked.LinkedRun`` on the CPU oracle, same interface: install it with
    ``monkeypatch.setattr(linked, "LinkedRun", OracleLinkedRun)`` and ParallelSimulation's whole host path (lowering,
    ring sizing, the retry loop, the summary, the write-back) runs without a GPU.  Replica r of partition q draws from
    the replica word ``q + g * (P + 1)``, the coordinator from ``P + g * (P + 1)``, exactly as on the device, and the
    recorder rings are the ``caps`` passed in: a ring that is too small wraps as the device's does.

    The oracle's queues are unbounded (hs_oracle.c never reads ``queue_ring`` and never sets HS_ST_QUEUE_OVERFLOW), so
    this stand-in never reports a queue overflow and ``overflowed`` is all zeros.  ``calls`` keeps the keyword
    arguments of every ``run``."""

    def __init__(self, lm, *, device=0):
        lm.validate()
        self.lm, self.device = lm, device
        self.windows = 0
        self.calls = []

    def close(self):
        pass

    def run(self, *, seed, end_ns, n_replicas=1, replica_index_base=0, caps=None, flags=A.HS_RUN_ORDER_HASH, queue_ring=0):
        nP = self.lm.n_partitions
        caps = caps or {}
        per = [dict(caps[q] if isinstance(caps, (list, tuple)) else caps) for q in range(nP)]
        self.calls.append(dict(seed=seed, end_ns=end_ns, n_replicas=n_replicas, replica_index_base=replica_index_base,
                               caps=[dict(c) for c in per], flags=flags, queue_ring=queue_ring))
        ps = [make_params(seed=seed, end_ns=end_ns, n_replicas=n_replicas, rid_base=q, rid_stride=nP + 1,
                          replica_index_base=replica_index_base, queue_ring=queue_ring, flags=flags, **per[q])
              for q in range(nP)]
        outs, delivered, lost, ends = oracle_run_linked(self.lm, ps, end_ns=end_ns, cseed=seed)
        self.windows = len(ends)
        return outs, (delivered, lost, np.zeros(n_replicas, np.uint64))


def oracle_run_trace(model, p: A.RunParams, targets, service):
    """One replica fed with externally captured draws (the reference's stock RNG outputs)."""
    d = model.desc()
    bufs, o = alloc_outputs(model.n_entities, p)
    t = np.ascontiguousarray(targets, dtype=np.float64)
    s = np.ascontiguousarray(service, dtype=np.float64)
    rc = lib().hs_oracle_run_trace(C.byref(d), C.byref(p), C.byref(o),
                                   t.ctypes.data_as(C.POINTER(C.c_double)), len(t),
                                   s.ctypes.data_as(C.POINTER(C.c_double)), len(s))
    assert rc == 0, rc
    return bufs
