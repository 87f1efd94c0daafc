"""ctypes binding of the CPU oracle (oracle/libhs_oracle.so), and the one way the tests build and call the other host
libraries they check against (build, run_range_parallel, run_linked_on, run_slices).  Test infrastructure."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import re
import subprocess
import tempfile

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
        L.hs_oracle_run_trace_range.argtypes = list(L.hs_oracle_run_trace.argtypes) + [
            C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.hs_oracle_run_trace_range.restype = C.c_int
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


_INCLUDE = re.compile(rb'^[ \t]*#[ \t]*include[ \t]*"([^"]+)"', re.M)
_built: dict = {}


def _sources(path: str, seen: dict) -> dict:
    """{path: contents} of ``path`` and of every file it includes with quotes, transitively"""
    path = os.path.normpath(path)
    if path not in seen:
        seen[path] = data = open(path, "rb").read()
        for inc in _INCLUDE.findall(data):
            _sources(os.path.join(os.path.dirname(path), inc.decode()), seen)
    return seen


def build(src: str, defines=()) -> C.CDLL:
    """``src`` (a path under the repository) compiled by oracle/Makefile's rule, with ``-D`` for each of ``defines``,
    and loaded.  The library goes to a per-user temporary directory, under a name keyed by every file ``src``
    includes, the Makefile and the defines, so the repository tree stays as it is and an edit rebuilds it."""
    key = (src, tuple(defines))
    if key not in _built:
        src, mk = os.path.join(_ROOT, src), os.path.join(_ROOT, "oracle", "Makefile")
        h = hashlib.sha256()
        for data in _sources(src, {mk: open(mk, "rb").read()}).values():
            h.update(data)
        h.update(repr(key[1]).encode())
        d = os.path.join(tempfile.gettempdir(), f"hs_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"lib{os.path.splitext(os.path.basename(src))[0]}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}"
            subprocess.check_call(["make", "-s", "-f", mk, f"SRC={src}", f"OUT={tmp}",
                                   "DEFS=" + " ".join(f"-D{x}" for x in defines)])
            os.replace(tmp, so)
        _built[key] = C.CDLL(so)
    return _built[key]


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


def _pool_map(fn, items):
    from concurrent.futures import ThreadPoolExecutor
    lib()                                       # load once, before the threads
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as ex:
        return list(ex.map(fn, items))


def run_range_parallel(fn, model: happysim_b200.FlatModel, p: A.RunParams, chunk: int = 256, *extra):
    """``fn`` -- hs_oracle_run_range or an entry point with its arguments, then ``extra`` -- on a thread pool over
    slices of ``chunk`` replicas into one set of buffers (ctypes releases the GIL for the call, and a replica only
    writes its own rows)."""
    d = model.desc()
    bufs, o = alloc_outputs(model.n_entities, p, model.sketch_layout()[2])
    n = p.n_replicas

    def part(r0):
        assert fn(C.byref(d), C.byref(p), C.byref(o), r0, min(n, r0 + chunk), *extra) == 0

    _pool_map(part, range(0, n, chunk))
    return bufs


def oracle_run_parallel(model: happysim_b200.FlatModel, p: A.RunParams, chunk: int = 256):
    """oracle_run on a thread pool: hs_oracle_run_range over slices of ``chunk`` replicas."""
    return run_range_parallel(lib().hs_oracle_run_range, model, p, chunk)


def _cat(xs):
    """the per-replica results of consecutive slices joined: arrays concatenated, lists and dicts of them item by item"""
    if xs[0] is None:
        return None
    if isinstance(xs[0], dict):
        return {k: _cat([x[k] for x in xs]) for k in xs[0]}
    if isinstance(xs[0], list):
        return [_cat([x[q] for x in xs]) for q in range(len(xs[0]))]
    return np.concatenate(xs)


def run_slices(run, params: list, chunk: int):
    """``run(ps)`` of a linked run on a thread pool over slices of ``chunk`` replicas (``ps``: ``params`` with
    replica_index_base moved along, so every replica keeps its global index and with it its draws and its cell).  What
    ``run`` returns, every item per replica, is concatenated in replica order."""
    n = params[0].n_replicas

    def part(r0):
        ps = []
        for p in params:
            q = A.RunParams.from_buffer_copy(p)
            q.n_replicas, q.replica_index_base = min(n, r0 + chunk) - r0, p.replica_index_base + r0
            ps.append(q)
        return run(ps)

    parts = _pool_map(part, range(0, n, chunk))
    return [_cat([pt[i] for pt in parts]) for i in range(len(parts[0]))]


def run_linked_on(fn, lm, params: list, *, end_ns, cseed, cseed_stride=0, crid_base=None, crid_stride=None,
                  replicas_per_cell=None, hw_rows=None):
    """``fn`` -- hs_oracle_run_linked or an entry point with its arguments -- on a linked run
    (happysim_b200.linked.LinkedModel): per partition the usual output buffers, per replica the delivered / lost
    cross-partition events, and the window ends.  Partition q runs ``params[q]``; the coordinator draws with key
    ``cseed + g * cseed_stride`` and replica word ``crid_base + g * crid_stride`` (default P and P + 1, LinkedRun's).
    Where ``fn`` takes them: ``replicas_per_cell`` passes the cell table (every partition's link count, the cells,
    replicas per cell) after the link destinations, ``hw_rows`` (a uint32 array per partition) goes last."""
    nP = lm.n_partitions
    descs = [m.desc() for m in lm.models]
    outs = [alloc_outputs(m.n_entities, p, m.sketch_layout()[2]) for m, p in zip(lm.models, params)]
    ends = np.array(lm.window_ends(end_ns), dtype=np.int64)
    link_arrs, dsts = zip(*(lm.link_descs(q) for q in range(nP)))
    dst_arrs = [(C.c_uint32 * max(1, len(d)))(*d) for d in dsts]
    PP = lambda T, xs: (C.POINTER(T) * nP)(*[C.cast(x if isinstance(x, C.Array) else C.pointer(x), C.POINTER(T)) for x in xs])  # noqa: E731
    n = params[0].n_replicas
    delivered, lost = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    u32, u64 = C.c_uint32, C.c_uint64
    args = [u32(nP), PP(A.ModelDesc, descs), PP(A.RunParams, params), PP(A.Outputs, [o for _, o in outs]),
            PP(A.LinkDesc, link_arrs), PP(C.c_uint32, dst_arrs)]
    if replicas_per_cell is not None:
        args += [(C.c_uint32 * nP)(*[len(ls) for ls in lm.links]), u32(max(1, lm.n_cells)), u32(max(1, int(replicas_per_cell)))]
    args += [ends.ctypes.data_as(C.POINTER(C.c_int64)), u32(len(ends)), u32(lm.n_streams), u64(cseed), u64(cseed_stride),
             u32(nP if crid_base is None else crid_base), u32(nP + 1 if crid_stride is None else crid_stride),
             delivered.ctypes.data_as(C.POINTER(C.c_uint64)), lost.ctypes.data_as(C.POINTER(C.c_uint64))]
    if hw_rows is not None:
        args.append((C.POINTER(C.c_uint32) * nP)(*[r.ctypes.data_as(C.POINTER(C.c_uint32)) for r in hw_rows]))
    rc = fn(*args)
    assert rc == 0, rc
    return [b for b, _ in outs], delivered, lost, ends


def oracle_run_linked_parallel(lm, params: list, *, end_ns, cseed, chunk: int = 64):
    """oracle_run_linked on a thread pool (run_slices)."""
    outs, delivered, lost = run_slices(lambda ps: oracle_run_linked(lm, ps, end_ns=end_ns, cseed=cseed)[:3], params, chunk)
    return outs, delivered, lost, np.array(lm.window_ends(end_ns), dtype=np.int64)


def oracle_run_linked(lm, params: list, *, end_ns, cseed, cseed_stride=0, crid_base=None, crid_stride=None):
    """A linked run (happysim_b200.linked.LinkedModel) on the oracle: per partition the usual output buffers,
    plus per-replica counts of delivered / lost cross-partition events (run_linked_on)."""
    return run_linked_on(lib().hs_oracle_run_linked, lm, params, end_ns=end_ns, cseed=cseed, cseed_stride=cseed_stride,
                         crid_base=crid_base, crid_stride=crid_stride)


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


def _trace_rows(x, n):
    """Draws of one stream as [n_replicas, n_draws] float64 rows (a 1-D array: the row of a single replica)."""
    a = np.ascontiguousarray(np.zeros((n, 0)) if x is None else x, dtype=np.float64)
    a = a[None, :] if a.ndim == 1 else a
    assert a.ndim == 2 and a.shape[0] == n, (a.shape, n)
    return a


def oracle_run_trace(model, p: A.RunParams, targets, service, chunk: int = 64):
    """Replicas fed with externally captured draws (the reference's stock RNG outputs): ``targets`` and ``service``
    hold one row per replica slot, [n_replicas, n] as ``Engine.set_trace`` takes them (a 1-D array is the row of a
    single replica; None or zero columns leave that stream to Philox).  Returns the output buffers plus
    ``arr_used`` / ``svc_used``: how many draws of each stream every replica asked for, whether or not its row had
    them (a draw past the end of a row is a target of 1e300).  Runs on a thread pool in slices of ``chunk``."""
    d = model.desc()
    n = p.n_replicas
    bufs, o = alloc_outputs(model.n_entities, p, model.sketch_layout()[2])
    t, s = _trace_rows(targets, n), _trace_rows(service, n)
    bufs["arr_used"], bufs["svc_used"] = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    dp = C.POINTER(C.c_double)
    up = C.POINTER(C.c_uint64)

    def part(r0):
        assert lib().hs_oracle_run_trace_range(C.byref(d), C.byref(p), C.byref(o), t.ctypes.data_as(dp), t.shape[1],
                                               s.ctypes.data_as(dp), s.shape[1], r0, min(n, r0 + chunk),
                                               bufs["arr_used"].ctypes.data_as(up), bufs["svc_used"].ctypes.data_as(up)) == 0

    _pool_map(part, range(0, n, chunk))
    return bufs
