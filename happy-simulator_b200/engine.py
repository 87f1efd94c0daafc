"""ctypes binding of the C-ABI (include/hs_b200.h -> libhs_b200.so).

``Engine`` is the host-side handle behind ``Simulation.run()`` and
``ParallelRunner.run_replicas``: upload a FlatModel, run replicas, read results.
The CUDA library is mandatory: if it is missing or no GPU is visible the
constructor raises (there is no CPU path in the product).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _abi as A
from .build import LIB_PATH
from .model import FlatModel


class EngineError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"hs_b200 error {code}: {msg}")
        self.code = code


_lib = None

EXPORTED_SYMBOLS = ["hs_version", "hs_last_error", "hs_engine_create", "hs_engine_destroy", "hs_model_upload",
                    "hs_model_validate", "hs_run", "hs_set_trace", "hs_sync", "hs_last_run_ms", "hs_launch_count",
                    "hs_last_launch", "hs_read_outputs", "hs_read_totals", "hs_read_cell_totals", "hs_totals_device_ptr",
                    "hs_sketch_layout", "hs_read_sketches", "hs_coordinator_create", "hs_coordinator_destroy",
                    "hs_coordinator_exchange", "hs_coordinator_exchange_cells", "hs_link_cells_validate",
                    "hs_coordinator_read", "hs_read_outbox", "hs_read_inbox",
                    "hs_partition_upload", "hs_partition_validate", "hs_set_buckets", "hs_read_buckets",
                    "hs_read_bucket_totals", "hs_set_bucket_percentiles", "hs_read_bucket_percentiles",
                    "hs_read_bucket_percentile_totals"]


def load_library(path: str | None = None):
    """dlopen libhs_b200.so and declare every entry point of include/hs_b200.h."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise EngineError(A.HS_ERR_STATE, f"{p} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
    L = C.CDLL(p)
    # the version first: a library built from older sources says so, instead of lacking a newer entry point below
    L.hs_version.argtypes, L.hs_version.restype = [], C.c_uint32
    if L.hs_version() != A.HS_ABI_VERSION:
        raise EngineError(A.HS_ERR_STATE, f"{p} has ABI version {L.hs_version()}, this package needs {A.HS_ABI_VERSION}; "
                                          "rebuild it with `python -c 'import __graft_entry__ as g; g.build()'`")
    H = C.c_void_p
    sigs = {
        "hs_version": ([], C.c_uint32),
        "hs_last_error": ([C.c_char_p, C.c_int], C.c_int),
        "hs_engine_create": ([C.c_int, C.c_void_p, C.POINTER(H)], C.c_int),
        "hs_engine_destroy": ([H], C.c_int),
        "hs_model_upload": ([H, C.POINTER(A.ModelDesc)], C.c_int),
        "hs_model_validate": ([C.POINTER(A.ModelDesc)], C.c_int),
        "hs_partition_upload": ([H, C.POINTER(A.ModelDesc)], C.c_int),
        "hs_partition_validate": ([C.POINTER(A.ModelDesc)], C.c_int),
        "hs_run": ([H, C.POINTER(A.RunParams)], C.c_int),
        "hs_set_trace": ([H, C.POINTER(C.c_double), C.c_uint64, C.POINTER(C.c_double), C.c_uint64, C.c_uint32], C.c_int),
        "hs_sync": ([H], C.c_int),
        "hs_last_run_ms": ([H, C.POINTER(C.c_float)], C.c_int),
        "hs_launch_count": ([H, C.POINTER(C.c_uint64)], C.c_int),
        "hs_last_launch": ([H, C.POINTER(A.LaunchInfo)], C.c_int),
        "hs_read_outputs": ([H, C.POINTER(A.Outputs)], C.c_int),
        "hs_read_totals": ([H, C.POINTER(A.Totals)], C.c_int),
        "hs_read_cell_totals": ([H, C.POINTER(A.CellTotals), C.c_uint32], C.c_int),
        "hs_totals_device_ptr": ([H, C.POINTER(C.c_void_p)], C.c_int),
        "hs_sketch_layout": ([C.POINTER(A.ModelDesc), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                              C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)], C.c_int),
        "hs_read_sketches": ([H, C.c_void_p, C.c_uint64], C.c_int),
        "hs_coordinator_create": ([C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32,
                                   C.c_uint32, C.POINTER(H)], C.c_int),
        "hs_coordinator_destroy": ([H], None),
        "hs_coordinator_exchange": ([H, H, C.c_uint32, C.POINTER(A.LinkDesc), C.POINTER(H)], C.c_int),
        "hs_coordinator_exchange_cells": ([H, H, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(A.LinkDesc), C.POINTER(H)], C.c_int),
        "hs_link_cells_validate": ([C.c_uint32, C.c_uint32, C.POINTER(A.LinkDesc)], C.c_int),
        "hs_coordinator_read": ([H, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)], C.c_int),
        "hs_read_outbox": ([H, C.c_void_p, C.POINTER(C.c_uint32)], C.c_int),
        "hs_read_inbox": ([H, C.c_void_p, C.POINTER(C.c_uint32)], C.c_int),
        "hs_set_buckets": ([H, C.c_double, C.c_uint32], C.c_int),
        "hs_read_buckets": ([H, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)], C.c_int),
        "hs_read_bucket_totals": ([H, C.c_void_p, C.c_uint32], C.c_int),
        "hs_set_bucket_percentiles": ([H, C.c_uint32], C.c_int),
        "hs_read_bucket_percentiles": ([H, C.c_void_p], C.c_int),
        "hs_read_bucket_percentile_totals": ([H, C.c_void_p, C.c_uint32], C.c_int),
    }
    for name, (args, res) in sigs.items():
        fn = getattr(L, name)
        fn.argtypes, fn.restype = args, res
    if path is None:
        _lib = L
    return L


def _check(L, rc: int):
    if rc != 0:
        buf = C.create_string_buffer(512)
        L.hs_last_error(buf, 512)
        raise EngineError(rc, buf.value.decode(errors="replace"))


def validate_model(model: FlatModel, partition: bool = False) -> None:
    """hs_model_validate, or hs_partition_validate for ``partition`` (a partition of a linked run)"""
    L = load_library()
    d = model.desc()
    _check(L, (L.hs_partition_validate if partition else L.hs_model_validate)(C.byref(d)))


def make_params(*, seed=1234, end_ns, n_replicas=1, seed_stride=0, rid_base=0, rid_stride=1,
                replica_index_base=0, replicas_per_cell=1, record_cap=0, sample_cap=0, service_cap=0,
                queue_ring=0, engine=0, window_end_ns=-1, resume=0, flags=A.HS_RUN_ORDER_HASH,
                max_events=0) -> A.RunParams:
    p = A.RunParams()
    p.seed, p.seed_stride, p.rid_base, p.rid_stride = seed, seed_stride, rid_base, rid_stride
    p.end_ns = int(end_ns)
    p.n_replicas, p.replica_index_base = n_replicas, replica_index_base
    p.replicas_per_cell = max(1, replicas_per_cell)
    p.record_cap, p.sample_cap, p.service_cap = record_cap, sample_cap, service_cap
    p.queue_ring, p.engine = queue_ring, engine
    p.window_end_ns, p.resume, p.flags = int(window_end_ns), resume, flags
    p.max_events = int(max_events)
    return p


def validate_link_cells(links, n_links: int, n_cells: int) -> None:
    """hs_link_cells_validate: the checks hs_coordinator_exchange_cells makes of a per-cell link table (ctypes
    hs_link_desc array of n_cells * n_links), without a device."""
    L = load_library()
    _check(L, L.hs_link_cells_validate(n_links, n_cells, links))


class Coordinator:
    """The window barrier of a linked run (hs_coordinator_*, parallel/coordinator.py:182-227): per-replica draw
    counters of the loss stream and the links' latency streams, delivery totals."""

    def __init__(self, device: int, n_replicas: int, n_streams: int, *, seed, seed_stride=0, rid_base, rid_stride,
                 replica_index_base=0, stream: int | None = None):
        self._L = load_library()
        self._h = C.c_void_p()
        self.n_replicas = int(n_replicas)
        _check(self._L, self._L.hs_coordinator_create(device, C.c_void_p(stream or 0), n_replicas, n_streams, seed, seed_stride, rid_base,
                                                      rid_stride, replica_index_base, C.byref(self._h)))

    def exchange(self, src: "Engine", links, dsts, n_cells: int = 0, replicas_per_cell: int = 1) -> None:
        """Drain ``src``'s outboxes through its outgoing ``links`` (ctypes hs_link_desc array) into the inboxes of the
        engines ``dsts`` (one per link slot).  With ``n_cells`` > 0, ``links`` is the per-cell table [n_cells][slot]
        and replica g sends through row (g / replicas_per_cell) % n_cells (hs_coordinator_exchange_cells)."""
        arr = (C.c_void_p * max(1, len(dsts)))(*[d._h for d in dsts])
        if n_cells:
            _check(self._L, self._L.hs_coordinator_exchange_cells(self._h, src._h, len(dsts), n_cells, replicas_per_cell,
                                                                   links, arr))
        else:
            _check(self._L, self._L.hs_coordinator_exchange(self._h, src._h, len(dsts), links, arr))

    def read(self):
        """(delivered, lost, overflowed) uint64[n_replicas] since creation."""
        out = [np.zeros(self.n_replicas, np.uint64) for _ in range(3)]
        _check(self._L, self._L.hs_coordinator_read(self._h, *[o.ctypes.data_as(C.POINTER(C.c_uint64)) for o in out]))
        return tuple(out)

    def close(self):
        if self._h:
            self._L.hs_coordinator_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """One engine per (process, device); not thread-safe (one host thread per handle)."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self._L = load_library()
        self._h = C.c_void_p()
        _check(self._L, self._L.hs_engine_create(device, C.c_void_p(stream or 0), C.byref(self._h)))
        self.device = device
        self._model: FlatModel | None = None
        self._params: A.RunParams | None = None

    def close(self):
        if self._h:
            self._L.hs_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload(self, model: FlatModel, partition: bool = False) -> None:
        """hs_model_upload, or hs_partition_upload for ``partition`` (a partition of a linked run)"""
        d = model.desc()
        _check(self._L, (self._L.hs_partition_upload if partition else self._L.hs_model_upload)(self._h, C.byref(d)))
        self._model = model

    def set_trace(self, arrival_targets=None, service_samples=None) -> None:
        """Externally supplied draws, float64 [n_replicas, n] each (None/None: back to Philox)."""
        if arrival_targets is None and service_samples is None:
            _check(self._L, self._L.hs_set_trace(self._h, None, 0, None, 0, 0))
            return
        a = np.ascontiguousarray(arrival_targets, dtype=np.float64)
        s = np.ascontiguousarray(service_samples, dtype=np.float64)
        assert a.ndim == 2 and s.ndim == 2 and a.shape[0] == s.shape[0]
        _check(self._L, self._L.hs_set_trace(self._h, a.ctypes.data_as(C.POINTER(C.c_double)), a.shape[1],
                                             s.ctypes.data_as(C.POINTER(C.c_double)), s.shape[1], a.shape[0]))

    def set_buckets(self, width_s: float = 0.0, n: int = 0) -> None:
        """hs_set_buckets: time buckets of width_s seconds, n per row, for the following runs (n = 0: off)."""
        _check(self._L, self._L.hs_set_buckets(self._h, float(width_s), int(n)))

    def read_buckets(self, n: int):
        """(BUCKET_DTYPE [n_replicas, rows, n + 1], int64 past-end index [n_replicas, rows]) of the last run, which had
        n buckets per row (hs_read_buckets)."""
        rows = C.c_uint32()
        _check(self._L, self._L.hs_read_buckets(self._h, None, None, C.byref(rows)))
        nr, nb = int(self._params.n_replicas), int(rows.value)
        buf, past = np.zeros((nr, nb, n + 1), A.BUCKET_DTYPE), np.zeros((nr, nb), np.int64)
        _check(self._L, self._L.hs_read_buckets(self._h, buf.ctypes.data, past.ctypes.data, None))
        return buf, past

    def read_bucket_totals(self, n_cells: int, rows: int, n: int):
        """BUCKET_TOTAL_DTYPE [n_cells, rows, n + 1]: the last run's buckets reduced per sweep cell (hs_read_bucket_totals)."""
        out = np.zeros((n_cells, rows, n + 1), A.BUCKET_TOTAL_DTYPE)
        _check(self._L, self._L.hs_read_bucket_totals(self._h, out.ctypes.data, n_cells))
        return out

    def set_bucket_percentiles(self, sample_cap: int = 0) -> None:
        """hs_set_bucket_percentiles: p50 / p99 of every time bucket, from at most sample_cap values per bucket, for the
        following runs (0: off)."""
        _check(self._L, self._L.hs_set_bucket_percentiles(self._h, int(sample_cap)))

    def read_bucket_percentiles(self, n: int):
        """float64 [n_replicas, rows, n + 1, 2]: {p50, p99} of every bucket of the last run, which had n buckets per row
        (hs_read_bucket_percentiles; NaN where a bucket overflowed its sample capacity, 0 where it is empty)."""
        rows = C.c_uint32()
        _check(self._L, self._L.hs_read_buckets(self._h, None, None, C.byref(rows)))
        out = np.zeros((int(self._params.n_replicas), int(rows.value), n + 1, 2), np.float64)
        _check(self._L, self._L.hs_read_bucket_percentiles(self._h, out.ctypes.data))
        return out

    def read_bucket_percentile_totals(self, n_cells: int, rows: int, n: int):
        """BUCKET_PCT_TOTAL_DTYPE [n_cells, rows, n + 1]: the last run's bucket percentiles reduced per sweep cell
        (hs_read_bucket_percentile_totals)."""
        out = np.zeros((n_cells, rows, n + 1), A.BUCKET_PCT_TOTAL_DTYPE)
        _check(self._L, self._L.hs_read_bucket_percentile_totals(self._h, out.ctypes.data, n_cells))
        return out

    def read_box(self, which: str = "outbox"):
        """(entries XEVENT_DTYPE[n_replicas, cap], counts uint32[n_replicas]) of the partition's outbox / inbox."""
        cap = int(self._model.outbox_cap if which == "outbox" else self._model.inbox_cap)
        n = int(self._params.n_replicas)
        buf, cnt = np.zeros((n, max(1, cap)), A.XEVENT_DTYPE), np.zeros(n, np.uint32)
        fn = self._L.hs_read_outbox if which == "outbox" else self._L.hs_read_inbox
        _check(self._L, fn(self._h, buf.ctypes.data, cnt.ctypes.data_as(C.POINTER(C.c_uint32))))
        return buf, cnt

    def run(self, params: A.RunParams) -> None:
        _check(self._L, self._L.hs_run(self._h, C.byref(params)))
        self._params = params

    def sync(self) -> None:
        _check(self._L, self._L.hs_sync(self._h))

    def last_run_ms(self) -> float:
        ms = C.c_float()
        _check(self._L, self._L.hs_last_run_ms(self._h, C.byref(ms)))
        return float(ms.value)

    def launch_count(self) -> int:
        n = C.c_uint64()
        _check(self._L, self._L.hs_launch_count(self._h, C.byref(n)))
        return int(n.value)

    def last_launch(self) -> dict:
        """The kernel the last run launched and its geometry (hs_last_launch): engine, kernel family ("lane", "warp",
        "thread", "thread_wide"), template flags, lane_stride, heap_top, grid, block, smem."""
        li = A.LaunchInfo()
        _check(self._L, self._L.hs_last_launch(self._h, C.byref(li)))
        d = {f: int(getattr(li, f)) for f, _ in A.LaunchInfo._fields_}
        d["kernel"] = A.KERNEL_NAMES[d["kernel"]]
        return d

    def alloc_host_outputs(self, params: A.RunParams | None = None, *, pinned: bool = False):
        """Caller-owned host buffers shaped for ``params`` (numpy; pinned via torch if asked)."""
        p = params or self._params
        ne = self._model.n_entities
        n = p.n_replicas
        keep: list = []

        def mk(shape, dtype):
            if pinned:
                import torch
                nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
                t = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)
                arr = t.numpy()[:nbytes].view(dtype).reshape(shape)
                keep.append(t)
                return arr
            return np.zeros(shape, dtype)

        bufs = {
            "summaries": mk((n,), A.SUMMARY_DTYPE),
            "entity_stats": mk((n, ne), A.STATS_DTYPE),
            "records": mk((n, p.record_cap), A.RECORD_DTYPE) if p.record_cap else None,
            "sink_samples": mk((n, p.sample_cap), A.SAMPLE_DTYPE) if p.sample_cap else None,
            "service_samples": mk((n, p.service_cap), np.float64) if p.service_cap else None,
            "histograms": mk((n, A.HS_HISTOGRAM_BINS), np.uint32) if (p.flags & A.HS_RUN_HISTOGRAM) else None,
            "sketches": mk((n, self._model.sketch_layout()[2]), np.uint8) if self._model.sketch_layout()[2] else None,
        }
        bufs["_keep"] = keep
        return bufs

    def read_outputs(self, bufs: dict | None = None) -> dict:
        if bufs is None:
            bufs = self.alloc_host_outputs()
        o = A.Outputs()
        o.summaries = bufs["summaries"].ctypes.data_as(C.POINTER(A.ReplicaSummary))
        o.entity_stats = bufs["entity_stats"].ctypes.data_as(C.POINTER(A.EntityStats))
        if bufs.get("records") is not None:
            o.records = bufs["records"].ctypes.data_as(C.POINTER(A.EventRecord))
        if bufs.get("sink_samples") is not None:
            o.sink_samples = bufs["sink_samples"].ctypes.data_as(C.POINTER(A.SinkSample))
        if bufs.get("service_samples") is not None:
            o.service_samples = bufs["service_samples"].ctypes.data_as(C.POINTER(C.c_double))
        if bufs.get("histograms") is not None:
            o.histograms = bufs["histograms"].ctypes.data_as(C.POINTER(C.c_uint32))
        if bufs.get("sketches") is not None:
            o.sketches = bufs["sketches"].ctypes.data_as(C.POINTER(C.c_uint8))
        _check(self._L, self._L.hs_read_outputs(self._h, C.byref(o)))
        return bufs

    def read_sketches(self) -> dict:
        """The last run's sketches merged over its replicas on the device (HyperLogLog.merge = register
        max, CountMinSketch.merge = counter sum): {entity id: uint8[2^p] | uint64[depth, width]}."""
        total = self._model.sketch_layout()[3]
        img = np.zeros(total, np.uint8)
        _check(self._L, self._L.hs_read_sketches(self._h, img.ctypes.data_as(C.c_void_p), total))
        return self._model.merged_sketch_views(img)

    def read_totals(self) -> A.Totals:
        t = A.Totals()
        _check(self._L, self._L.hs_read_totals(self._h, C.byref(t)))
        return t

    def read_cell_totals(self, n_cells: int):
        """Per-cell aggregates of the last run: list of (totals dict, uint64[64] histogram)."""
        arr = (A.CellTotals * n_cells)()
        _check(self._L, self._L.hs_read_cell_totals(self._h, arr, n_cells))
        return [(totals_to_dict(c.totals), np.array(list(c.histogram), dtype=np.uint64)) for c in arr]

    def totals_device_ptr(self) -> int:
        p = C.c_void_p()
        _check(self._L, self._L.hs_totals_device_ptr(self._h, C.byref(p)))
        return int(p.value)


def totals_to_dict(t: A.Totals) -> dict:
    i, f = list(t.i), list(t.fsum)
    return {"events_processed": i[0], "sink_events": i[1], "server_completions": i[2], "source_ticks": i[3],
            "dropped": i[4], "replicas": i[5], "replicas_flagged": i[6], "sum_final_time_us": i[7],
            "sum_latency": f[0], "sum_latency_sq": f[1], "sum_service": f[2],
            "min_latency": t.fmin, "max_latency": t.fmax}
