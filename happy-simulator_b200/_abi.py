"""ctypes mirror of include/hs_b200.h (the C-ABI structs and constants)."""
from __future__ import annotations

import ctypes as C

HS_ABI_VERSION = 7

HS_OK, HS_ERR_INVALID, HS_ERR_CUDA, HS_ERR_NO_DEVICE, HS_ERR_STATE, HS_ERR_OVERFLOW = 0, -1, -2, -3, -4, -5

HS_ENT_SOURCE, HS_ENT_SERVER, HS_ENT_SINK, HS_ENT_COUNTER, HS_ENT_LB, HS_ENT_PROBE, HS_ENT_SKETCH = 1, 2, 3, 4, 5, 6, 7
HS_ENT_CACHE_SERVER = 8
HS_ENT_REMOTE = 9
HS_ENT_FAULT = 10
HS_SK_HLL, HS_SK_CMS, HS_SK_BLOOM, HS_SK_TOPK, HS_SK_TDIGEST, HS_SK_RESERVOIR = 1, 2, 3, 4, 5, 6
METRICS = {"depth": 0, "active_requests": 1, "utilization": 2, "available_capacity": 3, "stats_accepted": 4,
           "stats_dropped": 5, "events_received": 6, "total": 7, "generated_count": 8}
HS_ARR_CONSTANT, HS_ARR_POISSON = 0, 1
HS_SVC_CONSTANT, HS_SVC_EXPONENTIAL = 0, 1
HS_Q_FIFO, HS_Q_LIFO, HS_Q_PRIORITY = 0, 1, 2
HS_LB_ROUND_ROBIN, HS_LB_KEY_TABLE = 0, 1
HS_PROF_CONSTANT, HS_PROF_LINEAR_RAMP, HS_PROF_SPIKE, HS_PROF_STEP = 0, 1, 2, 3

(HS_EV_SOURCE_TICK, HS_EV_REQ_LB, HS_EV_REQ_ENQUEUE, HS_EV_NOTIFY, HS_EV_POLL, HS_EV_DELIVER,
 HS_EV_REQ_WORKER, HS_EV_CONTINUATION, HS_EV_REQ_SINK, HS_EV_LB_RESPONSE, HS_EV_REQ_COUNTER,
 HS_EV_PROBE, HS_EV_REQ_SKETCH, HS_EV_FAULT) = range(14)

EVENT_KIND_NAMES = ["SOURCE_TICK", "REQ_LB", "REQ_ENQUEUE", "NOTIFY", "POLL", "DELIVER",
                    "REQ_WORKER", "CONTINUATION", "REQ_SINK", "LB_RESPONSE", "REQ_COUNTER", "PROBE", "REQ_SKETCH", "FAULT"]

HS_ST_QUEUE_OVERFLOW, HS_ST_FEL_OVERFLOW, HS_ST_REJECT_PATH, HS_ST_TRACE_EXHAUSTED, HS_ST_EVENT_LIMIT = 1, 2, 4, 8, 16
HS_ST_SKETCH_OVERFLOW = 32
HS_RUN_LINKED = 4
HS_ST_LINK_OVERFLOW = 64
HS_ST_LINK_TIE = 128
HS_ST_FAULT_TIE = 256
HS_ST_BUCKET_OVERFLOW = 512

HS_STREAM_ARRIVAL, HS_STREAM_SERVICE, HS_STREAM_ROUTING, HS_STREAM_LINK_LOSS, HS_STREAM_LINK_LATENCY = 0, 1, 2, 3, 4

HS_TOTALS_I64, HS_TOTALS_F64_SUM = 8, 3


class EntityDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("target", C.c_int32), ("i0", C.c_int32), ("i1", C.c_int32),
                ("i2", C.c_int32), ("i3", C.c_int32), ("l0", C.c_int64), ("d0", C.c_double),
                ("d1", C.c_double)]


class ModelDesc(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("n_entities", C.c_uint32),
                ("entities", C.POINTER(EntityDesc)),
                ("n_backends", C.c_uint32), ("key_population", C.c_uint32),
                ("backends", C.POINTER(C.c_int32)), ("key_table", C.POINTER(C.c_int32)),
                ("n_cells", C.c_uint32), ("outbox_cap", C.c_uint32),
                ("cell_d0", C.POINTER(C.c_double)), ("cell_i0", C.POINTER(C.c_int32)),
                ("n_profiles", C.c_uint32), ("inbox_cap", C.c_uint32), ("profiles", C.c_void_p),
                ("n_sketch_table", C.c_uint32), ("n_key_cdf", C.c_uint32),
                ("sketch_tables", C.POINTER(C.c_int32)), ("key_cdf", C.POINTER(C.c_double)),
                ("profile_table", C.POINTER(C.c_double)), ("n_profile_table", C.c_uint64)]


class LinkDesc(C.Structure):
    _fields_ = [("latency_kind", C.c_int32), ("stream", C.c_int32), ("latency_mean_s", C.c_double),
                ("packet_loss", C.c_double)]


class RunParams(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("seed_stride", C.c_uint64),
                ("rid_base", C.c_uint32), ("rid_stride", C.c_uint32),
                ("end_ns", C.c_int64),
                ("n_replicas", C.c_uint32), ("replica_index_base", C.c_uint32),
                ("replicas_per_cell", C.c_uint32), ("record_cap", C.c_uint32),
                ("sample_cap", C.c_uint32), ("service_cap", C.c_uint32),
                ("queue_ring", C.c_uint32), ("engine", C.c_uint32),
                ("window_end_ns", C.c_int64), ("resume", C.c_uint32), ("flags", C.c_uint32),
                ("max_events", C.c_int64)]


class ReplicaSummary(C.Structure):
    _fields_ = [("events_processed", C.c_int64), ("final_time_ns", C.c_int64),
                ("order_hash", C.c_uint64), ("next_sort_index", C.c_uint64),
                ("n_sink_samples", C.c_int64), ("n_service_samples", C.c_int64),
                ("heap_left", C.c_int32), ("status", C.c_uint32)]


class EntityStats(C.Structure):
    _fields_ = [("c0", C.c_int64), ("c1", C.c_int64), ("c2", C.c_int64), ("c3", C.c_int64),
                ("f0", C.c_double), ("f1", C.c_double), ("f2", C.c_double), ("f3", C.c_double)]


class EventRecord(C.Structure):
    _fields_ = [("time_ns", C.c_int64), ("sort_index", C.c_uint32), ("kind", C.c_uint8),
                ("pad", C.c_uint8), ("entity", C.c_uint16)]


class SinkSample(C.Structure):
    _fields_ = [("completion_ns", C.c_int64), ("latency_s", C.c_double)]


class Outputs(C.Structure):
    _fields_ = [("summaries", C.POINTER(ReplicaSummary)), ("entity_stats", C.POINTER(EntityStats)),
                ("records", C.POINTER(EventRecord)), ("sink_samples", C.POINTER(SinkSample)),
                ("service_samples", C.POINTER(C.c_double)), ("histograms", C.POINTER(C.c_uint32)),
                ("sketches", C.POINTER(C.c_uint8))]


class Totals(C.Structure):
    _fields_ = [("i", C.c_int64 * HS_TOTALS_I64), ("fsum", C.c_double * HS_TOTALS_F64_SUM),
                ("fmin", C.c_double), ("fmax", C.c_double)]


class CellTotals(C.Structure):
    _fields_ = [("totals", Totals), ("histogram", C.c_uint64 * 64)]


HS_KERNEL_LANE, HS_KERNEL_WARP, HS_KERNEL_THREAD, HS_KERNEL_THREAD_WIDE = 1, 2, 3, 4
KERNEL_NAMES = {HS_KERNEL_LANE: "lane", HS_KERNEL_WARP: "warp", HS_KERNEL_THREAD: "thread",
                HS_KERNEL_THREAD_WIDE: "thread_wide"}


class LaunchInfo(C.Structure):
    _fields_ = [("engine", C.c_uint32), ("kernel", C.c_uint32), ("flags", C.c_uint32), ("lane_stride", C.c_uint32),
                ("heap_top", C.c_uint32), ("grid", C.c_uint32), ("block", C.c_uint32), ("smem", C.c_uint32)]


assert C.sizeof(EntityDesc) == 48
assert C.sizeof(ReplicaSummary) == 56
assert C.sizeof(EntityStats) == 64
assert C.sizeof(EventRecord) == 16
assert C.sizeof(SinkSample) == 16
assert C.sizeof(RunParams) == 88
assert C.sizeof(LaunchInfo) == 32
HS_RUN_ORDER_HASH = 1
HS_RUN_HISTOGRAM = 2
HS_HISTOGRAM_BINS = 64

# numpy views of the same layouts (host buffers are numpy structured arrays)
import numpy as _np

SUMMARY_DTYPE = _np.dtype([("events_processed", "<i8"), ("final_time_ns", "<i8"), ("order_hash", "<u8"),
                           ("next_sort_index", "<u8"), ("n_sink_samples", "<i8"), ("n_service_samples", "<i8"),
                           ("heap_left", "<i4"), ("status", "<u4")])
STATS_DTYPE = _np.dtype([("c0", "<i8"), ("c1", "<i8"), ("c2", "<i8"), ("c3", "<i8"),
                         ("f0", "<f8"), ("f1", "<f8"), ("f2", "<f8"), ("f3", "<f8")])
RECORD_DTYPE = _np.dtype([("time_ns", "<i8"), ("sort_index", "<u4"), ("kind", "u1"), ("pad", "u1"),
                          ("entity", "<u2")])
SAMPLE_DTYPE = _np.dtype([("completion_ns", "<i8"), ("latency_s", "<f8")])
XEVENT_DTYPE = _np.dtype([("time_ns", "<i8"), ("sort_index", "<u8"), ("created_ns", "<i8"), ("aux", "<u8"), ("key", "<i4"),
                          ("ent", "<i4")])        # hs_xevent, 40 bytes
ENTITY_DTYPE = _np.dtype([("kind", "<i4"), ("target", "<i4"), ("i0", "<i4"), ("i1", "<i4"), ("i2", "<i4"),
                          ("i3", "<i4"), ("l0", "<i8"), ("d0", "<f8"), ("d1", "<f8")])
assert SUMMARY_DTYPE.itemsize == 56 and STATS_DTYPE.itemsize == 64 and RECORD_DTYPE.itemsize == 16
assert ENTITY_DTYPE.itemsize == 48
# time buckets (hs_set_buckets): hs_bucket, 32 bytes, and hs_bucket_total, 48 bytes
BUCKET_DTYPE = _np.dtype([("count", "<i8"), ("sum", "<f8"), ("comp", "<f8"), ("max", "<f8")])
BUCKET_TOTAL_DTYPE = _np.dtype([("replicas", "<i8"), ("count", "<i8"), ("sum", "<f8"), ("mean_sum", "<f8"),
                                ("mean_sq_sum", "<f8"), ("max", "<f8")])
assert BUCKET_DTYPE.itemsize == 32 and BUCKET_TOTAL_DTYPE.itemsize == 48
# bucket percentiles (hs_set_bucket_percentiles): hs_bucket_pct_total, 32 bytes
BUCKET_PCT_TOTAL_DTYPE = _np.dtype([("p50_sum", "<f8"), ("p50_sq_sum", "<f8"), ("p99_sum", "<f8"), ("p99_sq_sum", "<f8")])
assert BUCKET_PCT_TOTAL_DTYPE.itemsize == 32
PROFILE_DTYPE = _np.dtype([("kind", "<i4"), ("pad", "<i4"), ("p", "<f8", (4,))])
assert PROFILE_DTYPE.itemsize == 40


def unroll_ring(buf, count: int, cap: int):
    """Items of a flight-recorder ring in stream order (oldest retained first)."""
    count = int(count)
    if count <= cap:
        return buf[:count]
    h = count % cap
    return _np.concatenate([buf[h:cap], buf[:h]])


def histogram_bin_edges_ns():
    """Lower edges (ns) of the 64 latency bins of hs_latency_bin (bin 0 starts at 0)."""
    edges = [0]
    for b in range(1, 64):
        e, m = 10 + (b - 1) // 2, (b - 1) % 2
        edges.append((1 << e) + m * (1 << (e - 1)))
    return _np.array(edges, dtype=_np.int64)
