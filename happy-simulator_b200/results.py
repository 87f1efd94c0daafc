"""Publishing one replica's device outputs: onto the script's own entity objects (``write_back``: ``sink.latencies_s``,
``server._service_times``, sketch states, ...), mirrors or the reference's own classes, and as its ``SimulationSummary``
(``replica_summary``).  Both need only the lowered model and its objects, so every kind of run publishes the same way."""
from __future__ import annotations

import sys
from dataclasses import dataclass, field
from typing import Any

import numpy as np

from . import _abi as A
from . import sketching


@dataclass
class QueueStats:
    """instrumentation/summary.py:14-20"""
    peak_depth: int
    total_accepted: int
    total_dropped: int


@dataclass
class EntitySummary:
    """instrumentation/summary.py:23-44"""
    name: str
    entity_type: str
    events_handled: int
    queue_stats: QueueStats | None = None


@dataclass
class SimulationSummary:
    """instrumentation/summary.py:47-87"""
    duration_s: float
    total_events_processed: int
    events_cancelled: int = 0
    events_per_second: float = 0.0
    wall_clock_seconds: float = 0.0
    entities: dict[str, EntitySummary] = field(default_factory=dict)

    def to_dict(self) -> dict[str, Any]:
        return {"duration_s": self.duration_s, "total_events_processed": self.total_events_processed,
                "events_cancelled": self.events_cancelled, "events_per_second": self.events_per_second,
                "wall_clock_seconds": self.wall_clock_seconds,
                "entities": {k: vars(v) for k, v in self.entities.items()}}


def _dropped_sink_requests(model, rec):
    """Mask of the REQ_SINK records aimed at a sink that a node fault had crashed or paused when the event was popped.
    The engines record and count such an event, but Event.invoke drops it (core/event.py:261-262): it leaves no sample.
    The crashed flag at each record is the set / clear of the last FAULT record of that sink before it."""
    dropped = np.zeros(len(rec), bool)
    fr = model.ids_of(A.HS_ENT_FAULT)
    if not len(fr):
        return dropped
    E = model.entities
    fpos = np.flatnonzero(rec["kind"] == A.HS_EV_FAULT)
    frow = rec["entity"][fpos]
    ftgt, fset = E["target"][frow], E["i1"][frow]
    req = np.flatnonzero(rec["kind"] == A.HS_EV_REQ_SINK)
    for s in np.unique(ftgt):
        p, v = fpos[ftgt == s], fset[ftgt == s]
        q = req[rec["entity"][req] == s]
        k = np.searchsorted(p, q) - 1              # the sink's last FAULT record before each request
        dropped[q[k >= 0]] = v[k[k >= 0]] != 0
    return dropped


def demultiplex(model, out, r: int):
    """Replica ``r``'s Sink samples and service times per entity row: ({sink or probe row: samples, None if none were
    recorded}, {server row: [float]}).  One collector (server) takes the whole stream; several are told apart by the
    entity of each REQ_SINK / PROBE (REQ_WORKER) event record, in stream order, leaving out the requests a crashed sink
    dropped."""
    s = out["summaries"][r]
    sinks = model.ids_of(A.HS_ENT_SINK) + model.ids_of(A.HS_ENT_PROBE)
    servers = model.ids_of(A.HS_ENT_SERVER)
    per_sink = {i: None for i in sinks}
    per_server = {i: [] for i in servers}
    rec = out["records"][r][: int(s["events_processed"])] if out.get("records") is not None else None
    if out.get("sink_samples") is not None:
        samples = out["sink_samples"][r][: int(s["n_sink_samples"])]
        if len(sinks) == 1:
            per_sink[sinks[0]] = samples
        elif rec is not None:
            sel = ((rec["kind"] == A.HS_EV_REQ_SINK) | (rec["kind"] == A.HS_EV_PROBE)) & ~_dropped_sink_requests(model, rec)
            who = rec["entity"][sel][: len(samples)]
            for i in sinks:
                per_sink[i] = samples[who == i]
    if out.get("service_samples") is not None:
        svc = out["service_samples"][r][: int(s["n_service_samples"])]
        if len(servers) == 1:
            per_server[servers[0]] = [float(x) for x in svc]
        elif rec is not None:
            who = rec["entity"][rec["kind"] == A.HS_EV_REQ_WORKER][: len(svc)]
            for ent, x in zip(who, svc):
                per_server[int(ent)].append(float(x))
    return per_sink, per_server


def write_back(model, objects, out, r: int, instant_cls) -> None:
    """Publish replica ``r`` onto ``objects``, the entity objects of ``model``, where the reference's callers look;
    ``sink.completion_times`` hold ``instant_cls`` time points (the mirror's Instant or the reference's)."""
    st = out["entity_stats"][r]
    kinds = model.entities["kind"]
    per_sink, per_server = demultiplex(model, out, r)
    # Probe objects: their ticking is objects[i] (a SOURCE row); the measurement row it targets
    # (kind PROBE, beyond len(objects)) carries the samples
    for i, o in enumerate(objects):
        if int(kinds[i]) == A.HS_ENT_SOURCE and hasattr(o, "data_sink"):
            sm = per_sink.get(int(model.entities["target"][i]))
            if sm is not None:
                o.data_sink._samples = [(float(int(t)) / 1_000_000_000, float(x))
                                        for t, x in zip(sm["completion_ns"], sm["latency_s"])]
    for i, o in enumerate(objects):
        k = int(kinds[i])
        row = st[i]
        if k == A.HS_ENT_SOURCE:
            o._generated_count = int(row["c0"])
            if hasattr(o._event_provider, "_generated"):
                o._event_provider._generated = int(row["c1"])
        elif k == A.HS_ENT_SERVER:
            o._queue.stats_accepted, o._queue.stats_dropped = int(row["c0"]), int(row["c1"])
            if int(model.entities["i1"][i]) == A.HS_Q_PRIORITY:      # PriorityQueue._insert_counter: successful pushes
                o._queue.policy._insert_counter = int(row["c0"])
            o._requests_completed, o._requests_rejected = int(row["c2"]), int(row["c3"])
            o._total_service_time = float(row["f0"])
            o._service_times = per_server[i]
        elif k == A.HS_ENT_CACHE_SERVER:
            o._queue.stats_accepted, o._queue.stats_dropped = int(row["c0"]), int(row["c1"])
            o.stats.requests_processed, o.stats.cache_misses, o.stats.cache_hits = int(row["c2"]), int(row["c3"]), int(row["f0"])
            if out.get("sketches") is not None:
                ins = model.cache_views(out["sketches"])[i][r]
                K = len(ins) - 1
                times = {("customer:unknown" if j == K else f"customer:{j}"): float(t) for j, t in enumerate(ins) if t != 0.0}
                if hasattr(o, "_insert_times"):
                    o._insert_times = times
                elif getattr(o, "_eviction_policy", None) is not None:      # the example's own object, already initialised
                    o._eviction_policy._insert_times = times
        elif k == A.HS_ENT_SINK and hasattr(o, "data"):          # LatencyTracker / ThroughputTracker
            o.count = int(row["c0"])
            sm = per_sink[i]
            if sm is not None:
                one = getattr(o, "_sample_value", None) == "one" or type(o).__name__ == "ThroughputTracker"
                o.data._samples = [(float(int(t)) / 1_000_000_000, 1.0 if one else float(x))
                                   for t, x in zip(sm["completion_ns"], sm["latency_s"])]
        elif k == A.HS_ENT_SINK:
            o.events_received = int(row["c0"])
            o._latency_sum = float(row["f0"])
            sm = per_sink[i]
            if sm is not None:
                o.completion_times = [instant_cls(int(t)) for t in sm["completion_ns"]]
                o.latencies_s = [float(x) for x in sm["latency_s"]]
        elif k == A.HS_ENT_COUNTER:
            o.total = int(row["c0"])
            o.by_type = {"Request": o.total} if o.total else {}
        elif k == A.HS_ENT_LB:
            o._requests_received, o._requests_forwarded = int(row["c0"]), int(row["c1"])
        elif k == A.HS_ENT_SKETCH:
            _write_back_sketch(model, o, i, row, out, r)
    _write_back_crashed(model, objects, st)


def _write_back_crashed(model, objects, st) -> None:
    """Entity._crashed after the run: the action of the last FAULT event that fired on the entity (FAULT events fire
    in (time, sort index) order); entities no fault event reached keep theirs."""
    last = {}
    for i in model.ids_of(A.HS_ENT_FAULT):
        if int(st[i]["c0"]):
            e = model.entities[i]
            key = (int(e["l0"]), int(e["i3"]))
            tgt = int(e["target"])
            if tgt not in last or key > last[tgt][0]:
                last[tgt] = (key, bool(int(e["i1"])))
    for tgt, (_, crashed) in last.items():
        objects[tgt]._crashed = crashed


def fault_cancelled(model, st) -> int:
    """SimulationSummary.events_cancelled of one replica (``st`` its entity stats): the FAULT events popped while
    cancelled."""
    return int(sum(int(st[i]["c1"]) for i in model.ids_of(A.HS_ENT_FAULT)))


def _write_back_sketch(model, o, i: int, row, out, r: int) -> None:
    """A sketch collector's count and sketch state.  The mirror's sketches load the device state themselves; the
    reference's get their own fields filled, TopK / TDigest / Reservoir cells rebuilt from their own classes."""
    o._events_processed = int(row["c0"])
    sk = o._topk if hasattr(o, "_topk") else o._tdigest if hasattr(o, "_tdigest") else o._sketch
    if out.get("sketches") is None:
        return
    state = model.sketch_views(out["sketches"])[i][r]
    if hasattr(sk, "_load_device_state"):
        sk._load_device_state(state, int(row["c1"]))
        return
    algo = int(model.entities["i0"][i])
    if algo == A.HS_SK_HLL:
        sk._registers = [int(x) for x in state]
    elif algo == A.HS_SK_CMS:
        sk._counters = [[int(x) for x in rowc] for rowc in state]
    elif algo == A.HS_SK_BLOOM:
        sk._bits = [int(x) for x in state]
        sk._bits_set = sum(bin(w).count("1") for w in sk._bits)
    elif algo == A.HS_SK_RESERVOIR:
        sketching.load_reservoir_state(sk, state)
    else:                                  # TopK / TDigest: rebuild the reference's own cells
        mod = sys.modules[type(sk).__module__]
        if algo == A.HS_SK_TOPK:
            t = sketching.TopK(int(model.entities["i2"][i])); t._load_device_state(state, int(row["c1"]))
            sk._counters = {it: mod._Counter(item=it, count=c[0], error=c[1]) for it, c in t._counters.items()}
        else:
            d = sketching.TDigest(float(model.entities["d0"][i])); d._load_device_state(state)
            sk._centroids = [mod._Centroid(mean=m_, count=c_) for m_, c_ in zip(d._means, d._counts)]
            sk._buffer = list(d._buffer)
            sk._min_value, sk._max_value = d._min_value, d._max_value
    sk._total_count = int(row["c1"])


def entity_summaries(entities) -> dict[str, EntitySummary]:
    """core/simulation.py:560-591: only objects passed as entities=, events_handled from
    count | events_received | stats_processed, queue stats for queued resources."""
    res = {}
    for o in entities:
        qs = None
        if hasattr(o, "_queue") and hasattr(o, "_concurrency_model"):
            qs = QueueStats(peak_depth=0, total_accepted=o.stats_accepted, total_dropped=o.stats_dropped)
        handled = 0
        for attr in ("count", "events_received", "stats_processed"):
            v = getattr(o, attr, None)
            if isinstance(v, int):
                handled = v
                break
        res[o.name] = EntitySummary(name=o.name, entity_type=type(o).__name__, events_handled=handled, queue_stats=qs)
    return res


def replica_summary(row, wall_s: float, entities, events_cancelled: int = 0) -> SimulationSummary:
    """The SimulationSummary of one replica: its hs_replica_summary ``row``, the run's wall time and the summaries of
    ``entities`` (read after write_back has published the replica onto them)."""
    duration_s = float(int(row["final_time_ns"])) / 1_000_000_000
    ev = int(row["events_processed"])
    return SimulationSummary(duration_s=duration_s, total_events_processed=ev, events_cancelled=int(events_cancelled),
                             events_per_second=ev / duration_s if duration_s > 0 else 0.0,
                             wall_clock_seconds=wall_s, entities=entity_summaries(entities))
