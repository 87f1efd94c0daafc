"""Mirror of happysimulator/parallel for partitioned runs.

``ParallelSimulation`` without links runs every partition as its own Simulation (own heap,
own creation counter -- parallel/simulation.py:170-195) and aggregates the summaries exactly
as the reference's ``_build_summary`` does.  Partitions connected by ``PartitionLink``s run under the
windowed coordinator (parallel/coordinator.py:75-227) on the device: one engine per partition, one
``hs_run`` per window and partition, ``hs_coordinator_exchange`` at every barrier (linked.py)."""
from __future__ import annotations

import time as _time

import numpy as np
from dataclasses import dataclass, field
from typing import Any

from . import _abi as A
from .api import Instant, Simulation
from .lowering import UnsupportedModelError
from .results import EntitySummary, SimulationSummary, fault_cancelled, replica_summary, write_back


@dataclass
class SimulationPartition:
    """parallel/partition.py:20-38"""
    name: str
    entities: list = field(default_factory=list)
    sources: list = field(default_factory=list)
    probes: list = field(default_factory=list)
    fault_schedule: Any = None
    trace_recorder: Any = None


@dataclass(frozen=True)
class PartitionLink:
    """parallel/link.py:18-79.  ``latency``: a ConstantLatency / ExponentialLatency (this package's or the
    reference's): the coordinator overrides every cross-partition event's time with send time + a sample of it
    (coordinator.py:207-210).  Without it the reference insists on ``event.time - send_time >= min_latency``
    (coordinator.py:211-221), which no stock component can satisfy -- Entity.forward stamps the event with the current
    time -- so such a link cannot carry a lowered model's events."""
    source_partition: str
    dest_partition: str
    min_latency: float
    latency: Any = None
    packet_loss: float = 0.0

    def __post_init__(self) -> None:
        if self.min_latency <= 0:
            raise ValueError(f"PartitionLink min_latency must be > 0, got {self.min_latency}")
        if not (0.0 <= self.packet_loss < 1.0):
            raise ValueError(f"PartitionLink packet_loss must be in [0, 1), got {self.packet_loss}")
        if self.source_partition == self.dest_partition:
            raise ValueError(f"PartitionLink source and dest must differ, got '{self.source_partition}'")


@dataclass
class ParallelSimulationSummary:
    """parallel/summary.py:11-86"""
    duration_s: float
    total_events_processed: int
    events_per_second: float
    wall_clock_seconds: float
    partitions: dict[str, SimulationSummary] = field(default_factory=dict)
    entities: dict[str, EntitySummary] = field(default_factory=dict)
    partition_wall_times: dict[str, float] = field(default_factory=dict)
    speedup: float = 1.0
    parallelism_efficiency: float = 1.0
    total_windows: int = 0
    total_cross_partition_events: int = 0
    window_size_s: float = 0.0
    barrier_overhead_seconds: float = 0.0
    coordination_efficiency: float = 1.0


def _reaching_rates(lm) -> list[float]:
    """Per partition of a LinkedModel: the summed peak rate of every source whose requests can reach it -- its own
    and those of every partition upstream of it over links, followed transitively.  With sweep cells: the largest
    over the cells, each with its own rates."""
    from .lowering import source_rate_bound
    if lm.n_cells:
        return [max(v) for v in zip(*(_reaching_rates(lm.cell(c)) for c in range(lm.n_cells)))]
    own = [source_rate_bound(m) for m in lm.models]
    upstream: list[set[int]] = [set() for _ in lm.models]
    for p, ls in enumerate(lm.links):
        for l in ls:
            upstream[l.dest].add(p)
    rates = []
    for q in range(lm.n_partitions):
        seen, todo = {q}, [q]
        while todo:
            for p in upstream[todo.pop()] - seen:
                seen.add(p)
                todo.append(p)
        rates.append(sum(own[p] for p in seen))
    return rates


def _events_bound(rate: float, inbox_cap: int, end_ns: int) -> float:
    """First estimate of the Sink samples / service starts one replica of a partition produces (ring sizing):
    ``rate`` is the partition's entry of ``_reaching_rates``.  _run_linked checks the counts against it after the run."""
    return (rate * 4 + 50.0) * (end_ns / 1e9 + 1.0) + 4.0 * max(inbox_cap, 0)


# status bits a linked run reports instead of raising: a tie the reference orders by heapq's array layout (a delivered
# event with another event; any pushed event with a pending fault event), as Simulation.run reports HS_ST_FAULT_TIE
_TIES = A.HS_ST_LINK_TIE | A.HS_ST_FAULT_TIE

_RINGS = (("sample_cap", "n_sink_samples", "Sink sample"), ("service_cap", "n_service_samples", "service time"),
          ("record_cap", "events_processed", "event record"))


def _short_rings(outs, caps) -> list[tuple[int, str, int]]:
    """(partition, cap name, largest count over the replicas) of every recorder ring a linked run wrapped.  A record
    ring of 0 slots is not in use (the partition's samples need no split by entity)."""
    short = []
    for q, (o, c) in enumerate(zip(outs, caps)):
        s = o["summaries"]
        for cap, count, _ in _RINGS:
            n = int(s[count].max()) if len(s) else 0
            if (cap != "record_cap" or c[cap]) and n > c[cap]:
                short.append((q, cap, n))
    return short


def _linked_difference(a, b) -> str | None:
    """What keeps two linked ParallelSimulations from running as the cells of one linked ensemble, or None when they
    can: the same partitions in the same order, partition models of one topology (``api._same_topology``), the same
    links (source, destination, latency kind, which links share a latency object), the same windows and end time, the
    same ``link_buffer`` and device.  Latency means, packet losses, rates, mean service times and concurrency may
    differ: they are the per-cell columns."""
    from .api import _same_topology
    la, lb = a._linked, b._linked
    if la is None or lb is None:
        return "a ParallelSimulation without PartitionLinks"
    if la.names != lb.names:
        return f"partitions {la.names} and {lb.names}"
    for q, name in enumerate(la.names):
        if not _same_topology(la.models[q], lb.models[q]):
            return f"partition {name!r}: the models differ in more than rates, mean service times and concurrency"
        x, y = la.links[q], lb.links[q]
        if [(l.dest, l.latency_kind, l.stream) for l in x] != [(l.dest, l.latency_kind, l.stream) for l in y]:
            return f"partition {name!r}: links differ in destination, latency kind or shared latency objects"
    if la.n_streams != lb.n_streams:
        return "links differ in shared latency objects"
    if la.window_s != lb.window_s:
        return f"window {la.window_s} s and {lb.window_s} s"
    if a._end_ns != b._end_ns:
        return f"end time {a._end_ns} ns and {b._end_ns} ns"
    if a.link_buffer != b.link_buffer:
        return f"link_buffer {a.link_buffer} and {b.link_buffer}"
    if a._device != b._device:
        return f"device {a._device} and {b._device}"
    return None


def _same_linked_topology(a, b) -> bool:
    """Two linked ParallelSimulations that can run as cells of one linked ensemble (``_linked_difference``)."""
    return _linked_difference(a, b) is None


def _replica_status(outs, r: int) -> int:
    st = 0
    for o in outs:
        st |= int(o["summaries"]["status"][r])
    return st


def _run_linked_sweep(sims) -> list:
    """ParallelRunner.run_sweep's ParallelSimulations: (ParallelSimulationSummary, status) per configuration, in order.
    Linked configurations of one topology (``_same_linked_topology``) whose seeds form an arithmetic progression run as
    ONE linked ensemble, configuration k as replica k of cell k with Philox key ``seed_0 + k * (seed_1 - seed_0)`` and
    the replica words of a single run (rid_stride 0), so that each equals its own ``run()``; results are written back
    onto each configuration's own objects.  The others, and ParallelSimulations without links, run one by one."""
    from .linked import LinkedModel
    from .lowering import refresh_fault_cancellation
    res: list = [None] * len(sims)
    groups: list[list[int]] = []
    for i, sm in enumerate(sims):
        if sm._linked is None:
            res[i] = (sm.run(), 0)
            continue
        for m in sm._linked.models:     # cancellations are part of the topology: read them before grouping
            refresh_fault_cancellation(m)
        for g in groups:
            if _same_linked_topology(sims[g[0]], sm):
                g.append(i)
                break
        else:
            groups.append([i])
    for g in groups:
        seeds = [int(sims[i]._seed) for i in g]
        ds = {b - a for a, b in zip(seeds, seeds[1:])}
        if len(g) > 1 and len(ds) <= 1 and min(ds | {0}) >= 0:
            lead = sims[g[0]]
            lm = LinkedModel.from_cells([sims[i]._linked for i in g])
            ring = max(int(getattr(sims[i], "queue_ring", 0) or 0) for i in g)
            outs, delivered, lost, wall, windows = lead._run_linked(
                len(g), 0, lm=lm, seed=seeds[0], seed_stride=ds.pop() if ds else 0, rid_stride=0, queue_ring=ring)
            for k, i in enumerate(g):
                res[i] = (sims[i]._summarise_linked(outs, delivered, lost, wall, windows, replica=k), _replica_status(outs, k))
        else:            # seeds that are not an arithmetic progression: one run each
            for i in g:
                summ = sims[i].run()
                res[i] = (summ, _replica_status(sims[i].last_outputs, 0))
    return res


def _aggregate(summaries: dict[str, SimulationSummary]) -> dict:
    """parallel/summary.py: total events, longest duration, events per second and merged entities of the partitions."""
    total = sum(s.total_events_processed for s in summaries.values())
    duration_s = max((s.duration_s for s in summaries.values()), default=0.0)
    merged = {}
    for s in summaries.values():
        merged.update(s.entities)
    return dict(duration_s=duration_s, total_events_processed=total,
                events_per_second=total / duration_s if duration_s > 0 else 0.0, partitions=summaries, entities=merged)


class ParallelSimulation:
    """parallel/simulation.py:31-284"""

    def __init__(self, partitions, *, start_time=None, end_time=None, duration=None, max_workers=None,
                 links=None, window_size=None, seed: int = 42, device: int = 0):
        if not partitions:
            raise ValueError("At least one partition is required")
        if duration is not None and end_time is not None:
            raise ValueError("Cannot specify both 'duration' and 'end_time'")
        names = [p.name for p in partitions]
        if len(set(names)) != len(names):
            raise ValueError("Partition names must be unique")       # parallel/validation.py
        self._seed = seed
        self._partitions = partitions
        self._device = device
        self._links = list(links or [])
        self._simulations: dict[str, Simulation] = {}
        self._linked = None
        if self._links:
            self._init_linked(start_time, end_time, duration, window_size)
            return
        for k, p in enumerate(partitions):
            self._simulations[p.name] = Simulation(start_time=start_time, end_time=end_time, duration=duration,
                                                   sources=p.sources or None, entities=p.entities or None,
                                                   probes=p.probes or None, trace_recorder=p.trace_recorder,
                                                   fault_schedule=p.fault_schedule, seed=seed, replica=k,
                                                   device=device)

    @property
    def simulations(self) -> dict[str, Simulation]:
        return dict(self._simulations)

    # ---- partitions joined by links --------------------------------------------------------------------------
    def _init_linked(self, start_time, end_time, duration, window_size):
        """parallel/validation.py:19-110 + parallel/simulation.py:84-150: check the declarations, find the events that
        cross partitions (a Server whose downstream lives elsewhere) and lower every partition to a model of its own."""
        from . import _abi as A
        from .api import Instant, _start_schedule
        from .linked import LinkedModel, LinkSpec
        from .lowering import _service, lower
        parts = self._partitions
        names = [p.name for p in parts]
        if start_time is not None and int(start_time.nanoseconds) != 0:
            raise UnsupportedModelError("linked partitions start at Instant.Epoch")
        if duration is not None:
            end_time = Instant.Epoch + duration
        if end_time is None:
            raise UnsupportedModelError("linked partitions need an end time (auto-termination cannot end a Source)")
        self._end_ns = int(end_time.nanoseconds)
        index = {n: k for k, n in enumerate(names)}
        for l in self._links:                                    # validation.py:73-84
            if l.source_partition not in index:
                raise ValueError(f"PartitionLink references unknown source partition '{l.source_partition}'")
            if l.dest_partition not in index:
                raise ValueError(f"PartitionLink references unknown dest partition '{l.dest_partition}'")
        min_lat = min(l.min_latency for l in self._links)
        if window_size is not None and window_size > min_lat:    # validation.py:103-110
            raise ValueError(f"window_size ({window_size}s) must be <= min(link.min_latency) ({min_lat}s)")
        window = float(window_size if window_size is not None else min_lat)
        owner: dict[int, int] = {}
        for k, p in enumerate(parts):                            # validation.py:40-51
            for e in list(p.entities) + list(p.sources) + list(p.probes):
                if id(e) in owner and owner[id(e)] != k:
                    raise ValueError(f"Entity '{getattr(e, 'name', e)}' is in partitions '{names[owner[id(e)]]}' and '{p.name}'")
                owner[id(e)] = k
        streams: dict[int, int] = {}
        out_links: list[list] = [[] for _ in parts]
        slot_of: list[dict[int, int]] = [dict() for _ in parts]    # destination partition -> link slot
        for l in self._links:
            if l.latency is None:
                raise UnsupportedModelError(
                    f"PartitionLink {l.source_partition}->{l.dest_partition} has no latency override: the reference then "
                    "requires event.time - send_time >= min_latency (coordinator.py:211-221), and every stock component "
                    "forwards with the current time, so the reference itself raises on the first cross-partition event")
            kind, mean = _service(l.latency)
            s = streams.setdefault(id(l.latency), len(streams))
            q, d = index[l.source_partition], index[l.dest_partition]
            slot_of[q][d] = len(out_links[q])
            out_links[q].append(LinkSpec(d, kind, mean, float(l.packet_loss), s))
        models, objects = [], []
        hidden = lambda ents: {id(getattr(o, a)) for o in ents for a in ("queue", "driver", "worker")
                               if hasattr(o, "_concurrency_model") and hasattr(o, a)}
        for k, p in enumerate(parts):
            skip = hidden(p.entities)       # a reference script has to list a Server's hidden parts for its router
            ents = [e for e in p.entities if id(e) not in skip]
            remote = {}
            for e in ents:                  # the only edge that may leave a partition: Server -> downstream
                t = getattr(e, "_downstream", None) if hasattr(e, "_concurrency_model") else None
                if t is not None and id(t) in owner and owner[id(t)] != k:
                    d = owner[id(t)]
                    if d not in slot_of[k]:
                        raise ValueError(f"Entity '{getattr(e, 'name', e)}' in partition '{p.name}' references entity "
                                         f"'{getattr(t, 'name', t)}' in partition '{names[d]}' without a PartitionLink "
                                         f"('{p.name}' -> '{names[d]}')")       # validation.py:160-200
                    remote[id(t)] = slot_of[k][d]
            if p.fault_schedule is not None:
                # the partition's own Simulation bootstraps its schedule (parallel/simulation.py:94-104): names resolve
                # among its objects only, sort indices follow its own sources and probes
                _start_schedule(p.fault_schedule, p.sources, ents, p.probes)
            m, objs = lower(p.sources or [], ents, probes=p.probes or None, horizon_s=self._end_ns / 1e9, remote=remote,
                            fault_schedule=p.fault_schedule)
            models.append(m)
            objects.append(objs)
        for k, m in enumerate(models):      # REMOTE rows: the entity's id over there
            m.entities = m.entities.copy()
            for i in m.ids_of(A.HS_ENT_REMOTE):
                d = out_links[k][int(m.entities["i0"][i])].dest
                where = [j for j, o in enumerate(objects[d]) if o is objects[k][i]]
                if not where:
                    raise UnsupportedModelError(f"'{getattr(objects[k][i], 'name', '?')}' is not an entity of partition '{names[d]}'")
                m.entities["i1"][i] = where[0]
            if m.ids_of(A.HS_ENT_REMOTE):
                m.outbox_cap = self.link_buffer
        for q in range(len(parts)):
            for l in out_links[q]:
                models[l.dest].inbox_cap = self.link_buffer * max(1, sum(1 for qq in range(len(parts)) for x in out_links[qq] if x.dest == l.dest))
        # a PriorityQueue server in a partition that receives over a link may see the keys of every partition's sources
        pops = [int(m.entities["i1"][i]) for m in models for i in m.ids_of(A.HS_ENT_SOURCE)
                if int(m.entities["kind"][int(m.entities["target"][i])]) != A.HS_ENT_PROBE]
        for d, m in enumerate(models):
            for i in m.ids_of(A.HS_ENT_SERVER) if m.inbox_cap else ():
                if int(m.entities["i1"][i]) == A.HS_Q_PRIORITY and \
                        (min(pops, default=0) <= 0 or len(objects[d][i]._queue.policy._key.values) < max(pops)):
                    raise UnsupportedModelError(f"server '{getattr(objects[d][i], 'name', '?')}' in partition '{names[d]}': "
                                                "its PriorityByKey table must cover the routing keys of every partition's "
                                                "sources, and every source must draw one")
        self._linked = LinkedModel(models, names, out_links, window_s=window, n_streams=max(1, len(streams)), objects=objects)
        self._linked.validate()
        self._linked.window_ends(self._end_ns)      # raises if the coordinator's clock could not reach the end time

    link_buffer = 256        # cross-partition events one replica may emit per window (class default; overflow is reported)
    queue_ring = 0           # device slots per server queue of a linked run (0: the engine's default); grown and re-run on overflow

    def _run_linked(self, n_replicas: int = 1, replica_index_base: int = 0, buckets=None, bucket_sample_cap: int = 0, *,
                    lm=None, seed=None, seed_stride: int = 0, rid_stride=None, replicas_per_cell: int = 1, queue_ring=None):
        """The linked run of ``self._linked``, or of ``lm`` (a LinkedModel with sweep cells, of this one's topology):
        ring sizing, growth and re-runs.  ``seed`` (default: this simulation's), ``seed_stride``, ``rid_stride`` and
        ``replicas_per_cell`` are LinkedRun.run's."""
        from . import _abi as A
        from . import buckets as _buckets
        from .api import EnsembleStatusError, Instant
        from .linked import LinkedRun
        from .lowering import refresh_fault_cancellation
        if lm is None:
            lm = self._linked
            for m in lm.models:             # FaultHandle.cancel() may have been called since the partitions were lowered
                refresh_fault_cancellation(m)
        seed = self._seed if seed is None else seed
        # a run without cells or strides calls LinkedRun.run exactly as before these existed
        stride_kw = {}
        if lm.n_cells:
            stride_kw["replicas_per_cell"] = replicas_per_cell
        if seed_stride:
            stride_kw["seed_stride"] = seed_stride
        if rid_stride is not None:
            stride_kw["rid_stride"] = rid_stride
        t0 = _time.monotonic()
        run = LinkedRun(lm, device=self._device)
        cap = bucket_sample_cap
        try:
            caps = []
            for m, rate in zip(lm.models, _reaching_rates(lm)):
                if buckets is not None:     # the buckets are the run's time series: no recorder rings
                    caps.append(dict(sample_cap=0, service_cap=0, record_cap=0))
                    continue
                ev = max(64, int(_events_bound(rate, m.inbox_cap, self._end_ns)))
                many = len(m.ids_of(A.HS_ENT_SINK)) + len(m.ids_of(A.HS_ENT_PROBE)) > 1 or len(m.ids_of(A.HS_ENT_SERVER)) > 1
                caps.append(dict(sample_cap=ev, service_cap=ev, record_cap=8 * ev if many else 0))   # records tell the sinks / servers apart
            # The reference's queues are unbounded, the device's are rings: a replica whose ring filled up stopped early
            # (HS_ST_QUEUE_OVERFLOW).  A recorder ring that was too small wrapped: it holds only the last `cap` items,
            # and a wrapped record ring credits samples to the wrong sink / server.  Like Simulation.run(), grow what was
            # too small and run the whole thing again (every window starts from scratch: resume = 0 at window 0, a fresh
            # coordinator) instead of handing that to the caller.  Growth happens before an attempt, so `ring` and
            # `caps` are always what the last attempt ran with.
            # With percentiles, a time bucket that outgrew the sample capacity is no failure either: the whole run is
            # repeated once with the capacity that holds every bucket (as Simulation.run_ensemble's "grow").
            ring = int((getattr(self, "queue_ring", 0) if queue_ring is None else queue_ring) or 0)
            ok = _TIES | (A.HS_ST_BUCKET_OVERFLOW if cap else 0)
            queue_full, short, cap_short, cap_grown = False, [], False, False
            for attempt in range(6):
                if queue_full:
                    ring = max(512, 4 * ring)
                for q, c, n in short:
                    caps[q][c] = 2 * n + 64
                if cap_short:
                    cap = max(_buckets.sample_cap_needed(o["buckets"]) for o in outs if "buckets" in o)
                    cap_grown = True
                bk = dict(buckets=buckets, bucket_sample_cap=cap) if buckets is not None else {}
                outs, (delivered, lost, over) = run.run(seed=seed, end_ns=self._end_ns, n_replicas=n_replicas,
                                                        replica_index_base=replica_index_base, caps=caps, flags=0, queue_ring=ring,
                                                        **bk, **stride_kw)
                status = 0
                for o in outs:
                    status |= int(np.bitwise_or.reduce(o["summaries"]["status"])) if len(o["summaries"]) else 0
                clean = not (status & ~ok) and not over.any()
                queue_full = bool(status & A.HS_ST_QUEUE_OVERFLOW and not (status & ~(A.HS_ST_QUEUE_OVERFLOW | ok))
                                  and not over.any())
                # counts of a run that stopped early mean nothing; a bucketed run has no rings
                short = _short_rings(outs, caps) if clean and buckets is None else []
                cap_short = clean and bool(status & A.HS_ST_BUCKET_OVERFLOW) and not cap_grown
                if not (queue_full or short or cap_short):
                    break
            self.last_queue_ring = ring
        finally:
            run.close()
        if short:
            q, cap, n = short[0]
            what = next(w for c, _, w in _RINGS if c == cap)
            raise RuntimeError(f"linked run: partition '{lm.names[q]}' recorded {n} items into its {what} ring of "
                               f"{caps[q][cap]} device slots ({cap}) in the last of {attempt + 1} attempts; the ring "
                               "wrapped, so its results are not published")
        wall = _time.monotonic() - t0
        bad = [(lm.names[q], int(s)) for q, o in enumerate(outs) for s in o["summaries"]["status"] if int(s) & ~ok]
        if bad or over.any():
            bits = 0
            for _, s_ in bad:
                bits |= s_
            why = []
            if bits & A.HS_ST_QUEUE_OVERFLOW:
                why.append(f"a server queue outgrew {ring} device slots (ParallelSimulation.queue_ring)")
            if (bits & A.HS_ST_LINK_OVERFLOW) or over.any():
                why.append(f"an outbox / inbox outgrew ParallelSimulation.link_buffer = {self.link_buffer}")
            if bits & ~(A.HS_ST_QUEUE_OVERFLOW | A.HS_ST_LINK_OVERFLOW | _TIES):
                why.append(f"status bits {bits & ~(A.HS_ST_QUEUE_OVERFLOW | A.HS_ST_LINK_OVERFLOW | _TIES):#x}")
            raise RuntimeError(f"linked run did not complete cleanly: partition status {bad[:4]}, inbox overflows {int(over.sum())}: "
                               + "; ".join(why))
        if status & A.HS_ST_BUCKET_OVERFLOW:
            st = np.stack([o["summaries"]["status"] for o in outs])
            need = max(_buckets.sample_cap_needed(o["buckets"]) for o in outs if "buckets" in o)
            n_over = int((np.bitwise_or.reduce(st, axis=0) & A.HS_ST_BUCKET_OVERFLOW != 0).sum())
            raise EnsembleStatusError(f"{n_over} of {n_replicas} replicas had a time bucket with more samples than "
                                      f"bucket_sample_cap={cap}; pass bucket_sample_cap={need}", st)
        self.link_ties = int(sum(int(s) & A.HS_ST_LINK_TIE != 0 for o in outs for s in o["summaries"]["status"]))
        self.fault_ties = int(sum(int(s) & A.HS_ST_FAULT_TIE != 0 for o in outs for s in o["summaries"]["status"]))
        self.last_outputs, self.last_delivered, self.last_lost = outs, delivered, lost
        return outs, delivered, lost, wall, run.windows

    def run(self) -> ParallelSimulationSummary:
        if self._linked is not None:
            return self._summarise_linked(*self._run_linked(1))
        return self._run_independent()

    def _summarise_linked(self, outs, delivered, lost, wall, windows, replica: int = 0) -> ParallelSimulationSummary:
        """coordinator.py:123-172: per-partition summaries from the partitions' final state, the aggregate like
        _build_summary; results are written back onto the script's own objects (replica ``replica`` of ``outs``)."""
        lm, r = self._linked, replica
        summaries = {}
        for q, name in enumerate(lm.names):
            write_back(lm.models[q], lm.objects[q], outs[q], r, Instant)
            entities = [o for o in self._partitions[q].entities if any(o is x for x in lm.objects[q])]
            summaries[name] = replica_summary(outs[q]["summaries"][r], wall, entities,
                                              events_cancelled=fault_cancelled(lm.models[q], outs[q]["entity_stats"][r]))
        n = len(summaries)
        return ParallelSimulationSummary(
            **_aggregate(summaries), wall_clock_seconds=wall,
            partition_wall_times={nm: wall / n for nm in summaries}, speedup=1.0, parallelism_efficiency=1.0 / n if n else 1.0,
            total_windows=windows, total_cross_partition_events=int(delivered[r]), window_size_s=lm.window_s)

    def run_ensemble(self, n_replicas: int, replica_index_base: int = 0, *, cells=None, replicas_per_cell: int = 1,
                     buckets=None, bucket_percentiles: bool = False, bucket_sample_cap: int = 64):
        """Linked partitions only: n replicas of the whole ParallelSimulation in one set of launches.  Returns
        {partition name: per-replica outputs (Engine.read_outputs)}, delivered and lost cross-partition events per
        replica.

        ``cells``: linked ParallelSimulations of this one's linked topology (``_same_linked_topology``: they may differ
        in rates, mean service times, concurrency, link latency means and packet losses) and seed, run as the sweep
        cells of this ensemble: replica g runs cell (g / replicas_per_cell) % len(cells), the configuration
        ``cells[cell]``, and draws exactly as replica g of ``cells[cell].run_ensemble(n)``.  Every partition's outputs
        then hold ``cell_totals`` (Engine.read_cell_totals), and bucket totals are per cell.

        ``buckets=(width_s, n)``, ``bucket_percentiles`` and ``bucket_sample_cap`` are those of
        ``Simulation.run_ensemble``: every partition with a Sink, tracker or Probe gets its time buckets (and p50 / p99)
        under the same keys, and ``buckets.bucketed_data(outs[name], obj, replica)`` reads them.  Such a run
        keeps no recorder rings, so its memory does not grow with the horizon.  A bucket with more than
        ``bucket_sample_cap`` samples makes the run repeat once with the capacity that holds them all."""
        from . import buckets as _buckets
        if self._linked is None:
            raise UnsupportedModelError("run_ensemble is for partitions joined by PartitionLinks")
        if int(replicas_per_cell) < 1:
            raise ValueError("replicas_per_cell must be >= 1")
        spec = _buckets.check_spec(buckets, self._end_ns) if buckets is not None else None
        cap = _buckets.check_sample_cap(bucket_sample_cap, spec) if bucket_percentiles else 0
        kw = {}
        if cells is not None:
            kw = dict(lm=self._cells_model(cells), replicas_per_cell=int(replicas_per_cell),
                      queue_ring=max(int(getattr(c, "queue_ring", 0) or 0) for c in [self, *cells]))
        outs, delivered, lost, wall, windows = self._run_linked(n_replicas, replica_index_base, spec, cap, **kw)   # a rank's shard: base = rank * n
        return {n: o for n, o in zip(self._linked.names, outs)}, delivered, lost

    def _cells_model(self, cells):
        """The LinkedModel whose cell c is ``cells[c]``; refuses cells of another linked topology or seed."""
        from .linked import LinkedModel
        from .lowering import refresh_fault_cancellation
        cells = list(cells)
        if not cells:
            raise ValueError("cells must hold at least one ParallelSimulation")
        for k, c in enumerate(cells):
            if not isinstance(c, ParallelSimulation) or c._linked is None:
                raise UnsupportedModelError(f"cells[{k}] is not a ParallelSimulation with PartitionLinks")
            for m in c._linked.models:
                refresh_fault_cancellation(m)
        for m in self._linked.models:
            refresh_fault_cancellation(m)
        for k, c in enumerate(cells):
            why = _linked_difference(self, c)
            if why is not None:
                raise UnsupportedModelError(f"cells[{k}] is not of this ParallelSimulation's linked topology: {why}")
            if int(c._seed) != int(self._seed):
                raise UnsupportedModelError(f"cells[{k}] has seed {c._seed}, this ParallelSimulation {self._seed}: the "
                                            "cells of one ensemble share its seed")
        return LinkedModel.from_cells([c._linked for c in cells])

    def _run_independent(self) -> ParallelSimulationSummary:
        """Independent partitions (parallel/simulation.py:170-195).  Partitions whose lowered models share a
        topology (``api._same_topology``: they differ at most in rates, mean service times and concurrency) are
        the replicas of ONE device launch, replica word = partition index as in the sequential case; the others
        get a launch each.  ``partition_wall_times`` are measured: a launch group's wall time split evenly over
        its partitions; ``speedup`` keeps the reference's definition (sum of partition times / wall time), which
        is ~1 here because launch groups run one after another -- the gain of batching shows in the wall time."""
        from .api import _group_by_topology, _run_many
        t0 = _time.monotonic()
        names = list(self._simulations)
        sims = [self._simulations[n] for n in names]
        summaries, walls = {}, {}
        self.launch_groups = []
        for g in _group_by_topology(sims):
            t1 = _time.monotonic()
            rids = [sims[i]._replica for i in g]
            dr = {b - a for a, b in zip(rids, rids[1:])}
            if len(g) > 1 and len(dr) == 1 and min(dr) > 0:
                res = _run_many([sims[i] for i in g], seed=self._seed, seed_stride=0, rid_base=rids[0], rid_stride=dr.pop())
            else:
                res = [sims[i].run() for i in g]
            dt = _time.monotonic() - t1
            self.launch_groups.append([names[i] for i in g])
            for i, r in zip(g, res):
                summaries[names[i]] = r
                walls[names[i]] = dt / len(g)
        summaries = {n: summaries[n] for n in names}
        wall = _time.monotonic() - t0
        seq = sum(walls.values())
        speedup = seq / wall if wall > 0 else 1.0
        n = len(summaries)
        return ParallelSimulationSummary(
            **_aggregate(summaries), wall_clock_seconds=wall, partition_wall_times=walls, speedup=speedup,
            parallelism_efficiency=speedup / n if n else 1.0)
