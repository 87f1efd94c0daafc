"""Lowering: the object graph ``Simulation.__init__`` receives -> FlatModel.

Works by duck typing on the attribute names of the reference's classes, so it accepts
both this package's mirror classes (api.py) and the reference's own objects
(happysimulator.*): ``Source._event_provider/_time_provider``, ``Server._queue /
_concurrency_model / _service_time / _downstream``, ``LoadBalancer._strategy /
_backends``, ``Sink``, ``Counter``.  Anything it does not recognise raises
``UnsupportedModelError`` naming the object -- a model is never silently approximated
and there is no CPU fallback.

Reference anchors: Simulation.__init__ (core/simulation.py:95-102), Entity.downstream_entities
(core/entity.py:115-127), Source (load/source.py:92-118), Server (components/server/server.py:64-122),
LoadBalancer (components/load_balancer/load_balancer.py:74-125), ConsistentHash
(components/load_balancer/strategies.py:336-433).
"""
from __future__ import annotations

import bisect
import hashlib
import struct
import math

import numpy as np

from . import _abi as A
from .model import ModelBuilder


class UnsupportedModelError(NotImplementedError):
    pass


def _cls(o) -> str:
    return type(o).__name__


def _ns(x) -> int:
    """Instant/Duration -> ns (both the reference's and ours expose .nanoseconds)."""
    return int(x.nanoseconds)


def consistent_hash_table(backend_names, virtual_nodes: int, population: int) -> np.ndarray:
    """key k (as the reference stringifies it, str(k)) -> index of the backend ConsistentHash.select
    returns: the first ring point >= md5(key), wrapping to ring[0] (strategies.py:371-433).  The
    reference scans the ring linearly; a bisect over the sorted ring gives the same point."""
    ring = []
    for bi, name in enumerate(backend_names):
        for i in range(virtual_nodes):
            h = int(hashlib.md5(f"{name}:{i}".encode()).hexdigest(), 16)
            ring.append((h, name, bi))
    # add_backend re-sorts by hash only (stable): equal hashes keep insertion order
    ring.sort(key=lambda x: x[0])
    hashes = [h for h, _, _ in ring]
    tab = np.zeros(population, np.int32)
    for k in range(population):
        hv = int(hashlib.md5(str(k).encode()).hexdigest(), 16)
        j = bisect.bisect_left(hashes, hv)
        tab[k] = ring[j][2] if j < len(ring) else ring[0][2]
    return tab


HASH_ON_DEVICE_ABOVE = 100_000      # key populations beyond this are hashed per event on the device (K = 0 rows)


def zipf_cdf(population: int, s: float) -> np.ndarray:
    """ZipfDistribution._cum_probs for values range(population) (distributions/zipf.py:96-110): weights
    1 / (k + 1)^s, normalised by Python's float sum(), accumulated left to right, last entry forced to 1.0.
    Computed with the very same Python float operations, so bisect_left on it picks the reference's keys."""
    n = int(population)
    if s == 0:
        probs = [1.0 / n] * n
    else:
        w = [1.0 / ((k + 1) ** s) for k in range(n)]
        total = sum(w)
        probs = [x / total for x in w]
    cum, run = [], 0.0
    for p in probs:
        run += p
        cum.append(run)
    cum[-1] = 1.0
    return np.array(cum, dtype=np.float64)


def hll_table(precision: int, seed: int | None, population: int) -> np.ndarray:
    """HyperLogLog.add's hashing evaluated once per key (sketching/hyperloglog.py:128-165):
    h = first 8 bytes (big endian) of sha256(pack(">Q", seed) + repr(k)); register index = h >> (64 - p),
    run length = leading zeros of the low (64 - p) bits + 1.  -> int32[2, K]."""
    p = int(precision)
    seed = 0 if seed is None else int(seed)
    tab = np.zeros((2, population), np.int32)
    low_bits = 64 - p
    for k in range(population):
        h = int.from_bytes(hashlib.sha256(struct.pack(">Q", seed) + repr(k).encode("utf-8")).digest()[:8], "big")
        rest = h & ((1 << low_bits) - 1)
        tab[0, k] = h >> low_bits
        tab[1, k] = (low_bits - rest.bit_length()) + 1      # all-zero rest: low_bits leading zeros
    return tab


def cms_table(width: int, depth: int, seed: int | None, population: int) -> np.ndarray:
    """CountMinSketch._hash per (row, key) (sketching/count_min_sketch.py:136-155): row seeds =
    sha256(pack(">QQ", seed, row))[:8]; column = sha256(pack(">Q", (hash(k) ^ row_seed) & (2^64 - 1)))[:8] % width,
    with hash(k) == k for the non-negative int keys the device generates.  -> int32[depth, K]."""
    seed = 0 if seed is None else int(seed)
    tab = np.zeros((depth, population), np.int32)
    for row in range(depth):
        rs = int.from_bytes(hashlib.sha256(struct.pack(">QQ", seed, row)).digest()[:8], "big")
        for k in range(population):
            c = (hash(k) ^ rs) & 0xFFFFFFFFFFFFFFFF
            tab[row, k] = int.from_bytes(hashlib.sha256(struct.pack(">Q", c)).digest()[:8], "big") % width
    return tab


def bloom_table(size_bits: int, num_hashes: int, seed: int | None, population: int) -> np.ndarray:
    """BloomFilter._hash per (hash i, key) (sketching/bloom_filter.py:147-160): digest = sha256(pack(">QQ", seed, i)
    + repr(k)); bit = (digest[0:8] + i * digest[8:16]) mod size_bits (big-endian words).  -> int32[num_hashes, K]."""
    seed = 0 if seed is None else int(seed)
    tab = np.zeros((num_hashes, population), np.int32)
    for i in range(num_hashes):
        pre = struct.pack(">QQ", seed, i)
        for k in range(population):
            dg = hashlib.sha256(pre + repr(k).encode("utf-8")).digest()
            tab[i, k] = (int.from_bytes(dg[:8], "big") + i * int.from_bytes(dg[8:16], "big")) % size_bits
    return tab


def profile_max_rate(pr, tables=None) -> float:
    """Largest rate a lowered profile row can return (buffer sizing only)."""
    kind = int(pr["kind"])
    if kind == A.HS_PROF_LINEAR_RAMP:
        return float(max(pr["p"][1:3]))
    if kind == A.HS_PROF_STEP:
        off, n = int(pr["p"][0]), int(pr["p"][1])
        return float(np.max(tables[off + n: off + 2 * n + 1]))
    return float(max(pr["p"][0:2]))


def source_rate_bound(model) -> float:
    """Sum over ``model``'s SOURCE rows of the largest rate each can reach: ``d0`` for a constant rate, the
    profile's peak (``profile_max_rate``) otherwise -- a profile source is lowered with d0 = 0 (buffer sizing only)."""
    ents = model.entities
    rate = 0.0
    for i in model.ids_of(A.HS_ENT_SOURCE):
        pi = int(ents["i3"][i])
        if pi == 0:
            rate += float(ents["d0"][i])
        else:
            rate += profile_max_rate(model.profiles[pi - 1], model.profile_table)
    return rate


class _Seconds:
    """Stand-in for an Instant when probing a user's Profile.get_rate: the reference evaluates
    ``profile.get_rate(Instant.from_seconds(t))`` and profiles read ``time.to_seconds()`` (load/profile.py:37-110),
    i.e. float(int(t * 1e9)) / 1e9 -- the rate is a function of the NANOSECOND count."""
    __slots__ = ("nanoseconds",)

    def __init__(self, ns: int):
        self.nanoseconds = int(ns)

    def to_seconds(self) -> float:
        return float(self.nanoseconds) / 1_000_000_000


def step_table_from_profile(profile, scan_end_s: float, scan_step_s: float | None = None, max_pieces: int = 4096):
    """Tabulate a piecewise-constant ``Profile.get_rate`` exactly: (breakpoints, rates) with
    ``rates[number of breakpoints <= t] == profile.get_rate(t)`` for every t the arrival solver can ask about.

    get_rate only ever sees times of the form float(ns) / 1e9, so the function is scanned on the integer
    nanosecond axis: a coarse grid finds the pieces, bisection on ns finds the first nanosecond of each new piece,
    and that nanosecond's to_seconds() value is the breakpoint -- ``t >= b`` then holds for exactly the same ns
    counts as in the user's own comparisons, whatever arithmetic they use (e.g. int((t - 65.0) / 11.0),
    examples/queuing/m_m_1_queue.py:160-166).  Assumptions, checked where they can be: the function is constant
    between changes (a second scan on an offset grid must agree with the table), pieces are not shorter than the
    scan step, and the profile keeps its last value beyond ``scan_end_s``.  Raises UnsupportedModelError for
    anything that is not a step function."""
    step = scan_step_s or max(1e-3, scan_end_s / 400_000.0)
    end_ns = int(scan_end_s * 1e9)
    step_ns = max(1, int(step * 1e9))

    def f(ns):
        return float(profile.get_rate(_Seconds(ns)))

    grid = list(range(0, end_ns + step_ns, step_ns))
    vals = [f(ns) for ns in grid]
    breaks_ns, rates = [], [vals[0]]
    for a, b, va, vb in zip(grid, grid[1:], vals, vals[1:]):
        if va == vb:
            continue
        lo, hi = a, b                         # f(lo) == va, f(hi) != va: first ns with a different value
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if f(mid) == va:
                lo = mid
            else:
                hi = mid
        if f(hi) != vb:
            raise UnsupportedModelError(f"profile {_cls(profile)}: two rate changes within one scan step of {step} s "
                                        f"near t = {a / 1e9} s (pass a smaller scan_step_s) or not a step function")
        breaks_ns.append(hi)
        rates.append(vb)
        if len(rates) > max_pieces:
            raise UnsupportedModelError(f"profile {_cls(profile)}: more than {max_pieces} pieces -- a continuously "
                                        "varying get_rate is a Python callback and cannot run on the device")
    breaks = [float(ns) / 1_000_000_000 for ns in breaks_ns]
    # verification on an offset grid: the table must reproduce the function
    import bisect
    for ns in range(step_ns // 3, end_ns, max(step_ns, (end_ns // 50_000) or 1)):
        if rates[bisect.bisect_right(breaks, float(ns) / 1_000_000_000)] != f(ns):
            raise UnsupportedModelError(f"profile {_cls(profile)} is not piecewise constant at the scan resolution "
                                        f"({step} s): table and get_rate disagree at t = {ns / 1e9} s")
    if any(not (r > 0.0) for r in rates):
        raise UnsupportedModelError(f"profile {_cls(profile)}: rates must stay > 0 (a zero rate sends the reference's "
                                    "bracket search beyond the int64 nanosecond range)")
    return breaks, rates


def _arrival(tp, horizon_s: float | None = None):
    """ArrivalTimeProvider -> (HS_ARR_*, rate, profile tuple or None).  The reference's built-in
    profile classes (load/profile.py) are lowered as they are; ``StepProfile`` tables directly; any other
    user-defined Profile is tabulated as a step function over the run's horizon when it is one
    (``step_table_from_profile``) -- a continuously varying get_rate is a Python callback and cannot run on
    the device."""
    name = _cls(tp)
    prof = getattr(tp, "profile", None)
    pname = _cls(prof)
    rate, ptuple = 0.0, None
    if pname == "ConstantRateProfile":
        rate = float(prof.rate)
    elif pname == "LinearRampProfile":
        ptuple = ("linear_ramp", float(prof.duration_s), float(prof.start_rate), float(prof.end_rate))
    elif pname == "SpikeProfile":
        ptuple = ("spike", float(prof.baseline_rate), float(prof.spike_rate), float(prof.warmup_s),
                  float(prof.spike_duration_s))
    elif hasattr(prof, "breakpoints") and hasattr(prof, "rates"):           # happysim_b200.StepProfile
        ptuple = ("step", [float(x) for x in prof.breakpoints], [float(x) for x in prof.rates])
    elif prof is not None and hasattr(prof, "get_rate") and horizon_s is not None:
        # the arrival solver brackets beyond the current time (arrival_time_provider.py:100-120): scan well past the run's end
        breaks, rates = step_table_from_profile(prof, scan_end_s=2.0 * float(horizon_s) + 120.0)
        ptuple = ("step", breaks, rates)
    else:
        raise UnsupportedModelError(f"arrival profile {pname}: ConstantRateProfile, LinearRampProfile, SpikeProfile and "
                                    "step functions (StepProfile, or any piecewise-constant get_rate when the run's "
                                    "horizon is known) are lowered; a continuously varying get_rate is a Python callback")
    if "Poisson" in name:
        return A.HS_ARR_POISSON, rate, ptuple
    if "Constant" in name:
        return A.HS_ARR_CONSTANT, rate, ptuple
    raise UnsupportedModelError(f"arrival time provider {name}")


def _service(dist):
    name = _cls(dist)
    mean = float(dist._mean_latency)
    if "Exponential" in name:
        return A.HS_SVC_EXPONENTIAL, mean
    if "Constant" in name:
        return A.HS_SVC_CONSTANT, mean
    raise UnsupportedModelError(f"service time distribution {name}")


def _queue_policy(q, *, owner: str = "?", key_population: int = 0, priority: bool = False):
    """-> (HS_Q_*, capacity or -1, priority table or None).  ``priority``: a PriorityQueue is lowered (Server rows);
    its key must be a ``PriorityByKey`` whose table covers ``key_population``, the largest key population of the
    model's sources."""
    pol = q.policy
    name = _cls(pol)
    if name not in ("FIFOQueue", "LIFOQueue") and not (priority and name == "PriorityQueue"):
        raise UnsupportedModelError(f"queue policy {name}")
    cap = pol.capacity
    cap = -1 if (isinstance(cap, float) and math.isinf(cap)) else int(cap)
    if name != "PriorityQueue":
        return (A.HS_Q_LIFO if name == "LIFOQueue" else A.HS_Q_FIFO), cap, None
    return A.HS_Q_PRIORITY, cap, _priority_table(getattr(pol, "_key", None), owner, key_population)


def _priority_table(key, owner: str, key_population: int) -> list[float]:
    """PriorityQueue._get_priority (queue_policy.py:245-253) as a table over the routing key."""
    if key is None:
        raise UnsupportedModelError(f"server {owner!r}: PriorityQueue without a key -- the reference falls back to "
                                    "float(event), which raises TypeError on the first push; use "
                                    "PriorityQueue(key=happysim_b200.PriorityByKey(values))")
    if not getattr(key, "priority_by_routing_key", False):
        raise UnsupportedModelError(f"server {owner!r}: PriorityQueue key {_cls(key)} is a Python callback and cannot run "
                                    "on the device (use happysim_b200.PriorityByKey(values): priority = values[routing key])")
    if key_population <= 0:
        raise UnsupportedModelError(f"server {owner!r}: PriorityByKey reads the request's routing key, and no source of the "
                                    "model draws one (context['metadata'] would be missing): use UniformKeyContext / "
                                    "ZipfKeyContext")
    values = list(key.values)
    if len(values) < key_population:
        raise UnsupportedModelError(f"server {owner!r}: PriorityByKey has {len(values)} values, the sources draw keys "
                                    f"from {key_population}")
    table = []
    for k, v in enumerate(values):
        if not isinstance(v, (int, float)):
            raise UnsupportedModelError(f"server {owner!r}: priority of key {k} is a {type(v).__name__} (int, float or "
                                        "bool only)")
        if isinstance(v, int) and abs(v) > 1 << 53:
            raise UnsupportedModelError(f"server {owner!r}: priority of key {k} ({v}) is an int a double cannot hold exactly")
        if isinstance(v, float) and math.isnan(v):
            raise UnsupportedModelError(f"server {owner!r}: priority of key {k} is NaN (it orders against nothing)")
        table.append(float(v))
    return table


def fault_events(fault_schedule, sources, entities, probes):
    """The node-fault events of ``fault_schedule`` (the reference's faults.FaultSchedule or the mirror's), in bootstrap
    order: a list of (target object, time_ns, crash, sort_index, event).  ``event`` is the Event (or the mirror's
    stand-in) whose ``_cancelled`` flag a FaultHandle.cancel() sets; it is read again when the model runs.

    Names resolve as FaultSchedule._build_context does (faults/schedule.py:112-135): the ``.name`` of every object in
    entities, sources and probes, in that order, the last one winning; an unknown name raises KeyError.  CrashNode
    gives a crash event at ``at`` and, with ``restart_at``, a restart event; PauseNode a pause at ``start`` and a
    resume at ``end`` (faults/node_faults.py:41-128).  Times and sort indices are those of the events the schedule
    generated when the Simulation was built; a schedule that has not generated them yet gets the times
    Instant.from_seconds gives and the indices that follow the sources' and probes' first ticks."""
    by_name = {}
    for o in list(entities or []) + list(sources or []) + list(probes or []):
        by_name[getattr(o, "name", None)] = o
    n_boot = len(list(sources or [])) + len(list(probes or []))
    res = []
    for fault, handle in zip(fault_schedule._faults, fault_schedule._handles):
        cls = _cls(fault)
        if cls == "CrashNode":
            spec = [(fault.at, True)] + ([] if fault.restart_at is None else [(fault.restart_at, False)])
        elif cls == "PauseNode":
            spec = [(fault.start, True), (fault.end, False)]
        else:
            raise UnsupportedModelError(f"fault {cls}: only the node faults CrashNode and PauseNode run on the device "
                                        "(network faults, ReduceCapacity and user-defined Fault classes do not)")
        target = by_name[fault.entity_name]          # KeyError, as ctx.entities[name] raises it
        evs = list(getattr(handle, "_events", []) or [])
        for k, (t_s, crash) in enumerate(spec):
            ev = evs[k] if k < len(evs) else None
            if ev is not None:
                t_ns, idx = int(ev.time.nanoseconds), int(ev._sort_index)
            else:
                t_ns = t_s * 1_000_000_000 if isinstance(t_s, int) else int(t_s * 1_000_000_000)   # Instant.from_seconds
                idx = n_boot
            n_boot = idx + 1
            res.append((target, t_ns, crash, idx, ev))
    return res


def lower(sources, entities, *, key_population: int | None = None, probes=None, horizon_s: float | None = None,
          remote: dict | None = None, fault_schedule=None):
    """-> (FlatModel, objects) where objects[i] is the Python object of entity id i.

    ``remote``: {id(object): link slot} for objects that live in ANOTHER partition of a ParallelSimulation: a Server
    may name one as its downstream; it becomes an HS_ENT_REMOTE row (its destination entity id is filled in by the
    caller once the other partition is lowered, parallel.py).

    ``fault_schedule``: a FaultSchedule of CrashNode / PauseNode faults (see ``fault_events``); every fault event
    becomes an HS_ENT_FAULT row, after all other rows, with its cancelled flag as it is now.

    Entity ids: sources first (in ``sources`` order, the bootstrap order of
    Simulation.__init__), then every entity reachable from them, in ``entities`` order
    first and discovery order after."""
    faults = fault_events(fault_schedule, sources, entities, probes) if fault_schedule is not None else []
    objs: list = []
    ids: dict[int, int] = {}

    def add(o):
        if id(o) not in ids:
            ids[id(o)] = len(objs)
            objs.append(o)
        return ids[id(o)]

    for s in sources or []:
        add(s)
    for p_ in probes or []:          # Simulation.__init__ bootstraps probes right after the sources
        add(p_)
    for e in entities or []:
        add(e)

    remote = remote or {}

    def kind_of(o):
        n = _cls(o)
        if id(o) in remote:
            return A.HS_ENT_REMOTE
        if hasattr(o, "_event_provider") and hasattr(o, "_time_provider"):
            return "probe" if _cls(o._event_provider) == "_ProbeEventProvider" else A.HS_ENT_SOURCE
        if hasattr(o, "_concurrency_model") and hasattr(o, "_service_time") and hasattr(o, "_queue"):
            return A.HS_ENT_SERVER
        if all(hasattr(o, a) for a in ("_cache_capacity", "_cache_ttl_s", "_cache_read_latency_s",
                                       "_datastore_read_latency_s", "_processing_latency_s", "_queue")):
            return A.HS_ENT_CACHE_SERVER          # examples/load-balancing/common.py:100 CachingServer (or the mirror)
        if hasattr(o, "latencies_s") and hasattr(o, "events_received"):
            return A.HS_ENT_SINK
        if hasattr(o, "data") and hasattr(o, "count") and hasattr(getattr(o, "data"), "_samples") and \
                _cls(o) in ("LatencyTracker", "ThroughputTracker"):
            return A.HS_ENT_SINK        # collectors.py:38-44,76-79: a Sink that appends to a Data
        if hasattr(o, "by_type") and hasattr(o, "total"):
            return A.HS_ENT_COUNTER
        if hasattr(o, "_strategy") and hasattr(o, "_backends") and hasattr(o, "_in_flight"):
            return A.HS_ENT_LB
        if (hasattr(o, "_sketch") or hasattr(o, "_topk") or hasattr(o, "_tdigest")) and hasattr(o, "_value_extractor") \
                and hasattr(o, "_events_processed"):
            return A.HS_ENT_SKETCH
        raise UnsupportedModelError(f"entity {getattr(o, 'name', o)!r} of type {n} cannot be lowered to the device "
                                    "engine (supported: Source, Server, CachingServer, Sink, Counter, LoadBalancer, SketchCollector)")

    # discover downstream objects (they may be missing from entities=, as in the reference)
    i = 0
    while i < len(objs):
        o = objs[i]
        k = kind_of(o)
        if k == "probe":
            add(o._event_provider.target)
        elif k == A.HS_ENT_SOURCE:
            t = getattr(o._event_provider, "_target", None)
            if t is None:
                raise UnsupportedModelError(f"source {o.name!r}: event provider {_cls(o._event_provider)} has no target")
            if id(t) in remote:        # parallel/validation.py:53-71
                raise ValueError(f"Source {o.name!r} targets entity {getattr(t, 'name', t)!r} of another partition")
            add(t)
        elif k == A.HS_ENT_SERVER:
            if o._downstream is not None:
                add(o._downstream)
        elif k == A.HS_ENT_LB:
            for info in o._backends.values():
                if id(info.backend) in remote:
                    raise UnsupportedModelError(f"load balancer {o.name!r}: backend {getattr(info.backend, 'name', '?')!r} lives in "
                                                "another partition (only a Server's downstream may cross a PartitionLink)")
                add(info.backend)
        i += 1

    # the routing keys the model's requests carry: a PriorityByKey table must cover every one, and every request needs one
    source_key_population, unkeyed = 0, []
    for o in objs:
        if kind_of(o) == A.HS_ENT_SOURCE:
            pop_ = int(getattr(getattr(o._event_provider, "_context_fn", None), "key_population", 0) or 0)
            source_key_population = max(source_key_population, pop_)
            if pop_ <= 0:
                unkeyed.append(getattr(o, "name", _cls(o)))
    b = ModelBuilder()
    pending_lb = []
    probe_rows = []
    for o in objs:
        k = kind_of(o)
        name = getattr(o, "name", _cls(o))
        if k == A.HS_ENT_REMOTE:
            b.remote(f"{name}@remote", link=int(remote[id(o)]), dest_entity=0)
            continue
        if k == "probe":
            ep = o._event_provider
            if ep.metric not in A.METRICS:
                raise UnsupportedModelError(f"probe {name!r}: metric {ep.metric!r} (supported: {sorted(A.METRICS)})")
            prof = o._time_provider.profile
            # the measurement row is appended after all objects; patch the target then
            sid = b.source(name, poisson=False, target=-1, profile=("constant", float(prof.rate)))
            probe_rows.append((sid, name, ids[id(ep.target)], ep.metric))
        elif k == A.HS_ENT_SOURCE:
            prov = o._event_provider
            if _cls(prov) not in ("SimpleEventProvider", "_SimpleEventProvider"):
                raise UnsupportedModelError(f"source {name!r}: event provider {_cls(prov)}")
            ctx = getattr(prov, "_context_fn", None)
            pop, cdf = 0, None
            if ctx is not None:
                pop = int(getattr(ctx, "key_population", 0))
                if pop <= 0:
                    raise UnsupportedModelError(f"source {name!r}: arbitrary context_fn callbacks cannot run on the "
                                                "device (use happysim_b200.UniformKeyContext / ZipfKeyContext)")
                if getattr(ctx, "zipf_s", None) is not None:
                    cdf = zipf_cdf(pop, float(ctx.zipf_s))
            kind, rate, ptuple = _arrival(o._time_provider, horizon_s)
            stop = prov._stop_after
            b.source(name, rate=rate, target=ids[id(prov._target)], poisson=(kind == A.HS_ARR_POISSON),
                     stop_after_ns=-1 if stop is None else _ns(stop), key_population=pop, profile=ptuple, key_cdf=cdf)
        elif k == A.HS_ENT_SERVER:
            cm = o._concurrency_model
            if _cls(cm) != "FixedConcurrency":
                raise UnsupportedModelError(f"server {name!r}: concurrency model {_cls(cm)}")
            skind, mean = _service(o._service_time)
            pol, cap, prio = _queue_policy(o._queue, owner=name, key_population=source_key_population, priority=True)
            if prio is not None and unkeyed:
                raise UnsupportedModelError(f"server {name!r}: PriorityByKey reads the request's routing key, and source "
                                            f"{unkeyed[0]!r} draws none (context['metadata'] would be missing)")
            if prio is not None and faults:
                raise UnsupportedModelError(f"server {name!r}: fault schedules do not run in a model with a PriorityQueue server")
            ds = o._downstream
            b.server(name, concurrency=int(cm.limit), mean_service_s=mean, exponential=(skind == A.HS_SVC_EXPONENTIAL),
                     downstream=-1 if ds is None else ids[id(ds)], capacity=cap, lifo=(pol == A.HS_Q_LIFO), priorities=prio)
        elif k == A.HS_ENT_CACHE_SERVER:
            pol, cap, _ = _queue_policy(o._queue)
            if cap >= 0:
                raise UnsupportedModelError(f"caching server {name!r}: bounded queue")
            pop = key_population or max((int(getattr(getattr(s_._event_provider, "_context_fn", None), "key_population", 0))
                                         for s_ in sources or []), default=0)
            if pop <= 0:
                raise UnsupportedModelError(f"caching server {name!r}: the cache key is the request's customer id -- the "
                                            "source needs a finite key population (UniformKeyContext / ZipfKeyContext)")
            if int(o._cache_capacity) <= pop:
                raise UnsupportedModelError(f"caching server {name!r}: cache_capacity {int(o._cache_capacity)} <= key population "
                                            f"{pop}: the cache could fill, and the reference's CachingServer raises "
                                            "FrozenInstanceError on its first eviction (examples/load-balancing/common.py:264)")
            b.cache_server(name, key_slots=pop, cache_ttl_s=float(o._cache_ttl_s),
                           cache_read_latency_s=float(o._cache_read_latency_s),
                           datastore_read_latency_s=float(o._datastore_read_latency_s),
                           processing_latency_s=float(o._processing_latency_s), lifo=(pol == A.HS_Q_LIFO))
        elif k == A.HS_ENT_SINK:
            b.sink(name)
        elif k == A.HS_ENT_COUNTER:
            b.counter(name)
        elif k == A.HS_ENT_SKETCH:
            # sketch_collector.py:79-98: value = value_extractor(event); only "the request's routing key"
            # is a value the device can see
            if hasattr(o, "_tdigest"):              # QuantileEstimator (quantile_estimator.py:35)
                if not getattr(o._value_extractor, "request_latency", False):
                    raise UnsupportedModelError(f"quantile estimator {name!r}: arbitrary value_extractor callbacks "
                                                "cannot run on the device (use happysim_b200.LatencyExtractor())")
                b.sketch_tdigest(name, compression=float(o._tdigest._compression))
                continue
            if not getattr(o._value_extractor, "routing_key", False):
                raise UnsupportedModelError(f"sketch collector {name!r}: arbitrary value_extractor callbacks cannot "
                                            "run on the device (use happysim_b200.KeyExtractor())")
            if getattr(o, "_weight_extractor", None) is not None or getattr(o, "_count_extractor", None) is not None:
                raise UnsupportedModelError(f"sketch collector {name!r}: weight / count extractor callbacks")
            pop = key_population or max((int(getattr(getattr(getattr(s, "_event_provider", None), "_context_fn", None),
                                                     "key_population", 0)) for s in sources or []), default=0)
            if pop <= 0:
                raise UnsupportedModelError(f"sketch collector {name!r}: needs a finite key population")
            sk = o._topk if hasattr(o, "_topk") else o._sketch       # TopKCollector keeps its TopK in _topk
            # large key populations: no per-key table, the device evaluates the SHA-256 hashes per event
            on_device = pop > HASH_ON_DEVICE_ABOVE
            if _cls(sk) == "TopK":
                b.sketch_topk(name, k=int(sk._k), key_population=pop)
            elif _cls(sk) == "BloomFilter":
                b.sketch_bloom(name, size_bits=int(sk._size_bits), num_hashes=int(sk._num_hashes), seed=sk._seed,
                               table=None if on_device else bloom_table(sk._size_bits, sk._num_hashes, sk._seed, pop))
            elif _cls(sk) == "HyperLogLog":
                b.sketch_hll(name, precision=int(sk._precision), seed=sk._seed,
                             table=None if on_device else hll_table(sk._precision, sk._seed, pop))
            elif _cls(sk) == "CountMinSketch":
                b.sketch_cms(name, width=int(sk._width), depth=int(sk._depth), seed=sk._seed,
                             table=None if on_device else cms_table(sk._width, sk._depth, sk._seed, pop))
            elif _cls(sk) == "ReservoirSampler":     # starts from the state the sampler's own generator is in now
                if sk._reservoir or sk._total_count:
                    raise UnsupportedModelError(f"sketch collector {name!r}: the reservoir already holds items")
                b.sketch_reservoir(name, size=int(sk._size), key_population=pop, state=sk._rng.getstate()[1])
            else:
                raise UnsupportedModelError(f"sketch collector {name!r}: sketch {_cls(sk)} (supported: HyperLogLog, "
                                            "CountMinSketch, BloomFilter, TopK, ReservoirSampler)")
        elif k == A.HS_ENT_LB:
            strat = o._strategy
            backs = [info.backend for info in o._backends.values() if info.is_healthy]
            if len(backs) != len(o._backends):
                raise UnsupportedModelError(f"load balancer {name!r}: unhealthy backends")
            sname = _cls(strat)
            table = None
            if sname == "ConsistentHash":
                gk = getattr(strat, "_get_key", None)
                if gk is not None and getattr(gk, "__func__", None) is not getattr(type(strat), "_default_get_key", object()):
                    raise UnsupportedModelError(f"load balancer {name!r}: custom get_key callbacks")
                pop = key_population or max((int(getattr(getattr(s._event_provider, "_context_fn", None),
                                                         "key_population", 0)) for s in sources or []), default=0)
                if pop <= 0:
                    raise UnsupportedModelError(f"load balancer {name!r}: ConsistentHash needs a finite key population")
                table = consistent_hash_table([bk.name for bk in backs], int(strat._virtual_nodes), pop)
            elif sname != "RoundRobin":
                raise UnsupportedModelError(f"load balancer {name!r}: strategy {sname}")
            pending_lb.append((name, [ids[id(bk)] for bk in backs], table))
            b._add(name, A.HS_ENT_LB)           # placeholder row, fixed below (ids must stay in objs order)
        else:  # pragma: no cover
            raise UnsupportedModelError(name)
    # fill LB rows (backend lists are concatenated in LB order)
    lb_iter = iter(pending_lb)
    for idx, o in enumerate(objs):
        if kind_of(o) != A.HS_ENT_LB:
            continue
        name, backs, table = next(lb_iter)
        off = len(b._backends)
        b._backends += backs
        strat = A.HS_LB_ROUND_ROBIN
        if table is not None:
            if b._key_table.size:
                raise UnsupportedModelError("more than one key-routed load balancer")
            strat = A.HS_LB_KEY_TABLE
            b._key_table = np.asarray(table, np.int32)
        b._rows[idx] = (A.HS_ENT_LB, -1, strat, off, len(backs), 0, -1, 0.0, 0.0)
    for sid, name, tgt, metric in probe_rows:
        pid = b._add(name + ".measure", A.HS_ENT_PROBE, tgt, A.METRICS[metric])
        b.set_target(sid, pid)
    for tgt, t_ns, crash, idx, ev in faults:
        if id(tgt) not in ids:
            raise UnsupportedModelError(f"fault on {getattr(tgt, 'name', tgt)!r}: the entity is not part of the model")
        b.fault(f"fault:{getattr(tgt, 'name', '?')}", target=ids[id(tgt)], time_ns=t_ns, crash=crash, sort_index=idx,
                cancelled=bool(getattr(ev, "_cancelled", False)))
    model = b.build()
    if faults:
        model.fault_events = [ev for *_, ev in faults]
    # a source whose key population is set needs the table length to match (validated by the C-ABI too)
    return model, objs


def refresh_fault_cancellation(model) -> bool:
    """Copy the ``_cancelled`` flags of the model's fault events into its FAULT rows: FaultHandle.cancel() may be
    called between building the Simulation and running it (faults/fault.py:80-87).  Returns whether a row changed."""
    evs = getattr(model, "fault_events", None)
    if not evs:
        return False
    changed = False
    for i, ev in zip(model.ids_of(A.HS_ENT_FAULT), evs):
        v = 1 if getattr(ev, "_cancelled", False) else 0
        if int(model.entities["i2"][i]) != v:
            model.entities["i2"][i] = v
            changed = True
    return changed
