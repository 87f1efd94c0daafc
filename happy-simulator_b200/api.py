"""Host-side mirror of the reference's modelling API for the accelerated path.

Same names, argument meaning and error behaviour as the reference classes they
stand for (cited per class), so models and tests read like the reference's own;
``Simulation.run()`` lowers the object graph (lowering.py), runs it on the CUDA
engine through the C-ABI (engine.py) and writes the results back onto the entity
objects, which is where the reference's callers read them
(``sink.latencies_s``, ``server.stats``, ``source.generated_count``, ``lb.stats``).

Randomness: the reference draws from Python's and numpy's global MT19937 streams;
here every stochastic consumer owns a Philox stream keyed by ``seed`` (the
``Simulation(seed=)`` argument, default ``happysim_b200.default_seed``) -- the same
streams the Philox plug-ins inject into the unmodified reference in the parity tests.
"""
from __future__ import annotations

from dataclasses import dataclass, field
import math
import time as _time
from typing import Any, Callable

import numpy as np

from . import _abi as A
from . import buckets as _buckets
from . import lowering
from .engine import Engine, make_params
from .results import EntitySummary, QueueStats, SimulationSummary, fault_cancelled, replica_summary, write_back  # noqa: F401

default_seed = 0


def seed(value: int) -> None:
    """Set the default Philox key of subsequent ``Simulation`` objects (cf. random.seed)."""
    global default_seed
    default_seed = int(value)


# ----------------------------------------------------------------------------- time
class Duration:
    """core/temporal.py:24-160 -- nanosecond duration; from_seconds truncates like the reference."""
    __slots__ = ("nanoseconds",)

    def __init__(self, nanoseconds: int):
        self.nanoseconds = nanoseconds

    @classmethod
    def from_seconds(cls, seconds):
        if isinstance(seconds, int):
            return cls(seconds * 1_000_000_000)
        if isinstance(seconds, float):
            return cls(int(seconds * 1_000_000_000))
        raise TypeError("seconds must be int or float")

    def to_seconds(self) -> float:
        return float(self.nanoseconds) / 1_000_000_000

    def __eq__(self, o):
        return isinstance(o, Duration) and self.nanoseconds == o.nanoseconds

    def __lt__(self, o):
        return self.nanoseconds < o.nanoseconds

    def __hash__(self):
        return hash(self.nanoseconds)

    def __repr__(self):
        return f"Duration({self.to_seconds()}s)"


class Instant:
    """core/temporal.py:165-300 -- nanosecond time point."""
    __slots__ = ("nanoseconds",)

    def __init__(self, nanoseconds: int):
        self.nanoseconds = nanoseconds

    @classmethod
    def from_seconds(cls, seconds):
        if isinstance(seconds, int):
            return cls(seconds * 1_000_000_000)
        if isinstance(seconds, float):
            return cls(int(seconds * 1_000_000_000))
        raise TypeError("seconds must be int or float")

    def to_seconds(self) -> float:
        return float(self.nanoseconds) / 1_000_000_000

    def __add__(self, other):
        if isinstance(other, Duration):
            return Instant(self.nanoseconds + other.nanoseconds)
        if isinstance(other, (int, float)):
            return Instant(self.nanoseconds + int(other * 1_000_000_000))
        return NotImplemented

    def __sub__(self, other):
        if isinstance(other, Instant):
            return Duration(self.nanoseconds - other.nanoseconds)
        if isinstance(other, Duration):
            return Instant(self.nanoseconds - other.nanoseconds)
        if isinstance(other, (int, float)):
            return Instant(self.nanoseconds - int(other * 1_000_000_000))
        return NotImplemented

    def __eq__(self, o):
        return isinstance(o, Instant) and self.nanoseconds == o.nanoseconds

    def __lt__(self, o):
        return self.nanoseconds < o.nanoseconds

    def __le__(self, o):
        return self.nanoseconds <= o.nanoseconds

    def __gt__(self, o):
        return self.nanoseconds > o.nanoseconds

    def __ge__(self, o):
        return self.nanoseconds >= o.nanoseconds

    def __hash__(self):
        return hash(self.nanoseconds)

    def __repr__(self):
        return f"Instant({self.to_seconds()}s)"


Instant.Epoch = Instant(0)


# ----------------------------------------------------------------------------- plug-ins
@dataclass(frozen=True)
class ConstantRateProfile:
    """load/profile.py:37-47"""
    rate: float

    def get_rate(self, time) -> float:
        return self.rate


@dataclass(frozen=True)
class LinearRampProfile:
    """load/profile.py:51-74"""
    duration_s: float
    start_rate: float
    end_rate: float

    def get_rate(self, time) -> float:
        t = time.to_seconds()
        if t <= 0:
            return self.start_rate
        if t >= self.duration_s:
            return self.end_rate
        return self.start_rate + (t / self.duration_s) * (self.end_rate - self.start_rate)


@dataclass(frozen=True)
class SpikeProfile:
    """load/profile.py:77-110"""
    baseline_rate: float = 10.0
    spike_rate: float = 150.0
    warmup_s: float = 10.0
    spike_duration_s: float = 15.0

    def get_rate(self, time) -> float:
        t = time.to_seconds()
        if t < self.warmup_s:
            return self.baseline_rate
        if t < self.warmup_s + self.spike_duration_s:
            return self.spike_rate
        return self.baseline_rate


@dataclass(frozen=True)
class StepProfile:
    """A piecewise-constant rate profile (not in the reference's load/profile.py; the reference's examples define
    such profiles themselves, e.g. examples/queuing/m_m_1_queue.py:104-169): ``rates[k]`` applies from
    ``breakpoints[k - 1]`` (inclusive) to ``breakpoints[k]`` (exclusive).  Lowered as HS_PROF_STEP."""
    breakpoints: tuple = ()
    rates: tuple = (1.0,)

    def __post_init__(self):
        if len(self.rates) != len(self.breakpoints) + 1:
            raise ValueError("StepProfile: n breakpoints need n + 1 rates")
        if any(b <= a for a, b in zip(self.breakpoints, self.breakpoints[1:])):
            raise ValueError("StepProfile: breakpoints must ascend")

    def get_rate(self, time) -> float:
        import bisect
        return float(self.rates[bisect.bisect_right(self.breakpoints, time.to_seconds())])

    @classmethod
    def from_profile(cls, profile, end_s: float, scan_step_s: float | None = None) -> "StepProfile":
        """Tabulate any step-function ``Profile`` (exactly, see lowering.step_table_from_profile)."""
        breaks, rates = lowering.step_table_from_profile(profile, scan_end_s=float(end_s), scan_step_s=scan_step_s)
        return cls(tuple(breaks), tuple(rates))


class _ArrivalTimeProvider:
    """load/arrival_time_provider.py:28-47 (constant-rate profiles only on the device)."""

    def __init__(self, profile, start_time: Instant):
        self.profile = profile
        self.current_time = start_time


class ConstantArrivalTimeProvider(_ArrivalTimeProvider):
    """load/providers/constant_arrival.py:11-23"""


class PoissonArrivalTimeProvider(_ArrivalTimeProvider):
    """load/providers/poisson_arrival.py:18-31"""


class _LatencyDistribution:
    """distributions/latency_distribution.py:17-41"""

    def __init__(self, mean_latency):
        self._mean_latency = mean_latency.to_seconds() if isinstance(mean_latency, Duration) else float(mean_latency)


class ConstantLatency(_LatencyDistribution):
    """distributions/constant.py:17-35"""


class ExponentialLatency(_LatencyDistribution):
    """distributions/exponential.py:17-45"""

    def __init__(self, mean_latency):
        super().__init__(mean_latency)
        self._lambda = 1 / self._mean_latency


class FIFOQueue:
    """components/queue_policy.py:75-114"""

    def __init__(self, capacity: float = float("inf")):
        self._capacity = capacity

    @property
    def capacity(self):
        return self._capacity


class LIFOQueue(FIFOQueue):
    """components/queue_policy.py:117-156"""


class PriorityQueue(FIFOQueue):
    """components/queue_policy.py:189-287: pops the request with the smallest (key(request), insertion order).  On the
    device the key is a ``PriorityByKey`` table over the request's routing key; ``_insert_counter`` (successful pushes)
    is published after a run, as the reference's object would hold it."""

    def __init__(self, capacity: float = float("inf"), key: Callable | None = None):
        super().__init__(capacity)
        self._key = key
        self._insert_counter = 0


class PriorityByKey:
    """key for PriorityQueue: the priority of a request is ``values[k]``, k its routing key
    (``context["metadata"]["client_id"]`` of ``UniformKeyContext`` / ``ZipfKeyContext``), the one per-request value
    that exists on the device.  Lower values leave first.  A plain callable, so the same object works as the key of
    the reference's own PriorityQueue."""

    priority_by_routing_key = True

    def __init__(self, values):
        self.values = list(values)

    def __call__(self, event):
        return self.values[event.context["metadata"]["client_id"]]


class FixedConcurrency:
    """components/server/concurrency.py:66-140"""

    def __init__(self, max_concurrent: int):
        if max_concurrent < 1:
            raise ValueError(f"max_concurrent must be >= 1, got {max_concurrent}")
        self._max_concurrent = max_concurrent

    @property
    def limit(self) -> int:
        return self._max_concurrent


class RoundRobin:
    """components/load_balancer/strategies.py:50-72"""


class ConsistentHash:
    """components/load_balancer/strategies.py:336-433 (default key extraction: metadata client_id)."""

    def __init__(self, virtual_nodes: int = 100, get_key: Callable | None = None):
        if virtual_nodes < 1:
            raise ValueError(f"virtual_nodes must be >= 1, got {virtual_nodes}")
        if get_key is not None:
            raise lowering.UnsupportedModelError("custom get_key callbacks cannot run on the device")
        self._virtual_nodes = virtual_nodes
        self._get_key = None


class UniformKeyContext:
    """context_fn for SimpleEventProvider: metadata {"client_id": k}, k ~ Uniform{0..population-1}
    drawn from the Philox routing stream (cf. the reference's
    SimpleEventProvider(context_fn=...) + distributions/uniform.py:57-63)."""

    def __init__(self, population: int):
        if population < 1:
            raise ValueError("population must be >= 1")
        self.key_population = int(population)


class ZipfKeyContext(UniformKeyContext):
    """context_fn for SimpleEventProvider: metadata {"client_id": k}, k ~ ZipfDistribution(range(population), s)
    (distributions/zipf.py:27-123: inverse transform, bisect_left over the cumulative probabilities) drawn from
    the Philox routing stream; rank 0 is the hottest key."""

    def __init__(self, population: int, s: float = 1.0):
        super().__init__(population)
        if s < 0:
            raise ValueError(f"s must be non-negative, got {s}")
        self.zipf_s = float(s)


# ----------------------------------------------------------------------------- entities
class Entity:
    """core/entity.py:31-127"""

    def __init__(self, name: str):
        self.name = name


class SimpleEventProvider:
    """load/source.py:31-86"""

    def __init__(self, target: Entity, event_type: str = "Request", stop_after: Instant | None = None,
                 context_fn=None):
        self._target = target
        self._event_type = event_type
        self._stop_after = stop_after
        self._context_fn = context_fn
        self._generated = 0


class Source(Entity):
    """load/source.py:92-341"""

    def __init__(self, name: str, event_provider, arrival_time_provider):
        super().__init__(name)
        self._event_provider = event_provider
        self._time_provider = arrival_time_provider
        self._generated_count = 0

    @staticmethod
    def _resolve_stop_after(stop_after):
        if stop_after is None or isinstance(stop_after, Instant):
            return stop_after
        return Instant.from_seconds(stop_after)

    @classmethod
    def _make(cls, provider_cls, rate, target, event_type, name, stop_after, event_provider):
        if event_provider is None:
            if target is None:
                raise ValueError("Either 'target' or 'event_provider' must be provided")
            event_provider = SimpleEventProvider(target, event_type, cls._resolve_stop_after(stop_after))
        return cls(name=name, event_provider=event_provider,
                   arrival_time_provider=provider_cls(ConstantRateProfile(rate=rate), start_time=Instant.Epoch))

    @classmethod
    def constant(cls, rate, target=None, event_type="Request", *, name="Source", stop_after=None, event_provider=None):
        return cls._make(ConstantArrivalTimeProvider, rate, target, event_type, name, stop_after, event_provider)

    @classmethod
    def poisson(cls, rate, target=None, event_type="Request", *, name="Source", stop_after=None, event_provider=None):
        return cls._make(PoissonArrivalTimeProvider, rate, target, event_type, name, stop_after, event_provider)

    @classmethod
    def with_profile(cls, profile, target=None, event_type="Request", *, poisson=True, name="Source",
                     stop_after=None, event_provider=None):
        """load/source.py:271-318"""
        if event_provider is None:
            if target is None:
                raise ValueError("Either 'target' or 'event_provider' must be provided")
            event_provider = SimpleEventProvider(target, event_type, cls._resolve_stop_after(stop_after))
        provider_cls = PoissonArrivalTimeProvider if poisson else ConstantArrivalTimeProvider
        return cls(name=name, event_provider=event_provider,
                   arrival_time_provider=provider_cls(profile, start_time=Instant.Epoch))

    @property
    def generated_count(self) -> int:
        return self._generated_count


class _Queue:
    """components/queue.py:76-170 (state holder; the protocol itself runs on the device)."""

    def __init__(self, name, policy):
        self.name = name
        self.policy = policy
        self.stats_dropped = 0
        self.stats_accepted = 0


@dataclass(frozen=True)
class ServerStats:
    """components/server/server.py:34-40"""
    requests_completed: int = 0
    requests_rejected: int = 0
    total_service_time: float = 0.0


class Server(Entity):
    """components/server/server.py:43-300 (QueuedResource + FixedConcurrency + service distribution)."""

    def __init__(self, name: str, concurrency=1, service_time=None, queue_policy=None, queue_capacity=None,
                 downstream: Entity | None = None):
        super().__init__(name)
        if queue_policy is None:
            queue_policy = FIFOQueue(capacity=queue_capacity if queue_capacity is not None else float("inf"))
        self._queue = _Queue(f"{name}.queue", queue_policy)
        self._concurrency_model = FixedConcurrency(concurrency) if isinstance(concurrency, int) else concurrency
        self._service_time = service_time or ConstantLatency(0.01)
        self._downstream = downstream
        self._requests_completed = 0
        self._requests_rejected = 0
        self._total_service_time = 0.0
        self._service_times: list[float] = []

    @property
    def downstream(self):
        return self._downstream

    @downstream.setter
    def downstream(self, target):
        self._downstream = target

    @property
    def concurrency(self) -> int:
        return self._concurrency_model.limit

    @property
    def stats_accepted(self) -> int:
        return self._queue.stats_accepted

    @property
    def stats_dropped(self) -> int:
        return self._queue.stats_dropped

    @property
    def stats(self) -> ServerStats:
        return ServerStats(self._requests_completed, self._requests_rejected, self._total_service_time)

    @property
    def average_service_time(self) -> float:
        return sum(self._service_times) / len(self._service_times) if self._service_times else 0.0


@dataclass
class CachingServerStats:
    """examples/load-balancing/common.py:90-97"""
    requests_processed: int = 0
    cache_hits: int = 0
    cache_misses: int = 0


class CachingServer(Entity):
    """examples/load-balancing/common.py:100-275: a server with a local TTL cache in front of a shared datastore.
    Same constructor; ``datastore`` is accepted and unused (its read latency is ``datastore_read_latency_s``).
    The request's customer id is its routing key (``UniformKeyContext`` / ``ZipfKeyContext`` on the source).
    ``cache_capacity`` must exceed the key population: the reference class raises on its first eviction."""

    def __init__(self, name: str, server_id: int = 0, datastore=None, cache_capacity: int = 100, cache_ttl_s: float = 30.0,
                 cache_read_latency_s: float = 0.0001, datastore_read_latency_s: float = 0.005,
                 processing_latency_s: float = 0.001):
        super().__init__(name)
        if cache_ttl_s <= 0:
            raise ValueError(f"ttl must be > 0, got {cache_ttl_s}")          # eviction_policies.py:174
        self.server_id = server_id
        self._datastore = datastore
        self._cache_capacity = cache_capacity
        self._cache_ttl_s = cache_ttl_s
        self._cache_read_latency_s = cache_read_latency_s
        self._datastore_read_latency_s = datastore_read_latency_s
        self._processing_latency_s = processing_latency_s
        self._queue = _Queue(f"{name}.queue", FIFOQueue())
        self.stats = CachingServerStats()
        self._insert_times: dict[str, float] = {}     # TTLEviction._insert_times after the run: "customer:<id>" -> seconds

    @property
    def stats_accepted(self) -> int:
        return self._queue.stats_accepted

    @property
    def stats_dropped(self) -> int:
        return self._queue.stats_dropped

    @property
    def hit_rate(self) -> float:
        total = self.stats.cache_hits + self.stats.cache_misses
        return self.stats.cache_hits / total if total else 0.0

    @property
    def miss_rate(self) -> float:
        total = self.stats.cache_hits + self.stats.cache_misses
        return self.stats.cache_misses / total if total else 0.0

    @property
    def cache_size(self) -> int:
        return len(self._insert_times)

    @property
    def requests_processed(self) -> int:
        return self.stats.requests_processed


class Sink(Entity):
    """components/common.py:18-76"""

    def __init__(self, name: str = "Sink"):
        super().__init__(name)
        self.events_received = 0
        self.completion_times: list[Instant] = []
        self.latencies_s: list[float] = []
        self._latency_sum = 0.0

    def average_latency(self) -> float:
        if not self.events_received:
            return 0.0
        # the device accumulates sum(latencies_s) exactly as CPython's float sum() does
        return self._latency_sum / self.events_received

    def latency_stats(self) -> dict:
        n = len(self.latencies_s)
        if n == 0:
            return {"count": 0, "avg": 0.0, "min": 0.0, "max": 0.0, "p50": 0.0, "p99": 0.0}
        v = sorted(self.latencies_s)

        def pct(p):
            pos = p * (n - 1)
            lo = int(pos)
            hi = min(lo + 1, n - 1)
            frac = pos - lo
            return v[lo] * (1.0 - frac) + v[hi] * frac
        return {"count": n, "avg": sum(v) / n, "min": v[0], "max": v[-1], "p50": pct(0.50), "p99": pct(0.99)}


class Counter(Entity):
    """components/common.py:79-95"""

    def __init__(self, name: str = "Counter"):
        super().__init__(name)
        self.total = 0
        self.by_type: dict[str, int] = {}


@dataclass
class BackendInfo:
    """components/load_balancer/load_balancer.py (BackendInfo)"""
    backend: Entity
    weight: int = 1
    is_healthy: bool = True
    total_requests: int = 0


@dataclass(frozen=True)
class LoadBalancerStats:
    requests_received: int = 0
    requests_forwarded: int = 0
    requests_failed: int = 0
    no_backend_available: int = 0
    backends_marked_unhealthy: int = 0
    backends_marked_healthy: int = 0


class LoadBalancer(Entity):
    """components/load_balancer/load_balancer.py:60-473"""

    def __init__(self, name: str, backends=None, strategy=None, on_no_backend: str = "reject"):
        super().__init__(name)
        if on_no_backend not in ("reject", "queue"):
            raise ValueError(f"on_no_backend must be 'reject' or 'queue', got {on_no_backend}")
        self._strategy = strategy or RoundRobin()
        self._backends: dict[str, BackendInfo] = {}
        self._in_flight: dict = {}
        self._requests_received = 0
        self._requests_forwarded = 0
        for b in backends or []:
            self.add_backend(b)

    def add_backend(self, backend: Entity, weight: int = 1) -> None:
        if weight < 1:
            raise ValueError(f"weight must be >= 1, got {weight}")
        self._backends[backend.name] = BackendInfo(backend=backend, weight=weight)

    @property
    def stats(self) -> LoadBalancerStats:
        return LoadBalancerStats(requests_received=self._requests_received,
                                 requests_forwarded=self._requests_forwarded)


# ----------------------------------------------------------------------------- faults/ (node faults)
@dataclass(frozen=True)
class FaultStats:
    """faults/fault.py:95-108"""
    faults_scheduled: int
    faults_activated: int
    faults_deactivated: int
    faults_cancelled: int


class _FaultEvent:
    """What the device needs of a fault's Event.once (core/event.py:372-401): its time, its sort index and the
    ``_cancelled`` flag FaultHandle.cancel() sets."""

    def __init__(self, time: Instant, sort_index: int):
        self.time, self._sort_index, self._cancelled = time, sort_index, False

    def cancel(self) -> None:
        self._cancelled = True


class FaultHandle:
    """faults/fault.py:55-87: cancel() before run() cancels the events the schedule has generated so far (a
    Simulation generates them when it is built)."""

    def __init__(self, fault):
        self.fault = fault
        self._events: list = []
        self._cancelled = False

    @property
    def cancelled(self) -> bool:
        return self._cancelled

    def cancel(self) -> None:
        if self._cancelled:
            return
        self._cancelled = True
        for ev in self._events:
            ev.cancel()


@dataclass(frozen=True)
class CrashNode:
    """faults/node_faults.py:16-78: crash ``entity_name`` at ``at`` s, restart at ``restart_at`` s (None: never)."""
    entity_name: str
    at: float
    restart_at: float | None = None


@dataclass(frozen=True)
class PauseNode:
    """faults/node_faults.py:81-128: pause ``entity_name`` from ``start`` s to ``end`` s."""
    entity_name: str
    start: float
    end: float


def _start_schedule(schedule, sources, entities, probes) -> None:
    """Generate the events of ``schedule`` (the mirror's or the reference's FaultSchedule) onto its handles, as
    FaultSchedule.start does when a Simulation is built: names resolve (KeyError otherwise), faults other than
    CrashNode / PauseNode raise UnsupportedModelError, and the sort indices follow the sources' and probes' first
    ticks.  A FaultHandle.cancel() from then on marks these events."""
    lowering.fault_events(schedule, sources, entities, probes)      # names and fault classes, before anything changes
    for h in schedule._handles:
        h._events = []
    k = len(list(sources or [])) + len(list(probes or []))
    for fault, h in zip(schedule._faults, schedule._handles):
        times = [fault.at] + ([] if fault.restart_at is None else [fault.restart_at]) \
            if type(fault).__name__ == "CrashNode" else [fault.start, fault.end]
        for t in times:
            h._events.append(_FaultEvent(Instant.from_seconds(t), k))
            k += 1


class FaultSchedule:
    """faults/schedule.py:29-135: ``add()`` node faults; the Simulation generates their events when it is built and
    runs them on the device.  Only CrashNode and PauseNode run there."""

    def __init__(self, name: str = "FaultSchedule"):
        self.name = name
        self._faults: list = []
        self._handles: list[FaultHandle] = []
        self._scheduled = 0

    def add(self, fault) -> FaultHandle:
        h = FaultHandle(fault)
        self._faults.append(fault)
        self._handles.append(h)
        self._scheduled += 1
        return h

    def start(self, sources, entities, probes) -> None:
        """FaultSchedule.start (schedule.py:64-96): every fault's events, with sort indices from the bootstrap
        counter that the sources' and probes' first ticks started."""
        _start_schedule(self, sources, entities, probes)

    @property
    def stats(self) -> FaultStats:
        """The reference never counts activations or deactivations (they stay 0)."""
        return FaultStats(faults_scheduled=self._scheduled, faults_activated=0, faults_deactivated=0,
                          faults_cancelled=sum(1 for h in self._handles if h.cancelled))


def stock_streams(seed: int, n_replicas: int, n_draws: int, seed_stride: int = 1):
    """The reference's two process-global MT19937 streams as unit-rate exponential variates:
    row r is what ``random.seed(seed + r*seed_stride); numpy.random.seed(seed + r*seed_stride)`` yields.
    arrival: -math.log(1.0 - numpy.random.random())   (load/providers/poisson_arrival.py:31)
    service: -math.log(1.0 - random.random())         (random.expovariate, distributions/exponential.py:43)
    math.log is the host libm the reference itself calls."""
    import random as _random
    arr = np.empty((n_replicas, n_draws), np.float64)
    svc = np.empty((n_replicas, n_draws), np.float64)
    for r in range(n_replicas):
        s = seed + r * seed_stride
        u = np.random.RandomState(s).random_sample(n_draws)
        arr[r] = [-math.log(1.0 - x) for x in u]
        rnd = _random.Random(s)
        svc[r] = [-math.log(1.0 - rnd.random()) for _ in range(n_draws)]
    return arr, svc


_engines: dict[int, Engine] = {}


def _engine(device: int) -> Engine:
    if device not in _engines:
        _engines[device] = Engine(device)
    return _engines[device]


class Simulation:
    """core/simulation.py:38-591 -- same constructor, ``run() -> SimulationSummary``.

    Extra keyword arguments (not in the reference): ``seed`` (Philox key), ``replica`` (Philox
    replica word), ``device``, ``queue_ring`` (first size of the device queue rings; they grow on overflow)."""

    def __init__(self, start_time: Instant | None = None, end_time: Instant | None = None, sources=None,
                 entities=None, probes=None, trace_recorder=None, fault_schedule=None, duration: float | None = None,
                 *, seed: int | None = None, replica: int = 0, device: int = 0, rng: str = "philox",
                 queue_ring: int | None = None, _lowered: tuple | None = None):
        if duration is not None and end_time is not None:
            raise ValueError("Cannot specify both 'duration' and 'end_time'")
        if start_time is not None and start_time.nanoseconds != 0:
            raise lowering.UnsupportedModelError("start_time must be Instant.Epoch on the device engine")
        if trace_recorder:
            raise lowering.UnsupportedModelError("trace_recorder= is outside the accelerated path (SURVEY.md section 8)")
        self._start_time = Instant.Epoch
        if duration is not None:
            self._end_time = self._start_time + duration
        elif end_time is not None:
            self._end_time = end_time
        else:
            raise lowering.UnsupportedModelError("the device engine needs an explicit end_time or duration "
                                                 "(auto-termination is the reference's slow loop)")
        self._sources = list(sources or [])
        self._entities = list(entities or [])
        self._probes = list(probes or [])
        self._seed = default_seed if seed is None else int(seed)
        self._replica = int(replica)
        self._device = device
        if rng not in ("philox", "stock"):
            raise ValueError("rng must be 'philox' or 'stock'")
        self._rng = rng
        self._queue_ring = int(queue_ring) if queue_ring else 0
        self.last_run_info: dict = {}
        self._summary: SimulationSummary | None = None
        self._fault_schedule = fault_schedule
        if _lowered is None:
            if fault_schedule is not None:      # Simulation.__init__ bootstraps the schedule (simulation.py:162-169)
                _start_schedule(fault_schedule, self._sources, self._entities, self._probes)
            _lowered = (*lowering.lower(self._sources, self._entities, probes=self._probes,
                                        horizon_s=self._end_time.to_seconds(), fault_schedule=fault_schedule), Instant)
        self.model, self.objects, self._instant_cls = _lowered

    @classmethod
    def _from_lowered(cls, model, objects, *, sources, entities, end_ns: int, seed: int | None = None, replica: int = 0,
                      device: int = 0, instant_cls=Instant) -> "Simulation":
        """A Simulation around a model lowered elsewhere, from a reference Simulation's object graph
        (``run_lowered``, ``install()``); its results are published with ``instant_cls`` time points."""
        return cls(end_time=Instant(int(end_ns)), sources=sources, entities=entities, seed=seed, replica=replica,
                   device=device, _lowered=(model, objects, instant_cls))

    @property
    def summary(self):
        return self._summary

    # -- single run -------------------------------------------------------------
    def _caps(self, n_hint: int | None = None):
        dur = self._end_time.to_seconds()
        rate = lowering.source_rate_bound(self.model)
        req = int(rate * dur * 1.3 + 6 * math.sqrt(rate * dur + 1) + 64)
        n_srv = len(self.model.ids_of(A.HS_ENT_SERVER))
        chain = 1 if (n_srv <= 1 or self.model.ids_of(A.HS_ENT_LB)) else n_srv     # tandem: one start per stage
        return dict(record_cap=0, sample_cap=req, service_cap=req * chain)

    def _events_per_request(self) -> int:
        """Upper bound of processed events per generated request: ~7 per server stage a request can pass
        (ENQUEUE, NOTIFY, POLL, DELIVER, WORKER, CONTINUATION, completion POLL) plus tick, routing and sink."""
        n_srv = len(self.model.ids_of(A.HS_ENT_SERVER))
        stages = 1 if (n_srv <= 1 or self.model.ids_of(A.HS_ENT_LB)) else n_srv
        return 8 * stages + 8 + 2 * len(self.model.ids_of(A.HS_ENT_PROBE))

    def _queue_ring_hint(self) -> int:
        """First device ring size: the backlog an overloaded model would build over the run, bounded."""
        if self._queue_ring:
            return int(self._queue_ring)
        dur = self._end_time.to_seconds()
        ents = self.model.entities
        cap = 0.0
        for i in self.model.ids_of(A.HS_ENT_SERVER):
            mean = float(ents["d0"][i])
            cap += (max(1, int(ents["i0"][i])) / mean) if mean > 0 else float("inf")
        backlog = max(0.0, (lowering.source_rate_bound(self.model) - cap) * dur)
        ring = 256
        while ring < min(2.5 * backlog + 64, 1 << 22):
            ring *= 2
        return ring

    def run(self) -> SimulationSummary:
        return _run_many([self], seed=self._seed, seed_stride=0, rid_base=self._replica, rid_stride=0)[0]

    # -- ensembles ----------------------------------------------------------------
    def run_ensemble(self, n_replicas: int, *, seed: int | None = None, seed_stride: int = 0, rid_base: int = 0,
                     rid_stride: int = 1, replica_index_base: int = 0, replicas_per_cell: int = 1,
                     window_end_s: float | None = None, resume: bool = False, host: dict | None = None,
                     upload: bool = True, totals: bool = True, on_overflow: str = "grow", buckets=None,
                     bucket_percentiles: bool = False, bucket_sample_cap: int = 64, **caps):
        """N independent replicas of this model on the device; returns the raw per-replica arrays
        (summaries, entity_stats, optional recorder rings) and the engine's totals.

        ``window_end_s`` / ``resume`` cut one continuing run into windows exactly like the reference's
        ``Simulation._run_window`` (core/simulation.py:527-541): state stays resident in HBM between calls.
        ``host`` = caller-owned (pinned) buffers from ``Engine.alloc_host_outputs`` to read into.

        Every replica's ``status`` is checked.  A device queue ring that overflowed (the reference's queues are
        unbounded) is handled per ``on_overflow``: "grow" re-runs the ensemble with doubled rings (fresh,
        unwindowed runs only), "raise" raises, "ignore" returns the flagged statuses to the caller.

        ``buckets=(width_s, n)`` reduces every replica's Sink / LatencyTracker / ThroughputTracker / Probe samples into
        ``Data.bucket(width_s)`` on the device (n buckets per row; n * width_s must exceed the end time) and adds
        ``out["buckets"]`` (BUCKET_DTYPE [replica, row, n + 1]; slot n holds the samples of the event processed past the
        end time, whose index is ``out["bucket_past_end"][replica, row]``), ``out["bucket_totals"]`` (BUCKET_TOTAL_DTYPE
        [cell, row, n + 1], cells as ``replicas_per_cell`` and the model's sweep cells define them, one for a plain
        ensemble), ``out["bucket_rows"]`` (entity ids) and ``out["bucket_objects"]`` (the object of each row).
        ``buckets.bucketed_data(out, obj, replica)`` gives one replica's ``BucketedData``.  A bucketed run has no
        recorder rings; every window of a windowed run passes the same ``buckets``, and only the window that reaches the
        end time reads them back (the records are gigabytes at full size; ``Engine.read_buckets`` reads them after any
        window).

        ``bucket_percentiles=True`` (with ``buckets``) adds every bucket's p50 and p99, bit for bit those of
        ``Data.bucket(width_s)``: ``out["bucket_percentiles"]`` (float64 [replica, row, n + 1, 2]) and
        ``out["bucket_percentile_totals"]`` (BUCKET_PCT_TOTAL_DTYPE [cell, row, n + 1]).  The device holds the values of
        each row's current bucket, at most ``bucket_sample_cap`` of them; a bucket with more samples is handled per
        ``on_overflow``: "grow" re-runs the ensemble once with the next power of two at or above the largest bucket
        count (fresh, unwindowed runs only), "raise" and a windowed or resumed run raise ``EnsembleStatusError`` naming
        the capacity to pass, "ignore" returns NaN for those buckets and the HS_ST_BUCKET_OVERFLOW status bit."""
        spec = _buckets.check_spec(buckets, self._end_time.nanoseconds) if buckets is not None else None
        cap = _buckets.check_sample_cap(bucket_sample_cap, spec) if bucket_percentiles else 0
        eng = _engine(self._device)
        if lowering.refresh_fault_cancellation(self.model) and not upload and not resume:
            upload = True                   # a FaultHandle was cancelled since the last upload
        if upload:
            eng.upload(self.model)
        if not resume:
            eng.set_trace(None, None)            # never inherit a stock-generator trace from an earlier run()
        end_ns = self._end_time.nanoseconds
        we = -1
        if window_end_s is not None:
            w = int(round(float(window_end_s) * 1e9))
            we = w if w < end_ns else -1
        ring = int(caps.pop("queue_ring", 0) or 0)
        eng.set_buckets(*(spec or (0.0, 0)))
        eng.set_bucket_percentiles(cap)
        try:
            run = (eng, n_replicas, seed, seed_stride, rid_base, rid_stride, replica_index_base, replicas_per_cell, end_ns,
                   we, resume)
            out, st, ring = self._run_windows(*run, ring, host, on_overflow, caps)
            if cap and on_overflow != "ignore" and int(np.bitwise_or.reduce(st)) & A.HS_ST_BUCKET_OVERFLOW:
                need = _buckets.sample_cap_needed(eng.read_buckets(spec[1])[0])
                if on_overflow == "grow" and not resume and we < 0:
                    cap = need
                    eng.set_bucket_percentiles(cap)
                    out, st, ring = self._run_windows(*run, ring, host, on_overflow, caps)
                if int(np.bitwise_or.reduce(st)) & A.HS_ST_BUCKET_OVERFLOW:
                    n_over = int((st & A.HS_ST_BUCKET_OVERFLOW != 0).sum())
                    raise EnsembleStatusError(f"{n_over} of {n_replicas} replicas had a time bucket with more samples than "
                                              f"bucket_sample_cap={cap}; pass bucket_sample_cap={need}"
                                              + (" (or more: later windows may need it)" if we >= 0 else ""), st.copy())
            if spec and we < 0:
                out.update(_buckets.read_outputs(eng, spec, cap, self.model, self.objects, max(1, int(self.model.n_cells))))
        finally:
            eng.set_bucket_percentiles(0)       # the engine is shared: other runs get no buckets unless they ask
            eng.set_buckets(0.0, 0)
        out["status"] = st
        out["queue_ring"] = ring
        if totals:
            out["totals"] = eng.read_totals()
        out["device_ms"] = eng.last_run_ms()
        return out

    def _run_windows(self, eng, n_replicas, seed, seed_stride, rid_base, rid_stride, replica_index_base, replicas_per_cell,
                     end_ns, we, resume, ring, host, on_overflow, caps):
        bad = A.HS_ST_QUEUE_OVERFLOW | A.HS_ST_FEL_OVERFLOW | A.HS_ST_SKETCH_OVERFLOW
        for _ in range(12):
            eng.run(make_params(seed=self._seed if seed is None else seed, seed_stride=seed_stride, rid_base=rid_base,
                                rid_stride=rid_stride, end_ns=end_ns, n_replicas=n_replicas,
                                replica_index_base=replica_index_base, replicas_per_cell=replicas_per_cell,
                                window_end_ns=we, resume=int(bool(resume)), queue_ring=ring, **caps))
            out = eng.read_outputs(host)
            st = out["summaries"]["status"]
            flagged = int((st & bad != 0).sum())
            if not flagged or on_overflow == "ignore":
                break
            only_queue = not (int(np.bitwise_or.reduce(st)) & (A.HS_ST_FEL_OVERFLOW | A.HS_ST_SKETCH_OVERFLOW))
            if on_overflow == "grow" and only_queue and not resume and we < 0 and ring < (1 << 22):
                ring = max(512, 2 * (ring or 256))
                continue
            raise EnsembleStatusError(f"{flagged} of {n_replicas} replicas stopped early (status bits "
                                      f"{int(np.bitwise_or.reduce(st))}: 1 queue ring full, 2 event list full, 32 sketch "
                                      f"full); pass a larger queue_ring=", st.copy())
        if "max_events" in caps and int((st & A.HS_ST_EVENT_LIMIT != 0).sum()) and on_overflow != "ignore":
            raise EnsembleStatusError("max_events reached before end_time", st.copy())
        return out, st, ring


class EnsembleStatusError(RuntimeError):
    """Replicas of an ensemble stopped early; ``.status`` holds every replica's status word."""

    def __init__(self, msg, status):
        super().__init__(msg)
        self.status = status


def _same_topology(a, b) -> bool:
    """Two lowered models that differ at most in the per-cell columns: d0 (rates, mean service times) of any
    row and i0 (concurrency) of SERVER rows.  Such models run as cells of ONE launch (hs_model_desc.cell_d0/i0)."""
    ea, eb = a.entities, b.entities
    if ea.shape != eb.shape or a.n_cells or b.n_cells:
        return False
    for f in ea.dtype.names:
        if f == "d0":
            continue
        if f == "i0":
            srv = ea["kind"] == A.HS_ENT_SERVER
            if not np.array_equal(ea["i0"][~srv], eb["i0"][~srv]):
                return False
            continue
        if not np.array_equal(ea[f], eb[f]):
            return False
    for f in ("backends", "key_table", "profiles", "profile_table", "sketch_tables", "key_cdf"):
        x, y = np.asarray(getattr(a, f)), np.asarray(getattr(b, f))
        if x.shape != y.shape or x.tobytes() != y.tobytes():
            return False
    return True


def _run_many(sims, *, seed: int, seed_stride: int, rid_base: int, rid_stride: int, trace_fn=None):
    """Run ``sims`` -- Simulations of one topology (``_same_topology``), same end time and device -- as the
    replicas of ONE device launch, replica k = sims[k] with Philox key ``seed + k * seed_stride`` and replica word
    ``rid_base + k * rid_stride``; results are written back onto each Simulation's own objects.  A single
    Simulation is the n = 1 case (``Simulation.run``).  Ring capacities that turn out too small (recorder
    streams, device queues, the event limit) are doubled and the launch repeated; ``last_run_info`` records how
    many launches that took and their wall time."""
    t0 = _time.monotonic()
    lead = sims[0]
    n = len(sims)
    eng = _engine(lead._device)
    for sm in sims:                     # FaultHandle.cancel() may have been called since the Simulation was built
        lowering.refresh_fault_cancellation(sm.model)
    model = lead.model
    if n > 1:
        import copy
        model = copy.copy(lead.model)
        model.cell_d0 = np.stack([np.asarray(sm.model.entities["d0"], np.float64) for sm in sims])
        model.cell_i0 = np.stack([np.asarray(sm.model.entities["i0"], np.int32) for sm in sims])
    eng.upload(model)
    caps = {k: max(sm._caps()[k] for sm in sims) for k in ("record_cap", "sample_cap", "service_cap")}
    stock = getattr(lead, "_rng", "philox") == "stock" or trace_fn is not None
    if trace_fn is None:           # the reference's two MT19937 streams for Simulation(seed=, rng="stock")
        trace_fn = lambda n_draws: stock_streams(seed, n, n_draws, seed_stride)      # noqa: E731
    eng.set_trace(None, None)
    if stock:
        eng.set_trace(*trace_fn(caps["sample_cap"] * 2 + 64))
    m = lead.model
    # per-server service-time lists / per-collector samples are demultiplexed with the event records
    n_streams = len(m.ids_of(A.HS_ENT_SINK)) + len(m.ids_of(A.HS_ENT_PROBE))
    need_events = len(m.ids_of(A.HS_ENT_SERVER)) > 1 or n_streams > 1
    if m.ids_of(A.HS_ENT_PROBE):        # probe samples share the sample stream
        dur = lead._end_time.to_seconds()
        caps["sample_cap"] += max(sum(int(dur * float(sm.model.profiles[int(sm.model.entities["i3"][i]) - 1]["p"][0])) + 8
                                      for i in sm.model.ids_of(A.HS_ENT_SOURCE) if int(sm.model.entities["i3"][i]) > 0)
                                  for sm in sims)
    ring = max(sm._queue_ring_hint() for sm in sims)
    per_req = max(sm._events_per_request() for sm in sims)
    max_events = per_req * caps["sample_cap"] + 1_000_000
    launches, prev_final = 0, None
    for _ in range(24):
        kw = dict(caps)
        if need_events:
            kw["record_cap"] = kw["service_cap"] * 12
        eng.run(make_params(seed=seed, seed_stride=seed_stride, rid_base=rid_base, rid_stride=rid_stride,
                            end_ns=lead._end_time.nanoseconds, n_replicas=n, replicas_per_cell=1, flags=0,
                            max_events=max_events, queue_ring=ring, **kw))
        launches += 1
        out = eng.read_outputs()
        summ = out["summaries"]
        status = int(np.bitwise_or.reduce(summ["status"]))
        if status & A.HS_ST_TRACE_EXHAUSTED:
            caps = {k: 2 * v for k, v in caps.items()}
            max_events = per_req * caps["sample_cap"] + 1_000_000
            eng.set_trace(*trace_fn(caps["sample_cap"] * 2 + 64))
            continue
        if status & A.HS_ST_QUEUE_OVERFLOW and not (status & A.HS_ST_FEL_OVERFLOW):
            if ring >= (1 << 24):
                raise RuntimeError(f"device queue ring overflow at {ring} entries per server; the queue of this model "
                                   f"grows without bound -- pass Simulation(queue_ring=...) if that is intended")
            ring *= 4            # the reference's queues are unbounded: grow the device rings and run again
            continue
        if status & (A.HS_ST_FEL_OVERFLOW | A.HS_ST_SKETCH_OVERFLOW):
            raise RuntimeError(f"device structure overflow (status {status})")
        if status & A.HS_ST_EVENT_LIMIT:
            final = int(summ["final_time_ns"][summ["status"] & A.HS_ST_EVENT_LIMIT != 0].min())
            if prev_final is not None and final <= prev_final:
                raise RuntimeError("event limit reached: the model's clock does not advance (a source faster than "
                                   "one event per nanosecond never terminates in the reference either)")
            prev_final = final
            max_events *= 4      # a valid model denser in events than estimated: raise the safety valve
            continue
        if (int(summ["n_sink_samples"].max()) <= kw["sample_cap"] and int(summ["n_service_samples"].max()) <= kw["service_cap"]
                and (not need_events or int(summ["events_processed"].max()) <= kw["record_cap"])):
            break
        caps = dict(record_cap=0, sample_cap=2 * int(summ["n_sink_samples"].max()) + 64,
                    service_cap=2 * int(summ["n_service_samples"].max()) + 64)
        max_events = max(max_events, per_req * caps["sample_cap"] + 1_000_000)
    else:
        raise RuntimeError("could not size the device buffers for this model")
    if stock:
        eng.set_trace(None, None)            # the trace must not leak into a later ensemble on this engine
    wall = _time.monotonic() - t0
    res = []
    for k, sm in enumerate(sims):
        write_back(sm.model, sm.objects, out, k, sm._instant_cls)
        sm.last_run_info = {"launches": launches, "wall_s": wall, "queue_ring": ring, "batched_with": n,
                            "device_ms_last_launch": eng.last_run_ms(), "status": int(summ[k]["status"])}
        sm._summary = replica_summary(summ[k], wall, sm._entities,
                                      events_cancelled=fault_cancelled(sm.model, out["entity_stats"][k]))
        res.append(sm._summary)
    return res


def _group_by_topology(sims):
    """Indices of ``sims`` grouped so that each group can run as one launch."""
    groups: list[list[int]] = []
    for i, sm in enumerate(sims):
        for g in groups:
            h = sims[g[0]]
            if (h._device == sm._device and h._end_time.nanoseconds == sm._end_time.nanoseconds
                    and getattr(h, "_rng", "philox") == getattr(sm, "_rng", "philox") and _same_topology(h.model, sm.model)):
                g.append(i)
                break
        else:
            groups.append([i])
    return groups


def run_lowered(ref_sim, model=None, objects=None, *, seed: int | None = None, replica: int = 0, device: int = 0,
                trace_fn=None):
    """Run a REFERENCE ``happysimulator.Simulation`` object on the device and write the results back
    onto its own entity objects (the hook shown in INTEGRATION.md section 3).  ``ref_sim`` only needs the
    reference's attributes ``_sources``, ``_entities``, ``_start_time``, ``_end_time``."""
    if model is None:
        model, objects = lowering.lower(ref_sim._sources, ref_sim._entities, probes=getattr(ref_sim, "_probes", None) or None,
                                        horizon_s=float(int(ref_sim._end_time.nanoseconds)) / 1e9,
                                        fault_schedule=getattr(ref_sim, "_fault_schedule", None))
    sim = Simulation._from_lowered(model, objects, sources=ref_sim._sources, entities=ref_sim._entities,
                                   end_ns=ref_sim._end_time.nanoseconds, seed=seed, replica=replica, device=device,
                                   instant_cls=type(ref_sim._start_time))
    return _run_many([sim], seed=sim._seed, seed_stride=0, rid_base=sim._replica, rid_stride=0, trace_fn=trace_fn)[0]


# ----------------------------------------------------------------------------- parallel/runner.py
@dataclass
class RunConfig:
    """parallel/runner.py:42-54"""
    name: str
    build_fn: Callable
    seed: int | None = None


@dataclass
class ParallelResult:
    """parallel/runner.py:57-70 (+ ``status``: the replica's device status word, 0 = ran to end_time)"""
    name: str
    summary: SimulationSummary
    artifacts: dict[str, Any] = field(default_factory=dict)
    status: int = 0


class _ReplicaResults:
    """List-like view of an ensemble's ``ParallelResult``s.  Results are materialised on access (the
    write-back of a replica onto the model's Python objects is O(samples)); ``len``, indexing, slicing and
    iteration behave like the reference's list."""

    def __init__(self, sim, out, wall: float):
        self._sim, self.raw, self._wall = sim, out, wall

    def __len__(self):
        return len(self.raw["summaries"])

    def _one(self, i: int) -> ParallelResult:
        sim, s = self._sim, self.raw["summaries"][i]
        write_back(sim.model, sim.objects, self.raw, i, sim._instant_cls)
        return ParallelResult(name=f"replica_{i}", status=int(s["status"]),
                              summary=replica_summary(s, self._wall, sim._entities,
                                                      events_cancelled=fault_cancelled(sim.model, self.raw["entity_stats"][i])))

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self._one(k) for k in range(*i.indices(len(self)))]
        n = len(self)
        if i < 0:
            i += n
        if not 0 <= i < n:
            raise IndexError(i)
        return self._one(i)

    def __iter__(self):
        return (self._one(i) for i in range(len(self)))

    @property
    def total_events_processed(self) -> int:
        return int(self.raw["summaries"]["events_processed"].sum())


class ParallelRunner:
    """parallel/runner.py:82-142 -- replicas run as one device ensemble instead of a process pool.

    Replica i uses Philox key ``base_seed + i`` (the reference seeds ``random`` with base_seed + i),
    so ``run_replicas(build, n, s)[i]`` equals ``Simulation(seed=s + i).run()``.  A sweep runs as one
    launch per topology: configurations whose lowered models differ only in rates, mean service times and
    server concurrency are the cells of one launch (hs_model_desc.cell_d0 / cell_i0)."""

    def __init__(self, max_workers: int | None = None, device: int = 0):
        self._max_workers = max_workers
        self._device = device

    def run_replicas(self, build_fn: Callable, n_replicas: int, base_seed: int = 42, **caps):
        """Returns a list-like of ParallelResult (materialised on access).  Device queue rings that overflow
        are grown and the ensemble re-run (``Simulation.run_ensemble``); every result carries ``status``.
        ``buckets=(width_s, n)``, ``bucket_percentiles`` and ``bucket_sample_cap`` go to ``run_ensemble``: the time
        buckets are in the returned list's ``.raw``."""
        sim = build_fn()
        t0 = _time.monotonic()
        out = sim.run_ensemble(n_replicas, seed=base_seed, seed_stride=1, rid_base=sim._replica, rid_stride=0,
                               queue_ring=sim._queue_ring_hint(), **caps)
        return _ReplicaResults(sim, out, _time.monotonic() - t0)

    def run_sweep(self, configs: list[RunConfig]) -> list[ParallelResult]:
        """Configurations of one topology run as the cells of one launch.  A ``build_fn`` may also return a
        ParallelSimulation: linked ones of one linked topology run as the cells of one linked ensemble
        (``parallel._run_linked_sweep``), and each result's ``summary`` is that configuration's
        ParallelSimulationSummary.  Results keep the order of ``configs``."""
        from .parallel import ParallelSimulation, _run_linked_sweep
        if not configs:
            return []
        built = []
        for cfg in configs:
            sim = cfg.build_fn()
            if cfg.seed is not None:
                sim._seed = int(cfg.seed)
            built.append(sim)
        res: list = [None] * len(built)
        par = [i for i, sm in enumerate(built) if isinstance(sm, ParallelSimulation)]
        if par:
            for i, (summ, status) in zip(par, _run_linked_sweep([built[i] for i in par])):
                res[i] = ParallelResult(name=configs[i].name, summary=summ, status=status)
        idx = [i for i, sm in enumerate(built) if not isinstance(sm, ParallelSimulation)]
        sims = [built[i] for i in idx]
        for sm in sims:                 # cancellations are part of the topology: read them before grouping
            lowering.refresh_fault_cancellation(sm.model)
        for g in _group_by_topology(sims):
            seeds = [sims[i]._seed for i in g]
            rids = [sims[i]._replica for i in g]
            ds = {b - a for a, b in zip(seeds, seeds[1:])}
            dr = {b - a for a, b in zip(rids, rids[1:])}
            if len(g) > 1 and len(ds) <= 1 and len(dr) <= 1 and min(ds | {0}) >= 0 and min(dr | {0}) >= 0:
                sums = _run_many([sims[i] for i in g], seed=seeds[0], seed_stride=(ds.pop() if ds else 0),
                                 rid_base=rids[0], rid_stride=(dr.pop() if dr else 0))
            else:            # seeds that are not an arithmetic progression: one launch each
                sums = [sims[i].run() for i in g]
            for i, sm in zip(g, sums):
                res[idx[i]] = ParallelResult(name=configs[idx[i]].name, summary=sm, status=sims[i].last_run_info.get("status", 0))
        return res
