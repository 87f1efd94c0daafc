"""The model families of the stock-generator ensemble fixtures (tests/golden/stockens_*.npz).  Test infrastructure.

Each family is built with the package's own classes, as a user script would build it, so that ``ParallelRunner.run_sweep``
can run it and the fixture's FlatModel is exactly what ``Simulation`` lowers it to.  In stock mode every draw comes from
one of the reference's two process-global streams -- numpy's for every Poisson source, ``random``'s for every
exponential server -- so the families differ in who shares a stream and in which order:

  two_sources     two Poisson sources bootstrap from the numpy stream in order, then draw in tick order
  tandem3         three exponential servers in a row draw from the ``random`` stream in processing order
  mmc3_lifo_cap   M/M/3, LIFO queue of capacity 4 that drops
  rr4_c2          round robin over four servers of concurrency 2
  ramp            a Poisson source with a LinearRampProfile (the profile's Simpson + Brent path) -> one server
  const_arrivals  constant-rate source -> exponential server: the service stream only
  const_service   Poisson source -> constant-service server: the arrival stream only
  counter         M/M/1 into a Counter

Horizons give every replica a few hundred draws of each stream it uses."""
from __future__ import annotations

import happysim_b200 as hs

N_SEEDS = 8                   # consecutive seeds s0 .. s0 + 7 per family


def two_sources():
    sink = hs.Sink()
    srv = hs.Server("Server", service_time=hs.ExponentialLatency(0.06), downstream=sink)
    return [hs.Source.poisson(rate=3.0, target=srv, name="A"), hs.Source.poisson(rate=5.0, target=srv, name="B")], [srv, sink]


def tandem3():
    sink = hs.Sink()
    c = hs.Server("C", service_time=hs.ExponentialLatency(0.08), downstream=sink)
    b = hs.Server("B", concurrency=2, service_time=hs.ExponentialLatency(0.15), downstream=c)
    a = hs.Server("A", service_time=hs.ExponentialLatency(0.05), downstream=b)
    return [hs.Source.poisson(rate=6.0, target=a)], [a, b, c, sink]


def mmc3_lifo_cap():
    sink = hs.Sink()
    srv = hs.Server("Server", concurrency=3, service_time=hs.ExponentialLatency(0.09),
                    queue_policy=hs.LIFOQueue(capacity=4), downstream=sink)
    return [hs.Source.poisson(rate=36.0, target=srv)], [srv, sink]


def rr4_c2():
    sink = hs.Sink()
    sv = [hs.Server(f"S{i}", concurrency=2, service_time=hs.ExponentialLatency(0.2), downstream=sink) for i in range(4)]
    lb = hs.LoadBalancer("LB", backends=sv, strategy=hs.RoundRobin())
    return [hs.Source.poisson(rate=30.0, target=lb)], [*sv, sink, lb]


def ramp():
    sink = hs.Sink()
    srv = hs.Server("Server", service_time=hs.ExponentialLatency(0.06), downstream=sink)
    return [hs.Source.with_profile(hs.LinearRampProfile(30.0, 2.0, 14.0), target=srv)], [srv, sink]


def const_arrivals():
    sink = hs.Sink()
    srv = hs.Server("Server", service_time=hs.ExponentialLatency(0.08), downstream=sink)
    return [hs.Source.constant(rate=10.0, target=srv)], [srv, sink]


def const_service():
    sink = hs.Sink()
    srv = hs.Server("Server", service_time=hs.ConstantLatency(0.09), downstream=sink)
    return [hs.Source.poisson(rate=9.0, target=srv)], [srv, sink]


def counter():
    cnt = hs.Counter("Counter")
    srv = hs.Server("Server", service_time=hs.ExponentialLatency(0.1), downstream=cnt)
    return [hs.Source.poisson(rate=8.0, target=srv)], [srv, cnt]


# name: (build, first seed, horizon in seconds, runs on the lane engine)
FAMILIES = {
    "two_sources": (two_sources, 101, 40.0, False),
    "tandem3": (tandem3, 201, 50.0, False),
    "mmc3_lifo_cap": (mmc3_lifo_cap, 301, 10.0, True),
    "rr4_c2": (rr4_c2, 401, 12.0, False),
    "ramp": (ramp, 501, 40.0, True),
    "const_arrivals": (const_arrivals, 601, 40.0, True),
    "const_service": (const_service, 701, 40.0, True),
    "counter": (counter, 801, 40.0, True),
}


def simulation(name, *, seed=None, rng="stock"):
    """A fresh Simulation of family ``name`` (new objects every call) with its own horizon."""
    build, s0, end_s, _ = FAMILIES[name]
    sources, entities = build()
    return hs.Simulation(end_time=hs.Instant.from_seconds(end_s), sources=sources, entities=entities,
                         seed=s0 if seed is None else seed, rng=rng)
