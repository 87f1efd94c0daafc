"""install() on the GPU: an unchanged reference script, stock-seeded, prints the reference's own numbers.
Needs the reference as build() installs it into oracle/_ref; skipped when it is absent."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
import golden_lib as G


@pytest.fixture(scope="module")
def ref():
    if not G.HAVE_REF:
        pytest.skip(G.NO_REF)
    return G.import_reference()


def quickstart(ref, end_s=60.0, rate=8, n_servers=0):
    from happysimulator import Instant, Simulation, Sink, Source
    from happysimulator.components.server.server import Server
    from happysimulator.distributions.exponential import ExponentialLatency
    sink = Sink()
    if n_servers:
        from happysimulator.components.load_balancer.load_balancer import LoadBalancer
        from happysimulator.components.load_balancer.strategies import RoundRobin
        servers = [Server(f"S{i}", service_time=ExponentialLatency(0.1), downstream=sink) for i in range(n_servers)]
        lb = LoadBalancer("LB", backends=servers, strategy=RoundRobin())
        src = Source.poisson(rate=rate, target=lb)
        return Simulation(sources=[src], entities=[*servers, sink, lb], end_time=Instant.from_seconds(end_s)), sink, servers
    server = Server("Server", service_time=ExponentialLatency(0.1), downstream=sink)
    src = Source.poisson(rate=rate, target=server)
    return Simulation(sources=[src], entities=[server, sink], end_time=Instant.from_seconds(end_s)), sink, [server]


@pytest.mark.parametrize("n_servers,rate,end_s", [(0, 8, 60.0), (0, 9.5, 200.0), (4, 32, 20.0)])
def test_unchanged_reference_script_gives_the_reference_numbers(ref, n_servers, rate, end_s):
    import happysim_b200 as hs

    def script():
        random.seed(42); np.random.seed(42)
        sim, sink, servers = quickstart(ref, end_s, rate, n_servers)
        summary = sim.run()
        tail = (random.random(), float(np.random.random()))          # where the global generators were left
        return summary, sink, servers, tail
    want_s, want_sink, want_srv, want_tail = script()                 # the reference's own loop
    hs.install()
    try:
        got_s, got_sink, got_srv, got_tail = script()
        st = hs.install_stats()
    finally:
        hs.uninstall()
    assert st["device_runs"] >= 1
    assert type(got_s) is type(want_s)
    assert got_s.total_events_processed == want_s.total_events_processed and got_s.duration_s == want_s.duration_s
    assert got_sink.events_received == want_sink.events_received
    assert got_sink.latencies_s == want_sink.latencies_s
    assert [t.nanoseconds for t in got_sink.completion_times] == [t.nanoseconds for t in want_sink.completion_times]
    assert got_sink.average_latency() == want_sink.average_latency()
    for a, b in zip(got_srv, want_srv):
        assert a.stats.requests_completed == b.stats.requests_completed and a.stats.total_service_time == b.stats.total_service_time
    assert {k: v.events_handled for k, v in got_s.entities.items()} == {k: v.events_handled for k, v in want_s.entities.items()}
    assert got_tail == want_tail
    if (n_servers, rate, end_s) == (0, 8, 60.0):     # the README quick-start's known answer (SURVEY.md 8(c))
        assert got_s.total_events_processed == 3621 and got_sink.average_latency() == 0.5696996189709543


def test_run_replicas_is_one_device_ensemble(ref):
    import happysim_b200 as hs
    from happysimulator.parallel.runner import ParallelRunner
    hs.install()
    try:
        res = ParallelRunner(max_workers=2).run_replicas(lambda: quickstart(ref, 30.0)[0], n_replicas=32, base_seed=7)
        st = hs.install_stats()
    finally:
        hs.uninstall()
    assert len(res) == 32 and st["device_runs"] >= 1
    ev = [r.summary.total_events_processed for r in res]
    assert len(set(ev)) > 8 and all(1200 < e < 2600 for e in ev)
    assert res[3].summary.entities["Sink"].events_handled > 150


def test_probes_and_trackers_survive_install(ref):
    """A script with a queue-depth Probe and a LatencyTracker sink (instrumentation/probe.py, collectors.py):
    the samples written back onto the script's own Data objects equal the reference loop's."""
    import happysim_b200 as hs
    from happysimulator import Instant, LatencyTracker, Probe, Simulation, Source
    from happysimulator.components.server.server import Server
    from happysimulator.distributions.exponential import ExponentialLatency

    def script():
        random.seed(3); np.random.seed(3)
        sink = LatencyTracker(name="Sink")
        server = Server("Server", service_time=ExponentialLatency(0.1), downstream=sink)
        probe, depth = Probe.on(server, "depth", interval=0.25)
        sim = Simulation(sources=[Source.poisson(rate=9, target=server)], entities=[server, sink], probes=[probe],
                         end_time=Instant.from_seconds(40.0))
        summary = sim.run()
        return summary, sink, depth
    want_s, want_sink, want_depth = script()
    hs.install()
    try:
        got_s, got_sink, got_depth = script()
        st = hs.install_stats()
    finally:
        hs.uninstall()
    assert st["device_runs"] >= 1 and st["fallbacks"] == 0
    assert got_s.total_events_processed == want_s.total_events_processed
    assert got_depth.raw_values() == want_depth.raw_values() and got_depth.times() == want_depth.times()
    assert got_sink.data.raw_values() == want_sink.data.raw_values() and got_sink.count == want_sink.count
