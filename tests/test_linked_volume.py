"""ParallelSimulation with PartitionLinks at volumes that fill the device's recorder rings (CPU: LinkedRun is replaced by
oracle_lib.OracleLinkedRun, whose rings wrap exactly like the device's).  The whole host path -- lowering, ring sizing,
the retry loop, the summary and the write-back onto the script's objects -- is compared with the truth: one more oracle
run of the same LinkedModel with rings large enough that nothing wraps.

The cases are the shapes whose volume the ring sizing has to see: a fast sender (tandem_heavy), several senders into one
server (fan_in), a receiving partition whose samples are told apart by the event records (two_sinks), a partition that
only relays (chain), a source whose rate lives in a profile (profile_source) and an ensemble of replicas."""
import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import oracle_lib as O
from happysim_b200 import _abi as A


def _link(src, dst, latency=0.05):
    return hs.PartitionLink(src, dst, min_latency=latency, latency=hs.ConstantLatency(latency))


def tandem_heavy(rate=500.0):
    """A: Poisson source -> Server(c=4, exp 1 ms) -> [50 ms link] -> B: Server(c=4, exp 2 ms) -> Sink; about 5 000
    Sink samples in B over 10 s."""
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=4, service_time=hs.ExponentialLatency(0.002), downstream=sink)
    sa = hs.Server("A.server", concurrency=4, service_time=hs.ExponentialLatency(0.001), downstream=sb)
    src = hs.Source.poisson(rate=rate, target=sa)
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src]), hs.SimulationPartition("B", entities=[sb, sink])]
    return parts, [_link("A", "B")], dict(duration=10.0, seed=5)


def tandem_light():
    """The 40 req/s x 4 s tandem of test_parallel_linked (the fixture linked_tandem_const): nothing comes near a cap."""
    from test_parallel_linked import tandem
    parts, link, _ = tandem()
    return parts, [link], dict(duration=4.0, seed=5)


def fan_in():
    """A and C both send into B.server: B has no source of its own, its inbox is twice the link buffer."""
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=4, service_time=hs.ExponentialLatency(0.001), downstream=sink)
    sa = hs.Server("A.server", concurrency=2, service_time=hs.ExponentialLatency(0.001), downstream=sb)
    sc = hs.Server("C.server", concurrency=2, service_time=hs.ExponentialLatency(0.001), downstream=sb)
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[hs.Source.poisson(rate=300.0, target=sa, name="A.src")]),
             hs.SimulationPartition("B", entities=[sb, sink]),
             hs.SimulationPartition("C", entities=[sc], sources=[hs.Source.poisson(rate=300.0, target=sc, name="C.src")])]
    return parts, [_link("A", "B"), _link("C", "B", 0.04)], dict(duration=6.0, seed=3)


def two_sinks():
    """B holds two servers with a Sink each, fed from A and from C: B's samples and service times are split between
    them by the event records."""
    k1, k2 = hs.Sink("B.sink1"), hs.Sink("B.sink2")
    s1 = hs.Server("B.s1", concurrency=2, service_time=hs.ExponentialLatency(0.002), downstream=k1)
    s2 = hs.Server("B.s2", concurrency=3, service_time=hs.ExponentialLatency(0.003), downstream=k2)
    sa = hs.Server("A.server", concurrency=2, service_time=hs.ExponentialLatency(0.001), downstream=s1)
    sc = hs.Server("C.server", concurrency=2, service_time=hs.ExponentialLatency(0.001), downstream=s2)
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[hs.Source.poisson(rate=350.0, target=sa, name="A.src")]),
             hs.SimulationPartition("B", entities=[s1, k1, s2, k2]),
             hs.SimulationPartition("C", entities=[sc], sources=[hs.Source.poisson(rate=250.0, target=sc, name="C.src")])]
    return parts, [_link("A", "B"), _link("C", "B")], dict(duration=6.0, seed=9)


def chain():
    """A -> B -> C: B both receives and sends, so its volume, and C's, is set by A's source alone."""
    sink = hs.Sink("C.sink")
    s_c = hs.Server("C.server", concurrency=4, service_time=hs.ExponentialLatency(0.002), downstream=sink)
    s_b = hs.Server("B.server", concurrency=4, service_time=hs.ExponentialLatency(0.001), downstream=s_c)
    s_a = hs.Server("A.server", concurrency=4, service_time=hs.ExponentialLatency(0.001), downstream=s_b)
    parts = [hs.SimulationPartition("A", entities=[s_a], sources=[hs.Source.poisson(rate=400.0, target=s_a)]),
             hs.SimulationPartition("B", entities=[s_b]),
             hs.SimulationPartition("C", entities=[s_c, sink])]
    return parts, [_link("A", "B"), _link("B", "C", 0.03)], dict(duration=6.0, seed=13)


def profile_source():
    """A's source ramps from 100 to 1 200 req/s over 5 s (rate left unset: it lives in the profile)."""
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=4, service_time=hs.ExponentialLatency(0.002), downstream=sink)
    sa = hs.Server("A.server", concurrency=4, service_time=hs.ExponentialLatency(0.001), downstream=sb)
    src = hs.Source.with_profile(hs.LinearRampProfile(duration_s=5.0, start_rate=100.0, end_rate=1200.0), target=sa)
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src]), hs.SimulationPartition("B", entities=[sb, sink])]
    return parts, [_link("A", "B")], dict(duration=6.0, seed=21)


CASES = {"tandem_heavy": tandem_heavy, "tandem_light": tandem_light, "fan_in": fan_in, "two_sinks": two_sinks,
         "chain": chain, "profile_source": profile_source}
# the cases whose volume the ring sizing of a linked run has to see (tandem_light is the control)
HEAVY = ["tandem_heavy", "fan_in", "two_sinks", "chain", "profile_source"]


def build(name):
    parts, links, kw = CASES[name]()
    ps = hs.ParallelSimulation(parts, duration=kw["duration"], links=links, seed=kw["seed"])
    return ps, parts


def _needs_records(m):
    return len(m.ids_of(A.HS_ENT_SINK)) > 1 or len(m.ids_of(A.HS_ENT_SERVER)) > 1


def truth(lm, *, seed, end_ns, n_replicas=1):
    """The oracle's linked run of ``lm`` with every recorder ring large enough that nothing wraps (grown until every
    count is below its cap): (outputs, delivered, lost, window ends).  Event records only where they are needed to tell
    a partition's sinks / servers apart."""
    nP = lm.n_partitions
    caps = [dict(sample_cap=4096, service_cap=4096, record_cap=65536 if _needs_records(m) else 0) for m in lm.models]
    for _ in range(8):
        ps = [O.make_params(seed=seed, end_ns=end_ns, n_replicas=n_replicas, rid_base=q, rid_stride=nP + 1, flags=0,
                            **caps[q]) for q in range(nP)]
        outs, delivered, lost, ends = O.oracle_run_linked(lm, ps, end_ns=end_ns, cseed=seed)
        grown = False
        for q, o in enumerate(outs):
            for cap, count in (("sample_cap", "n_sink_samples"), ("service_cap", "n_service_samples"),
                               ("record_cap", "events_processed")):
                n = int(o["summaries"][count].max())
                if (cap != "record_cap" or caps[q][cap]) and n >= caps[q][cap]:
                    caps[q][cap] = 2 * n + 64
                    grown = True
        if not grown:
            break
    for q, o in enumerate(outs):
        s = o["summaries"]
        assert (s["status"] == 0).all()
        assert (s["n_sink_samples"] < caps[q]["sample_cap"]).all() and (s["n_service_samples"] < caps[q]["service_cap"]).all()
        assert not caps[q]["record_cap"] or (s["events_processed"] < caps[q]["record_cap"]).all()
    return outs, delivered, lost, ends


def split(lm, q, o, r=0):
    """Replica r of partition q's unwrapped truth: {entity id: Sink samples} and {entity id: service times}, split
    between the partition's sinks / servers by the event records when there is more than one."""
    m = lm.models[q]
    s = o["summaries"][r]
    samples = o["sink_samples"][r][: int(s["n_sink_samples"])]
    svc = o["service_samples"][r][: int(s["n_service_samples"])]
    sinks, servers = m.ids_of(A.HS_ENT_SINK), m.ids_of(A.HS_ENT_SERVER)
    rec = o["records"][r][: int(s["events_processed"])] if o.get("records") is not None else None
    if len(sinks) > 1:
        who = rec["entity"][rec["kind"] == A.HS_EV_REQ_SINK]
        assert len(who) == len(samples)
        per_sink = {i: samples[who == i] for i in sinks}
    else:
        per_sink = {i: samples for i in sinks}
    if len(servers) > 1:
        who = rec["entity"][rec["kind"] == A.HS_EV_REQ_WORKER]
        assert len(who) == len(svc)
        per_server = {i: svc[who == i] for i in servers}
    else:
        per_server = {i: svc for i in servers}
    return per_sink, per_server


def check_published(ps, summ, want, delivered, ends, *, own_classes=False):
    """What ParallelSimulation.run() published -- on the script's own objects and in the summary -- against the
    unwrapped oracle truth, exactly."""
    lm = ps._linked
    assert summ.total_windows == len(ends)
    assert summ.total_cross_partition_events == int(delivered[0])
    for q, name in enumerate(lm.names):
        o, m = want[q], lm.models[q]
        s, st = o["summaries"][0], o["entity_stats"][0]
        assert summ.partitions[name].total_events_processed == int(s["events_processed"]), name
        per_sink, per_server = split(lm, q, o)
        for i, obj in enumerate(lm.objects[q]):
            kind, where = int(m.entities["kind"][i]), (name, obj.name)
            if kind == A.HS_ENT_SINK:
                smp = per_sink[i]
                assert len(obj.latencies_s) == len(smp) == int(st[i]["c0"]), (where, len(obj.latencies_s), len(smp))
                assert obj.latencies_s == [float(x) for x in smp["latency_s"]], where
                assert [int(t.nanoseconds) for t in obj.completion_times] == [int(x) for x in smp["completion_ns"]], where
                assert obj.events_received == int(st[i]["c0"]), where
                avg = sum(obj.latencies_s) / len(obj.latencies_s) if own_classes else float(st[i]["f0"]) / int(st[i]["c0"])
                assert obj.average_latency() == avg, where
            elif kind == A.HS_ENT_SERVER:
                svc = per_server[i]
                assert len(obj._service_times) == len(svc), (where, len(obj._service_times), len(svc))
                assert obj._service_times == [float(x) for x in svc], where
                assert (obj.stats.requests_completed, obj.stats.requests_rejected) == (int(st[i]["c2"]), int(st[i]["c3"])), where
                assert (obj.stats_accepted, obj.stats_dropped) == (int(st[i]["c0"]), int(st[i]["c1"])), where
                if not own_classes:
                    qs = summ.entities[obj.name].queue_stats
                    assert (qs.total_accepted, qs.total_dropped) == (int(st[i]["c0"]), int(st[i]["c1"])), where
            elif kind == A.HS_ENT_SOURCE:
                assert obj.generated_count == int(st[i]["c0"]), where


def run_published(name, monkeypatch):
    """ParallelSimulation(case).run() on the oracle: (ps, summary, stand-in run)."""
    from happysim_b200 import linked
    runs = []

    class Recording(O.OracleLinkedRun):
        def __init__(self, lm, *, device=0):
            super().__init__(lm, device=device)
            runs.append(self)
    monkeypatch.setattr(linked, "LinkedRun", Recording)
    ps, parts = build(name)
    summ = ps.run()
    assert len(runs) == 1
    return ps, summ, runs[0]


@pytest.mark.parametrize("name", list(CASES))
def test_published_results_equal_the_unwrapped_oracle_run(name, monkeypatch):
    ps, summ, run = run_published(name, monkeypatch)
    want, delivered, lost, ends = truth(ps._linked, seed=ps._seed, end_ns=ps._end_ns)
    check_published(ps, summ, want, delivered, ends)
    if name in HEAVY:         # the volume these cases exist for: more Sink samples / service starts than 1 000
        assert max(int(o["summaries"]["n_service_samples"][0]) for o in want) > 1000


def test_the_cases_fill_rings_that_the_sizing_of_a_partitions_own_sources_alone_would_give():
    """A ring sized from a partition's own constant-rate sources and its inbox (the first estimate before upstream
    partitions and profiles were counted) wraps in every heavy case: each case tests the sizing, not just the loop."""
    from happysim_b200 import parallel as P
    for name in HEAVY:
        ps, _ = build(name)
        lm = ps._linked
        want, *_ = truth(lm, seed=ps._seed, end_ns=ps._end_ns)
        wraps = []
        for q, m in enumerate(lm.models):
            own = sum(float(m.entities["d0"][i]) for i in m.ids_of(A.HS_ENT_SOURCE))
            ev = max(64, int(P._events_bound(own, m.inbox_cap, ps._end_ns)))
            s = want[q]["summaries"][0]
            wraps.append(max(int(s["n_sink_samples"]), int(s["n_service_samples"])) > ev
                         or (_needs_records(m) and int(s["events_processed"]) > 8 * ev))
        assert any(wraps), name


def test_the_first_caps_hold_every_case_without_a_rerun(monkeypatch):
    """Every source that can reach a partition -- its own, those upstream over links, profiles by their peak rate --
    enters its first ring sizes: none of the cases needs a second run."""
    for name in CASES:
        ps, summ, run = run_published(name, monkeypatch)
        assert len(run.calls) == 1, (name, [c["caps"] for c in run.calls])


def test_rings_that_turn_out_too_small_are_grown_and_the_run_repeated(monkeypatch):
    """A first estimate that is too small (here: forced to the floor) is caught after the run: the caps are grown from
    the counts and the whole linked run repeated from window 0; nothing wrapped reaches the objects."""
    from happysim_b200 import parallel as P
    monkeypatch.setattr(P, "_events_bound", lambda rate, inbox_cap, end_ns: 0.0)
    for name in ("tandem_heavy", "two_sinks"):
        ps, summ, run = run_published(name, monkeypatch)
        assert len(run.calls) == 2, name
        first, last = run.calls[0]["caps"], run.calls[-1]["caps"]
        assert all(c["sample_cap"] == 64 for c in first)
        assert any(b["sample_cap"] > 64 or b["service_cap"] > 64 for b in last)
        want, delivered, lost, ends = truth(ps._linked, seed=ps._seed, end_ns=ps._end_ns)
        check_published(ps, summ, want, delivered, ends)


def test_a_ring_that_never_suffices_raises_and_names_the_partition(monkeypatch):
    """A stand-in whose counts always exceed the caps: after the bounded number of attempts the run raises with the
    partition and the ring, instead of publishing a wrapped ring."""
    from happysim_b200 import linked

    class Overfull(O.OracleLinkedRun):
        def run(self, **kw):
            outs, counts = super().run(**kw)
            c = kw["caps"][1]
            outs[1]["summaries"]["n_service_samples"] = c["service_cap"] + 1
            return outs, counts
    monkeypatch.setattr(linked, "LinkedRun", Overfull)
    ps, parts = build("tandem_light")
    with pytest.raises(RuntimeError, match=r"partition 'B' .* service time ring .* 6 attempts"):
        ps.run()
    assert parts[1].entities[1].latencies_s == []          # nothing was written back


def test_ensemble_rings_hold_every_replicas_items(monkeypatch):
    """run_ensemble(16) of tandem_heavy: every replica's returned rings, unrolled, are that replica's unwrapped oracle
    run item for item; the rings may have been grown, but their widths hold every item."""
    from happysim_b200 import linked
    monkeypatch.setattr(linked, "LinkedRun", O.OracleLinkedRun)
    ps, _ = build("tandem_heavy")
    n = 16
    ens, delivered, lost = ps.run_ensemble(n)
    lm = ps._linked
    want, wd, wl, _ = truth(lm, seed=ps._seed, end_ns=ps._end_ns, n_replicas=n)
    assert np.array_equal(delivered, wd) and np.array_equal(lost, wl) and len({int(x) for x in wd}) > n // 2
    check_ensemble(lm, ens, want, n)


def check_ensemble(lm, ens, want, n):
    for q, name in enumerate(lm.names):
        got, w = ens[name], want[q]
        assert got["entity_stats"].tobytes() == w["entity_stats"].tobytes(), name
        for f in ("events_processed", "final_time_ns", "heap_left", "status", "n_sink_samples", "n_service_samples"):
            assert np.array_equal(got["summaries"][f], w["summaries"][f]), (name, f)
        for ring, count in (("sink_samples", "n_sink_samples"), ("service_samples", "n_service_samples"),
                            ("records", "events_processed")):
            if got.get(ring) is None:
                continue
            width = got[ring].shape[1]
            for r in range(n):
                k = int(w["summaries"][count][r])
                assert k <= width, (name, ring, r, k, width)
                items = A.unroll_ring(got[ring][r], k, width)
                if w.get(ring) is not None:
                    assert items.tobytes() == w[ring][r][:k].tobytes(), (name, ring, r)
        assert max(int(x) for x in w["summaries"]["n_service_samples"]) > 1000


def test_tandem_heavy_lowers_to_the_fixture_model():
    """The API declaration of tandem_heavy is the model of the reference fixture linked_tandem_heavy."""
    ps, _ = build("tandem_heavy")
    lm, kw, z = G.load_linked("linked_tandem_heavy")
    got = ps._linked
    assert got.window_s == lm.window_s and ps._end_ns == kw["end_ns"] and ps._seed == kw["seed"]
    for q in range(2):
        assert got.models[q].entities.tobytes() == lm.models[q].entities.tobytes()
    assert got.links == lm.links
    assert len(z["p1_sink_samples"]) > 4000


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
def test_tandem_heavy_with_the_references_own_objects(monkeypatch):
    """Case tandem_heavy declared with the reference's own classes: the same lists land on the reference's objects."""
    G.import_reference()
    from happysimulator.components.common import Sink
    from happysimulator.components.server.server import Server
    from happysimulator.distributions.constant import ConstantLatency
    from happysimulator.distributions.exponential import ExponentialLatency
    from happysimulator.load.source import Source
    from happysimulator.parallel.link import PartitionLink
    from happysimulator.parallel.partition import SimulationPartition
    from happysim_b200 import linked
    monkeypatch.setattr(linked, "LinkedRun", O.OracleLinkedRun)
    sink = Sink("B.sink")
    sb = Server("B.server", concurrency=4, service_time=ExponentialLatency(0.002), downstream=sink)
    sa = Server("A.server", concurrency=4, service_time=ExponentialLatency(0.001), downstream=sb)
    src = Source.poisson(rate=500.0, target=sa)
    parts = [SimulationPartition(name="A", entities=[sa, sa.queue, sa.driver, sa.worker], sources=[src]),
             SimulationPartition(name="B", entities=[sb, sb.queue, sb.driver, sb.worker, sink])]
    link = PartitionLink(source_partition="A", dest_partition="B", min_latency=0.05, latency=ConstantLatency(0.05))
    ps = hs.ParallelSimulation(parts, duration=10.0, links=[link], seed=5)
    summ = ps.run()
    want, delivered, lost, ends = truth(ps._linked, seed=ps._seed, end_ns=ps._end_ns)
    check_published(ps, summ, want, delivered, ends, own_classes=True)
    assert len(sink.latencies_s) > 4000
