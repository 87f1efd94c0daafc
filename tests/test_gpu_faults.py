"""Node faults (CrashNode, PauseNode) on the device: both general engines against the fixtures recorded from the
unmodified reference (tests/golden/fault_*.npz), larger ensembles against the fault oracle (tests/fault_oracle.c) on
every replica, windowed runs cut between a crash and its restart, ties, install() and the mirror's write-back."""
import random

import numpy as np
import pytest

import fault_oracle_lib as FO
import golden_lib as G
import happysim_b200 as hs
from happysim_b200 import engine, _abi as A

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.mark.parametrize("eng_id", [0, 1, 3])          # auto (the thread engine: faults are not lane-eligible), warp, thread
@pytest.mark.parametrize("name", [n for n in G.case_names("fault_") if not n.startswith("fault_tie")])
def test_engine_reproduces_fault_fixture(eng, name, eng_id):
    model, kw, z = G.load(name)
    eng.upload(model)
    kw = dict(kw)
    rid = kw.pop("rid_base")
    eng.run(engine.make_params(n_replicas=5, rid_base=rid - 2 if rid >= 2 else rid, rid_stride=1, engine=eng_id, **G.caps(z), **kw))
    info = eng.last_launch()
    assert info["engine"] == (1 if eng_id == 1 else 3)
    assert info["flags"] & 32, "the FAULTS instantiation"
    got = eng.read_outputs()
    G.check_against(z, got, r=2 if rid >= 2 else 0)
    assert int(got["summaries"]["status"][2 if rid >= 2 else 0]) == 0


def test_lane_engine_refuses_faults(eng):
    model, kw, z = G.load("fault_mm1_crash_restart")
    eng.upload(model)
    with pytest.raises(Exception, match="fault"):
        eng.run(engine.make_params(n_replicas=4, engine=2, **kw))


def _farm_with_faults(n_servers=64, n_crash=8):
    m = hs.lb_round_robin(n_servers=n_servers, rate=512.0)
    ents = list(m.entities.tolist())
    servers = [i for i in range(m.n_entities) if int(m.entities["kind"][i]) == A.HS_ENT_SERVER]
    rows, k = [], 1
    for j in range(n_crash):
        s = servers[j * (n_servers // n_crash)]
        rows.append((A.HS_ENT_FAULT, s, 0, 1, 0, k, int((3 + 0.25 * j) * 1e9), 0.0, 0.0)); k += 1
        rows.append((A.HS_ENT_FAULT, s, 0, 0, 0, k, int((6 + 0.25 * j) * 1e9), 0.0, 0.0)); k += 1
    m.entities = np.array(ents + rows, dtype=A.ENTITY_DTYPE)
    m.names = list(m.names) + [f"fault{i}" for i in range(len(rows))]
    return m


@pytest.mark.parametrize("n", [1024, 16384])
def test_ensembles_match_the_fault_oracle_on_every_replica(eng, n):
    """A configs[2]-shaped farm with 8 backends crashed and restarted: both geometries of the thread engine (one
    replica per warp at 1 024, several at 16 384) and the warp engine against the fault oracle, replica for replica,
    recorder rings included."""
    m = _farm_with_faults()
    eng.upload(m)
    kw = dict(seed=9, end_ns=8 * 10**9, n_replicas=n, record_cap=512, sample_cap=256, service_cap=256)
    want = FO.run(m, engine.make_params(**kw))
    for e in (3, 1):
        eng.run(engine.make_params(engine=e, **kw))
        got = eng.read_outputs(); li = eng.last_launch()
        assert li["flags"] & 32
        if e == 3:
            assert li["lane_stride"] == (32 if n == 1024 else 4)
        for k in ("summaries", "entity_stats", "records", "sink_samples", "service_samples"):
            assert got[k].tobytes() == want[k].tobytes(), (e, k)
    fr = m.ids_of(A.HS_ENT_FAULT)
    assert (want["entity_stats"][:, fr]["c0"] == 1).all()
    assert int(want["summaries"]["status"].max()) == 0


def test_mixed_fixture_ensemble_matches_the_fault_oracle_and_is_tie_free(eng):
    """Every replica of the mixed schedule (overlap, cancelled handle, t = 0, beyond end_time) on both engines equals
    the fault oracle, status words included: no replica is flagged with a tie the reference would not have."""
    model, kw, z = G.load("fault_mm1_mixed")
    eng.upload(model)
    kw = dict(kw); kw.pop("rid_base")
    p = dict(n_replicas=1024, rid_stride=1, record_cap=1024, sample_cap=512, service_cap=512, **kw)
    want = FO.run(model, engine.make_params(**p))
    assert int(want["summaries"]["status"].max()) == 0
    for e in (1, 3):
        eng.run(engine.make_params(engine=e, **p))
        got = eng.read_outputs()
        for k in ("summaries", "entity_stats", "records", "sink_samples", "service_samples"):
            assert got[k].tobytes() == want[k].tobytes(), (e, k)


@pytest.mark.parametrize("eng_id", [1, 3])
def test_windowed_run_cut_inside_a_crash_matches_the_uncut_run(eng, eng_id):
    model, kw, z = G.load("fault_mm1_crash_restart")
    eng.upload(model)
    kw = dict(kw)
    base = dict(n_replicas=64, record_cap=4096, sample_cap=2048, service_cap=2048, engine=eng_id, **kw)
    eng.run(engine.make_params(**base))
    whole = eng.read_outputs()
    for cut in (4.0, 5.0):
        eng.run(engine.make_params(window_end_ns=int(cut * 1e9), **base))
        eng.run(engine.make_params(resume=1, **base))
        got = eng.read_outputs()
        for k in ("summaries", "entity_stats", "records", "sink_samples", "service_samples"):
            assert got[k].tobytes() == whole[k].tobytes(), (cut, k)


def test_tie_with_a_pending_fault_is_flagged(eng):
    """The fixture recorded from the reference where the source's in-run tick at 2 s (sort index 1 from the run's
    counter) ties with the crash at 2.0 s (bootstrap index 1): both engines flag it on the device; the fault oracle,
    which restates heapq, flags it too (tests/test_faults.py)."""
    model, kw, z = G.load("fault_tie_constant")
    eng.upload(model)
    for e in (1, 3):
        eng.run(engine.make_params(n_replicas=4, engine=e, **G.caps(z), **kw))
        st = eng.read_outputs()["summaries"]["status"]
        assert (st == A.HS_ST_FAULT_TIE).all(), (e, st)


def test_mirror_write_back():
    sink = hs.Sink()
    src_srv = hs.Server("Server", service_time=hs.ExponentialLatency(0.1), downstream=sink)
    src = hs.Source.poisson(rate=8.0, target=src_srv, name="Source")
    fs = hs.api.FaultSchedule()
    fs.add(hs.api.CrashNode("Server", at=3.0, restart_at=6.5))
    fs.add(hs.api.CrashNode("Sink", at=8.0))
    h = fs.add(hs.api.PauseNode("Server", start=9.0, end=9.5))
    sim = hs.Simulation(sources=[src], entities=[src_srv, sink], end_time=hs.Instant.from_seconds(10.0), fault_schedule=fs)
    h.cancel()
    s = sim.run()
    assert s.events_cancelled == 2
    assert sink._crashed is True and src_srv._crashed is False
    st = fs.stats
    assert (st.faults_scheduled, st.faults_activated, st.faults_deactivated, st.faults_cancelled) == (3, 0, 0, 1)


def test_install_runs_a_faulted_quickstart_like_the_reference():
    """The stock-seeded README quick-start with a crash and restart of its server, once on the reference's loop and
    once under install() in the same process: every latency, every completion time, events_cancelled and the global
    generators' next draws match."""
    if not G.HAVE_REF:
        pytest.skip(G.NO_REF)
    G.import_reference()
    from happysimulator import Instant, Simulation, Sink, Source
    from happysimulator.components.server.server import Server
    from happysimulator.distributions.exponential import ExponentialLatency
    from happysimulator.faults import CrashNode, FaultSchedule

    def script():
        random.seed(42); np.random.seed(42)
        sink = Sink()
        server = Server("Server", service_time=ExponentialLatency(0.1), downstream=sink)
        src = Source.poisson(rate=8, target=server)
        fs = FaultSchedule()
        fs.add(CrashNode("Server", at=20.0, restart_at=35.0))
        h = fs.add(CrashNode("Sink", at=40.0, restart_at=41.0))
        sim = Simulation(sources=[src], entities=[server, sink], end_time=Instant.from_seconds(60.0), fault_schedule=fs)
        h.cancel()
        s = sim.run()
        return s, sink, server, (random.random(), float(np.random.random()))
    want = script()
    hs.install()
    try:
        got = script()
        st = hs.install_stats()
    finally:
        hs.uninstall()
    assert st["device_runs"] >= 1 and st["fallbacks"] == 0
    assert got[0].total_events_processed == want[0].total_events_processed
    assert got[0].events_cancelled == want[0].events_cancelled == 2
    assert got[1].latencies_s == want[1].latencies_s
    assert [t.nanoseconds for t in got[1].completion_times] == [t.nanoseconds for t in want[1].completion_times]
    assert got[2]._crashed == want[2]._crashed and got[3] == want[3]


def test_mirror_ensembles_read_cancellation_at_run_time():
    def build():
        sink = hs.Sink()
        srv = hs.Server("Server", service_time=hs.ExponentialLatency(0.1), downstream=sink)
        src = hs.Source.poisson(rate=8.0, target=srv, name="Source")
        fs = hs.FaultSchedule()
        h = fs.add(hs.CrashNode("Server", at=2.0, restart_at=4.0))
        sim = hs.Simulation(sources=[src], entities=[srv, sink], end_time=hs.Instant.from_seconds(6.0), fault_schedule=fs)
        h.cancel()
        return sim
    res = hs.ParallelRunner().run_replicas(build, 8, base_seed=3)
    assert all(r.summary.events_cancelled == 2 for r in res)
