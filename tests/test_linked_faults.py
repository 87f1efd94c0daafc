"""Node faults (CrashNode, PauseNode) in the partitions of a linked ParallelSimulation, on the CPU: the fault oracle's
linked run (tests/layered_oracle.c, hs_layered_oracle_run_linked) against the fixtures recorded from the unmodified
reference (tests/golden/lfault_*.npz) and the 48 random models (random_linked_faults.npz), the lowering of a
partition's schedule, the mirror's whole host path on the oracle, and the C-ABI's validation of linked partitions."""
import os

import numpy as np
import pytest

import layered_oracle_lib as LO
import golden_lib as G
import happysim_b200 as hs
import linked_fault_models as LF
import oracle_lib as O
from happysim_b200 import _abi as A, engine

CASES = G.case_names("lfault_")


def run_oracle(lm, kw, caps):
    nP = lm.n_partitions
    ps = [O.make_params(seed=kw["seed"], end_ns=kw["end_ns"], rid_base=q, rid_stride=nP + 1, **caps[q]) for q in range(nP)]
    return LO.run_linked(lm, ps, end_ns=kw["end_ns"], cseed=kw["seed"])


def check_partition(z, q, got, r=0):
    """partition q of a lfault_ fixture against replica r: golden_lib.check_linked_partition's comparisons, with the
    status word the reference implies (HS_ST_FAULT_TIE where a fault event tied) and events_cancelled"""
    pre = f"p{q}_"
    s, ws = got["summaries"][r], z[pre + "summaries"][0]
    for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
        assert int(s[f]) == int(ws[f]), (q, f, int(s[f]), int(ws[f]))
    assert got["entity_stats"][r].tobytes() == z[pre + "entity_stats"][0].tobytes(), f"partition {q}: entity statistics differ"
    for k in ("records", "sink_samples", "service_samples"):
        n = len(z[pre + k])
        assert got[k][r][:n].tobytes() == z[pre + k].tobytes(), f"partition {q}: {k} differ"
    fr = [i for i in range(len(got["entity_stats"][r])) if int(z[pre + "entities"]["kind"][i]) == A.HS_ENT_FAULT]
    assert int(got["entity_stats"][r][fr]["c1"].sum()) == int(z[pre + "events_cancelled"])


def test_there_are_fixtures():
    assert {"lfault_tandem_crash_downstream", "lfault_tandem_pause_sink", "lfault_sender_crash_drains", "lfault_fanin_mixed",
            "lfault_grid_tie"} <= set(CASES)


@pytest.mark.parametrize("name", CASES)
def test_linked_fault_oracle_reproduces_fixture(name):
    lm, kw, z = G.load_linked(name)
    caps = [G.linked_caps(z, q) for q in range(lm.n_partitions)]
    outs, delivered, lost, ends = run_oracle(lm, kw, caps)
    assert len(ends) == int(z["total_windows"]) and int(delivered[0]) == int(z["cross_events"])
    for q in range(lm.n_partitions):
        check_partition(z, q, outs[q])
        tie = bool(int(outs[q]["summaries"]["status"][0]) & A.HS_ST_FAULT_TIE)
        assert int(outs[q]["summaries"]["status"][0]) & ~A.HS_ST_FAULT_TIE == 0
        assert tie == bool(int(z[f"p{q}_tie"])), (q, "HS_ST_FAULT_TIE exactly where the reference tied")
    assert any(int(z[f"p{q}_tie"]) for q in range(lm.n_partitions)) == (name == "lfault_grid_tie")


def test_the_fixtures_cover_what_they_are_meant_to():
    """the sender-side crash drains across the link; faults fire at t = 0, at a window end and beyond end_time; a
    cancelled handle is popped and counted; deliveries reach a crashed entity"""
    lm, kw, z = G.load_linked("lfault_sender_crash_drains")
    rec = z["p0_records"]
    crash, restart = (int(t) for t in rec[rec["kind"] == A.HS_EV_FAULT]["time_ns"])
    cont = rec[(rec["kind"] == A.HS_EV_CONTINUATION) & (rec["time_ns"] > crash) & (rec["time_ns"] < restart)]
    assert len(cont) > 0, "the crashed sender still completes queued work"
    lm, kw, z = G.load_linked("lfault_fanin_mixed")
    ends = lm.window_ends(kw["end_ns"])
    fe = z["p2_entities"][z["p2_entities"]["kind"] == A.HS_ENT_FAULT]
    assert 0 in fe["l0"] and any(int(t) in ends for t in fe["l0"]) and int(fe["l0"].max()) > kw["end_ns"]
    assert int(z["p0_events_cancelled"]) == 2 and int(z["p2_summaries"]["heap_left"][0]) >= 1
    lm, kw, z = G.load_linked("lfault_tandem_crash_downstream")
    rec = z["p1_records"]
    crash, restart = (int(t) for t in rec[rec["kind"] == A.HS_EV_FAULT]["time_ns"])
    assert ((rec["kind"] == A.HS_EV_REQ_ENQUEUE) & (rec["time_ns"] > crash) & (rec["time_ns"] < restart)).sum() > 0


R = np.load(os.path.join(G.GOLDEN_DIR, "random_linked_faults.npz"))


@pytest.mark.parametrize("seed", range(LF.RANDOM_SEEDS))
def test_linked_fault_oracle_equals_the_reference_on_random_models(seed):
    lm, end_s, what, _ = LF.random_linked_fault_model(seed)
    nP, end_ns = lm.n_partitions, int(end_s * 1e9)
    ps = [O.make_params(seed=1000 + seed, end_ns=end_ns, rid_base=q, rid_stride=nP + 1) for q in range(nP)]
    outs, delivered, lost, ends = LO.run_linked(lm, ps, end_ns=end_ns, cseed=1000 + seed)
    top = R["tops"][R["tops"]["seed"] == seed][0]
    rows = R["rows"][R["rows"]["seed"] == seed]
    assert int(delivered[0]) == int(top["delivered"]), what
    # the reference's coordinator stops once every partition's heap is empty (a source crashed for good can empty
    # them); the windows after that change nothing
    assert len(ends) == int(top["windows"]) or (len(ends) > int(top["windows"]) and not rows["heap_left"].any()), what
    for q, o in enumerate(outs):
        s, w = o["summaries"][0], rows[rows["part"] == q][0]
        for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
            assert int(s[f]) == int(w[f]), (what, q, f, int(s[f]), int(w[f]))
        assert LF.digest(o["entity_stats"][0]) == int(w["stats_digest"]), (what, q)
        fr = lm.models[q].ids_of(A.HS_ENT_FAULT)
        assert int(o["entity_stats"][0][fr]["c1"].sum()) == int(w["events_cancelled"]), (what, q)
        if not int(w["tie"]):
            assert int(s["status"]) & A.HS_ST_FAULT_TIE == 0, (what, q)


def test_the_random_schedules_cover_what_they_are_meant_to():
    n = {"faults": 0, "cancelled": 0, "pause": 0, "no_restart": 0}
    for seed in range(LF.RANDOM_SEEDS):
        *_, sch = LF.random_linked_fault_model(seed)
        for faults in sch:
            n["faults"] += len(faults)
            n["cancelled"] += sum(f[4] for f in faults)
            n["pause"] += sum(f[0] == "pause" for f in faults)
            n["no_restart"] += sum(f[3] is None for f in faults)
    assert n["faults"] > 100 and min(n.values()) >= 10, n
    assert int(R["rows"]["events_cancelled"].sum()) > 10


# ---- lowering ---------------------------------------------------------------------------------------------------
def tandem(schedule_b=None, schedule_a=None):
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=2, service_time=hs.ExponentialLatency(0.015), downstream=sink)
    sa = hs.Server("A.server", service_time=hs.ExponentialLatency(0.01), downstream=sb)
    src = hs.Source.poisson(rate=40.0, target=sa)
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src], fault_schedule=schedule_a),
             hs.SimulationPartition("B", entities=[sb, sink], fault_schedule=schedule_b)]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=hs.ConstantLatency(0.05))
    return parts, link, (src, sa, sb, sink)


def test_the_mirrors_schedule_lowers_to_the_fixture_rows():
    fs = hs.FaultSchedule()
    fs.add(hs.CrashNode("B.server", at=1.0, restart_at=2.2))
    parts, link, _ = tandem(fs)
    ps = hs.ParallelSimulation(parts, duration=4.0, links=[link], seed=5)
    lm, kw, z = G.load_linked("lfault_tandem_crash_downstream")
    for q in range(2):
        assert ps._linked.models[q].entities.tobytes() == lm.models[q].entities.tobytes(), q
        hs.engine.validate_model(ps._linked.models[q], partition=True)


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
def test_the_references_schedule_and_objects_lower_to_the_fixture_rows():
    G.import_reference()
    from happysimulator.components.common import Sink
    from happysimulator.components.server.server import Server
    from happysimulator.distributions.constant import ConstantLatency
    from happysimulator.distributions.exponential import ExponentialLatency
    from happysimulator.faults import CrashNode, FaultSchedule
    from happysimulator.load.source import Source
    from happysimulator.parallel.link import PartitionLink
    from happysimulator.parallel.partition import SimulationPartition
    sink = Sink("B.sink")
    sb = Server("B.server", concurrency=2, service_time=ExponentialLatency(0.015), downstream=sink)
    sa = Server("A.server", service_time=ExponentialLatency(0.01), downstream=sb)
    src = Source.poisson(rate=40.0, target=sa)
    fs = FaultSchedule()
    fs.add(CrashNode("B.server", at=1.0, restart_at=2.2))
    parts = [SimulationPartition(name="A", entities=[sa, sa.queue, sa.driver, sa.worker], sources=[src]),
             SimulationPartition(name="B", entities=[sb, sb.queue, sb.driver, sb.worker, sink], fault_schedule=fs)]
    link = PartitionLink(source_partition="A", dest_partition="B", min_latency=0.05, latency=ConstantLatency(0.05))
    ps = hs.ParallelSimulation(parts, duration=4.0, links=[link], seed=5)
    lm, kw, z = G.load_linked("lfault_tandem_crash_downstream")
    for q in range(2):
        assert ps._linked.models[q].entities.tobytes() == lm.models[q].entities.tobytes(), q


def test_sort_indices_come_from_each_partitions_own_counter():
    """A's fault events follow A's one source; B has none, so its first fault event takes index 0 -- the same
    schedule in both partitions lowers to different indices"""
    fa, fb = hs.FaultSchedule(), hs.FaultSchedule()
    fa.add(hs.CrashNode("A.server", at=0.5, restart_at=0.7))
    fb.add(hs.PauseNode("B.sink", start=0.5, end=0.7))
    parts, link, _ = tandem(fb, fa)
    ps = hs.ParallelSimulation(parts, duration=1.0, links=[link])
    rows = [m.entities[m.entities["kind"] == A.HS_ENT_FAULT] for m in ps._linked.models]
    assert list(rows[0]["i3"]) == [1, 2] and list(rows[1]["i3"]) == [0, 1]


def test_a_fault_naming_another_partitions_entity_raises_key_error():
    fs = hs.FaultSchedule()
    fs.add(hs.CrashNode("A.server", at=1.0))            # A.server lives in partition A, the schedule is B's
    parts, link, _ = tandem(fs)
    with pytest.raises(KeyError):
        hs.ParallelSimulation(parts, duration=2.0, links=[link])


def test_other_fault_classes_are_refused():
    from dataclasses import dataclass

    @dataclass(frozen=True)
    class ReduceCapacity:
        entity_name: str
        at: float
    fs = hs.FaultSchedule()
    fs.add(ReduceCapacity("B.server", at=1.0))
    parts, link, _ = tandem(fs)
    with pytest.raises(hs.UnsupportedModelError, match="ReduceCapacity"):
        hs.ParallelSimulation(parts, duration=2.0, links=[link])


def test_partition_validation_accepts_faults_next_to_remote_rows():
    """hs_partition_validate takes FAULT and REMOTE rows in one model (a linked partition with a schedule) while
    hs_model_validate, which checks a model on its own, still refuses them; a FAULT row that targets the REMOTE row,
    and any row after a FAULT row, are refused either way"""
    b = hs.ModelBuilder()
    src = b.source(rate=4.0); srv = b.server()
    rem = b.remote(link=0, dest_entity=0)
    b.set_target(src, srv); b.set_target(srv, rem)
    b.fault(target=srv, time_ns=10**9, crash=True, sort_index=1)
    m = b.build(); m.outbox_cap = 16
    engine.validate_model(m, partition=True)
    with pytest.raises(Exception, match="hs_partition_upload"):
        engine.validate_model(m)
    bad = m.entities.copy()
    bad["target"][m.ids_of(A.HS_ENT_FAULT)[0]] = rem
    m.entities = bad
    with pytest.raises(Exception, match="REMOTE"):
        engine.validate_model(m, partition=True)
    m.entities = np.concatenate([m.entities, np.array([(A.HS_ENT_SINK, -1, 0, 0, 0, 0, -1, 0.0, 0.0)], dtype=A.ENTITY_DTYPE)])
    m.entities["target"][m.ids_of(A.HS_ENT_FAULT)[0]] = srv
    m.names = list(m.names) + ["Sink"]
    with pytest.raises(Exception, match="after every other row"):
        engine.validate_model(m, partition=True)


# ---- the mirror's host path, on the layered oracle -----------------------------------------------------------------
def test_run_writes_crashed_and_each_partition_reports_its_cancelled_events(monkeypatch):
    from happysim_b200 import linked
    monkeypatch.setattr(linked, "LinkedRun", LO.OracleCellsLinkedRun)
    fa, fb = hs.FaultSchedule(), hs.FaultSchedule()
    h = fa.add(hs.CrashNode("A.server", at=0.5, restart_at=0.7))
    fb.add(hs.CrashNode("B.sink", at=1.0))
    parts, link, (src, sa, sb, sink) = tandem(fb, fa)
    ps = hs.ParallelSimulation(parts, duration=2.0, links=[link], seed=3)
    h.cancel()                                           # after building: read when run() runs
    s = ps.run()
    assert s.partitions["A"].events_cancelled == 2 and s.partitions["B"].events_cancelled == 0
    assert sink._crashed is True and getattr(sa, "_crashed", False) is False
    assert ps.fault_ties == 0 and sb._requests_completed == int(ps.last_outputs[1]["entity_stats"][0][0]["c2"]) > 0
    # B's only pending event at its first barrier is the crash at 1 s: B processes it past its window end and its clock
    # moves to 1 s, so every request delivered before that is "time travel" -- and the sink crashes as it would start
    assert sink.events_received == 0 and s.partitions["B"].duration_s >= 1.0
