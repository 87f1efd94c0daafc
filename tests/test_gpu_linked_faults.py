"""Node faults in the partitions of a linked ParallelSimulation, on the device: the thread engine's LINKED | FAULTS
instantiations against the fixtures recorded from the unmodified reference (tests/golden/lfault_*.npz), ensembles
against the linked fault oracle (tests/layered_oracle.c) on every replica, the random models, and the mirror's
ParallelSimulation.run() / run_ensemble()."""
import numpy as np
import pytest

import layered_oracle_lib as LO
import golden_lib as G
import happysim_b200 as hs
import linked_fault_models as LF
from happysim_b200 import _abi as A, engine
from happysim_b200.linked import LinkedModel, LinkedRun, LinkSpec

pytestmark = pytest.mark.gpu

WF_HEAPTOP, WF_LINKED, WF_FAULTS = 8, 16, 32          # HS_WF_* template flags of csrc/hs_warp_engine.cuh
KEYS = ("summaries", "entity_stats", "records", "sink_samples", "service_samples")


def _params(lm, seed, end_ns, n, caps):
    nP = lm.n_partitions
    return [engine.make_params(seed=seed, end_ns=end_ns, n_replicas=n, rid_base=q, rid_stride=nP + 1,
                               flags=A.HS_RUN_ORDER_HASH, **(caps[q] if isinstance(caps, list) else caps)) for q in range(nP)]


def _launches(run, n, seed, end_ns, caps):
    """LinkedRun.run, keeping hs_last_launch of every partition's last window"""
    outs, counts = run.run(seed=seed, end_ns=end_ns, n_replicas=n, caps=caps, flags=A.HS_RUN_ORDER_HASH)
    return outs, counts, [e.last_launch() for e in run.engines]


@pytest.mark.parametrize("name", G.case_names("lfault_"))
def test_device_reproduces_linked_fault_fixture(name):
    """replica 0 of a small ensemble equals the reference's run, partition by partition; the tie case is flagged
    (HS_ST_FAULT_TIE) in the partition where the reference tied, and only there"""
    lm, kw, z = G.load_linked(name)
    caps = [G.linked_caps(z, q) for q in range(lm.n_partitions)]
    run = LinkedRun(lm)
    try:
        outs, (delivered, lost, over), infos = _launches(run, 3, kw["seed"], kw["end_ns"], caps)
    finally:
        run.close()
    assert run.windows == int(z["total_windows"]) and int(delivered[0]) == int(z["cross_events"]) and not over.any()
    for q, info in enumerate(infos):
        # a partition without a schedule keeps the LINKED kernel it ran before
        want_fl = WF_LINKED | (WF_FAULTS if lm.models[q].ids_of(A.HS_ENT_FAULT) else 0)
        assert info["engine"] == 3 and info["flags"] & (WF_LINKED | WF_FAULTS) == want_fl, (q, info)
        st = int(outs[q]["summaries"]["status"][0])
        tie = bool(int(z[f"p{q}_tie"]))
        assert bool(st & A.HS_ST_FAULT_TIE) == tie, (q, st)
        assert st & ~(A.HS_ST_FAULT_TIE | A.HS_ST_LINK_TIE) == 0, (q, st)
        if not any(int(z[f"p{k}_tie"]) for k in range(lm.n_partitions)):
            # a tied pair is ordered by heapq's layout in the reference, by slot number here: compared where none tied
            G.check_linked_partition(z, q, outs[q])
            fr = lm.models[q].ids_of(A.HS_ENT_FAULT)
            assert int(outs[q]["entity_stats"][0][fr]["c1"].sum()) == int(z[f"p{q}_events_cancelled"])


def _faulty_fanout():
    """A: Source(400/s) -> LB over 8 servers; 4 of them forward to B's server pool over a link, 4 to A's sink.  B: 4
    servers behind an LB -> Sink, and a source of its own.  Crashes and restarts on both sides, pauses of A's LB and B's
    sink, a crash for good, a crash at t = 0 and a cancelled crash."""
    a = hs.ModelBuilder()
    src = a.source("A.src", rate=400.0)
    ss = [a.server(f"A.s{k}", mean_service_s=0.015) for k in range(8)]
    lb = a.load_balancer("A.lb", backends=ss)
    snk = a.sink("A.sink")
    rem = a.remote("B.lb@A", link=0, dest_entity=4)
    a.set_target(src, lb)
    for k, s in enumerate(ss):
        a.set_target(s, rem if k % 2 else snk)
    ma = a.build(); ma.outbox_cap = 256
    b = hs.ModelBuilder()
    bs = [b.server(f"B.s{k}", concurrency=2, mean_service_s=0.02) for k in range(4)]
    b.load_balancer("B.lb", backends=bs)
    bsnk = b.sink("B.sink")
    for s in bs:
        b.set_target(s, bsnk)
    b.set_target(b.source("B.tick", rate=50.0), b.counter("B.ticks"))
    mb = b.build(); mb.inbox_cap = 512
    assert int(mb.entities["kind"][4]) == A.HS_ENT_LB and mb.names[4] == "B.lb"
    lm = LinkedModel([ma, mb], ["A", "B"], [[LinkSpec(1, A.HS_SVC_EXPONENTIAL, 0.04, 0.05, 0)], []], window_s=0.02)
    sch = [[("crash", "A.s1", 0.3, 0.9, False), ("crash", "A.s3", 0.5, None, False), ("pause", "A.lb", 1.1, 1.2, False),
            ("crash", "A.s5", 0.2, 0.4, True)],
           [("crash", "B.s0", 0.25, 0.8, False), ("pause", "B.sink", 0.6, 0.7, False), ("crash", "B.lb", 1.3, 1.35, False),
            ("crash", "B.s2", 0.0, 1.0, False)]]
    return LF.linked_with_faults(lm, sch)


@pytest.mark.parametrize("n", [1024, 16384])
def test_ensembles_match_the_linked_fault_oracle_on_every_replica(n):
    """every replica of every partition, recorder rings and status words included, against the linked fault oracle.
    1 024 replicas run one replica per warp (lane stride 32, no heap top), 16 384 several per warp with the heap's top
    levels in shared memory: both LINKED | FAULTS kernels, with and without HEAPTOP"""
    lm = _faulty_fanout()
    seed, end_ns = 21, int(1.5e9)
    caps = dict(record_cap=1024, sample_cap=512, service_cap=512)
    run = LinkedRun(lm)
    try:
        outs, (delivered, lost, over), infos = _launches(run, n, seed, end_ns, caps)
    finally:
        run.close()
    want, wd, wl, ends = LO.run_linked_parallel(lm, _params(lm, seed, end_ns, n, caps), end_ns=end_ns, cseed=seed)
    assert not over.any()
    assert (delivered == wd).all() and (lost == wl).all()
    for q, info in enumerate(infos):
        assert info["flags"] & (WF_LINKED | WF_FAULTS) == (WF_LINKED | WF_FAULTS), info
        if n == 1024:
            assert info["lane_stride"] == 32 and not info["flags"] & WF_HEAPTOP, info
        else:
            assert info["lane_stride"] < 32 and info["flags"] & WF_HEAPTOP and info["heap_top"] > 0, info
        for k in KEYS:
            g, w = outs[q][k], want[q][k]
            if k == "summaries":          # the oracle does not model HS_ST_LINK_TIE (a tie among delivered events)
                g = g.copy(); g["status"] &= ~np.uint32(A.HS_ST_LINK_TIE)
            assert g.tobytes() == w.tobytes(), (n, q, k)
    fired = want[0]["entity_stats"][:, lm.models[0].ids_of(A.HS_ENT_FAULT)]
    assert (fired["c1"][:, -2:] == 1).all() and int(want[1]["summaries"]["status"].max()) == 0


def test_random_linked_fault_models_on_the_device():
    """the 48 random models (oracle == reference on all of them, tests/test_linked_faults.py): 6 replicas each on the
    device against the linked fault oracle; a replica with a tie of either kind is left out of the comparison of its
    results (on the grid models that can be all of them), and at least half of all replicas are compared"""
    compared = 0
    for seed in range(LF.RANDOM_SEEDS):
        lm, end_s, what, _ = LF.random_linked_fault_model(seed)
        end_ns = int(end_s * 1e9)
        caps = dict(record_cap=8192, sample_cap=4096, service_cap=4096)
        run = LinkedRun(lm)
        try:
            outs, (delivered, lost, over), infos = _launches(run, 6, 1000 + seed, end_ns, caps)
        finally:
            run.close()
        want, wd, wl, _ = LO.run_linked(lm, _params(lm, 1000 + seed, end_ns, 6, caps), end_ns=end_ns, cseed=1000 + seed)
        tie = np.zeros(6, bool)
        for q in range(lm.n_partitions):
            tie |= (outs[q]["summaries"]["status"] & (A.HS_ST_LINK_TIE | A.HS_ST_FAULT_TIE)) != 0
            if lm.models[q].ids_of(A.HS_ENT_FAULT):
                assert infos[q]["flags"] & WF_FAULTS, (what, q)
        assert (delivered == wd)[~tie].all() and (lost == wl)[~tie].all(), what
        compared += int((~tie).sum())
        for q in range(lm.n_partitions):
            for r in np.nonzero(~tie)[0]:
                for k in KEYS:
                    g, w = outs[q][k][r], want[q][k][r]
                    assert g.tobytes() == w.tobytes(), (what, q, int(r), k)
    assert compared >= 6 * LF.RANDOM_SEEDS // 2, compared


def _tandem(schedule_a=None, schedule_b=None):
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=2, service_time=hs.ExponentialLatency(0.015), downstream=sink)
    sa = hs.Server("A.server", service_time=hs.ExponentialLatency(0.01), downstream=sb)
    src = hs.Source.poisson(rate=40.0, target=sa, name="A.src")
    ticks = hs.Counter("B.ticks")
    tick = hs.Source.constant(rate=100.0, target=ticks, name="B.tick")      # B's own events end its windows on time
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src], fault_schedule=schedule_a),
             hs.SimulationPartition("B", entities=[sb, sink, ticks], sources=[tick], fault_schedule=schedule_b)]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=hs.ConstantLatency(0.05))
    return parts, link, (src, sa, sb, sink)


def test_parallel_simulation_run_writes_back_onto_the_scripts_objects():
    fa, fb = hs.FaultSchedule(), hs.FaultSchedule()
    fa.add(hs.CrashNode("A.server", at=1.0, restart_at=1.5))
    h = fa.add(hs.PauseNode("A.server", start=2.0, end=2.5))
    fb.add(hs.CrashNode("B.sink", at=2.8))
    parts, link, (src, sa, sb, sink) = _tandem(fa, fb)
    ps = hs.ParallelSimulation(parts, duration=4.0, links=[link], seed=9)
    h.cancel()
    s = ps.run()
    outs = ps.last_outputs
    assert s.partitions["A"].events_cancelled == 2 and s.partitions["B"].events_cancelled == 0
    assert sink._crashed is True and sa._crashed is False
    st_b = outs[1]["entity_stats"][0]
    assert sink.events_received == int(st_b[lm_index(ps, 1, "B.sink")]["c0"]) > 0
    assert sb._requests_completed == int(st_b[lm_index(ps, 1, "B.server")]["c2"]) > 0
    assert s.total_events_processed == sum(int(o["summaries"]["events_processed"][0]) for o in outs)
    assert ps.fault_ties == 0 and s.partitions["B"].entities


def lm_index(ps, q, name):
    return ps._linked.models[q].names.index(name)


def test_run_ensemble_reads_a_cancellation_made_after_construction():
    fa = hs.FaultSchedule()
    h = fa.add(hs.CrashNode("A.server", at=0.5, restart_at=1.5))
    parts, link, _ = _tandem(fa)
    ps = hs.ParallelSimulation(parts, duration=2.0, links=[link], seed=4)
    before, *_ = ps.run_ensemble(64)
    h.cancel()
    after, *_ = ps.run_ensemble(64)
    fr = ps._linked.models[0].ids_of(A.HS_ENT_FAULT)
    assert (before["A"]["entity_stats"][:, fr]["c0"] == 1).all() and (before["A"]["entity_stats"][:, fr]["c1"] == 0).all()
    assert (after["A"]["entity_stats"][:, fr]["c0"] == 0).all() and (after["A"]["entity_stats"][:, fr]["c1"] == 1).all()


def test_a_fault_partition_runs_linked_only_when_uploaded_as_a_partition():
    """hs_model_upload checks a model on its own: it refuses FAULT rows next to REMOTE rows, and a receiving
    partition with FAULT rows that came through it does not run as a linked window"""
    lm, kw, z = G.load_linked("lfault_tandem_crash_downstream")
    e = engine.Engine(0)
    try:
        e.upload(lm.models[1])                           # B: an inbox and FAULT rows, no REMOTE row
        with pytest.raises(Exception, match="hs_partition_upload"):
            e.run(engine.make_params(seed=1, end_ns=10**9, n_replicas=4, engine=3, flags=A.HS_RUN_LINKED))
        lm2, _, _ = G.load_linked("lfault_sender_crash_drains")
        with pytest.raises(Exception, match="hs_partition_upload"):
            e.upload(lm2.models[0])                      # A: REMOTE and FAULT rows
        e.upload(lm2.models[0], partition=True)
    finally:
        e.close()


def test_the_warp_engine_still_refuses_linked_models():
    lm, kw, z = G.load_linked("lfault_tandem_crash_downstream")
    e = engine.Engine(0)
    try:
        e.upload(lm.models[1], partition=True)
        with pytest.raises(Exception, match=r"linked partitions run on the thread engine \(engine 3\)"):
            e.run(engine.make_params(seed=1, end_ns=10**9, n_replicas=4, engine=1, flags=A.HS_RUN_LINKED))
    finally:
        e.close()
