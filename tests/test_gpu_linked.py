"""SURVEY 8(f) row 4, first half on the device: partitions joined by PartitionLinks -- one engine per partition,
hs_run per window (HS_RUN_LINKED), hs_coordinator_exchange at every barrier -- against the fixtures produced by the
unmodified reference's ParallelSimulation / WindowedCoordinator and, for ensembles, against the oracle."""
import numpy as np
import pytest

import golden_lib as G
import oracle_lib as O
from happysim_b200 import _abi as A, engine
from happysim_b200.linked import LinkedRun
from test_gpu_lane_parity import assert_same

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", G.case_names("linked_"))
def test_linked_fixture_on_the_device(name):
    lm, kw, z = G.load_linked(name)
    run = LinkedRun(lm)
    try:
        outs, (delivered, lost, over) = run.run(seed=kw["seed"], end_ns=kw["end_ns"],
                                                caps=[G.linked_caps(z, q) for q in range(lm.n_partitions)])
    finally:
        run.close()
    assert run.windows == int(z["total_windows"]) and int(over[0]) == 0
    if name == "linked_aligned_ring":
        # a few delivered events tie with a local one on time AND sort index (indices of two partitions' counters): the
        # reference orders such a pair by the accident of heapq's array layout; the device says so instead of guessing
        st = [int(o["summaries"]["status"][0]) for o in outs]
        assert any(x & A.HS_ST_LINK_TIE for x in st) and not any(x & ~A.HS_ST_LINK_TIE for x in st)
        return
    assert int(delivered[0]) == int(z["cross_events"])
    for q in range(lm.n_partitions):
        G.check_linked_partition(z, q, outs[q])


@pytest.mark.parametrize("name", ["linked_lossy_fanout", "linked_aligned_ring_spread"])
def test_linked_ensemble_matches_the_oracle(name):
    lm, kw, z = G.load_linked(name)
    nP, n = lm.n_partitions, 41
    caps = [dict(record_cap=6000, sample_cap=600, service_cap=1200) for _ in range(nP)]
    run = LinkedRun(lm)
    try:
        outs, (delivered, lost, over) = run.run(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=n, replica_index_base=3, caps=caps)
    finally:
        run.close()
    ps = [O.make_params(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=n, rid_base=q, rid_stride=nP + 1,
                        replica_index_base=3, **caps[q]) for q in range(nP)]
    want, wd, wl, _ = O.oracle_run_linked(lm, ps, end_ns=kw["end_ns"], cseed=kw["seed"])
    assert np.array_equal(delivered, wd) and np.array_equal(lost, wl) and not over.any()
    for q in range(nP):
        assert_same(outs[q], want[q])
        if want[q].get("sketches") is not None:
            assert outs[q]["sketches"].tobytes() == want[q]["sketches"].tobytes()
    assert len({int(x) for x in outs[0]["summaries"]["order_hash"]}) == (1 if name == "linked_aligned_ring_spread" else n)


def test_outbox_and_inbox_between_windows():
    """After the first window and before its barrier the sender's outbox holds what its servers forwarded; the
    barrier moves it, delayed by the link latency, into the receiver's inbox; the next window schedules it."""
    lm, kw, z = G.load_linked("linked_tandem_const")
    run = LinkedRun(lm)
    try:
        a, b = run.engines
        ends = lm.window_ends(kw["end_ns"])
        mk = lambda q, w: engine.make_params(seed=kw["seed"], end_ns=ends[w], rid_base=q, rid_stride=3, engine=3,
                                             resume=1 if w else 0, flags=A.HS_RUN_ORDER_HASH | A.HS_RUN_LINKED)
        coord = engine.Coordinator(0, 1, 1, seed=kw["seed"], rid_base=2, rid_stride=3)
        sent_total = 0
        for w in range(6):
            a.run(mk(0, w)); b.run(mk(1, w))
            box, cnt = a.read_box("outbox")
            inbox_before = int(b.read_box("inbox")[1][0])
            assert inbox_before == 0                                   # drained by the run that just ended
            arr, dst = lm.link_descs(0)
            coord.exchange(a, arr, [b])
            ib, icnt = b.read_box("inbox")
            assert int(a.read_box("outbox")[1][0]) == 0 and int(icnt[0]) == int(cnt[0])
            k = int(cnt[0])
            assert np.array_equal(ib[0][:k]["time_ns"], box[0][:k]["time_ns"] + 50_000_000)
            assert np.array_equal(ib[0][:k]["sort_index"], box[0][:k]["sort_index"]) and (ib[0][:k]["ent"] == 0).all()
            assert (box[0][:k]["ent"] == 2).all() and (np.diff(box[0][:k]["time_ns"]) >= 0).all()
            sent_total += k
        assert sent_total > 5 and int(coord.read()[0][0]) == sent_total
        coord.close()
    finally:
        run.close()


def test_linked_models_need_the_thread_engine_and_an_outbox():
    lm, kw, z = G.load_linked("linked_tandem_const")
    e = engine.Engine(0)
    try:
        e.upload(lm.models[0])
        with pytest.raises(engine.EngineError, match="thread engine"):
            e.run(engine.make_params(seed=1, end_ns=10**8, engine=1))
        m = lm.models[0]
        m.outbox_cap = 0
        with pytest.raises(engine.EngineError, match="outbox_cap"):
            e.upload(m)
        # a link destination shaped like the lane engine's model: the lane kernel has no inbox, so the thread engine
        # runs it -- refused when asked for explicitly, chosen by auto selection (a window of it resumes on engine 3)
        import happysim_b200 as hs
        m = hs.mm1()
        m.inbox_cap = 16
        e.upload(m)
        with pytest.raises(engine.EngineError, match="thread engine"):
            e.run(engine.make_params(seed=1, end_ns=10**10, engine=2))
        e.run(engine.make_params(seed=1, end_ns=10**10, window_end_ns=5 * 10**9, engine=0))
        e.run(engine.make_params(seed=1, end_ns=10**10, resume=1, engine=3))
        s = e.read_outputs()["summaries"]
        assert int(s["status"][0]) == 0 and int(s["events_processed"][0]) > 0
    finally:
        e.close()


def test_api_parallel_simulation_with_a_link_equals_the_reference_fixture():
    """hs.ParallelSimulation(partitions, links=[...]).run(): the numbers the unmodified reference's ParallelSimulation
    produced for the same declaration (fixture linked_tandem_const), on the script's own objects."""
    import happysim_b200 as hs
    from test_parallel_linked import tandem
    parts, link, (src, sa, sb, sink) = tandem()
    ps = hs.ParallelSimulation(parts, duration=4.0, links=[link], seed=5)
    summ = ps.run()
    lm, kw, z = G.load_linked("linked_tandem_const")
    assert summ.total_windows == int(z["total_windows"]) and summ.total_cross_partition_events == int(z["cross_events"])
    assert summ.total_events_processed == int(z["total_events"]) and summ.window_size_s == 0.05
    assert [s.total_events_processed for s in summ.partitions.values()] == [int(z[f"p{q}_summaries"]["events_processed"][0]) for q in range(2)]
    assert sink.latencies_s == [float(x) for x in z["p1_sink_samples"]["latency_s"]]
    assert [t.nanoseconds for t in sink.completion_times] == [int(x) for x in z["p1_sink_samples"]["completion_ns"]]
    assert sa.stats.requests_completed == int(z["p0_entity_stats"][0][1]["c2"]) > 100
    assert sb.stats.requests_completed == int(z["p1_entity_stats"][0][0]["c2"]) > 100
    assert src.generated_count == int(z["p0_entity_stats"][0][0]["c0"]) and ps.link_ties == 0
    assert set(summ.entities) >= {"A.server", "B.server", "B.sink"}
    ens, delivered, lost = ps.run_ensemble(24)
    assert int(delivered[0]) == int(z["cross_events"]) and not lost.any() and len(set(int(x) for x in delivered)) > 3
    assert int(ens["B"]["summaries"]["events_processed"][0]) == int(z["p1_summaries"]["events_processed"][0])


def test_api_tandem_heavy_equals_the_reference_fixture():
    """The 500 req/s tandem (fixture linked_tandem_heavy, ~5 000 Sink samples in B) through hs.ParallelSimulation on
    the device: the unmodified reference's lists, in full, on the script's own objects."""
    import test_linked_volume as V
    ps, parts = V.build("tandem_heavy")
    summ = ps.run()
    lm, kw, z = G.load_linked("linked_tandem_heavy")
    (sa,), (sb, sink) = parts[0].entities, parts[1].entities
    assert summ.total_windows == int(z["total_windows"]) and summ.total_cross_partition_events == int(z["cross_events"])
    assert [s.total_events_processed for s in summ.partitions.values()] == [int(z[f"p{q}_summaries"]["events_processed"][0]) for q in range(2)]
    assert len(sink.latencies_s) == len(z["p1_sink_samples"]) > 4000
    assert sink.latencies_s == [float(x) for x in z["p1_sink_samples"]["latency_s"]]
    assert [t.nanoseconds for t in sink.completion_times] == [int(x) for x in z["p1_sink_samples"]["completion_ns"]]
    assert sb._service_times == [float(x) for x in z["p1_service_samples"]]
    assert sa._service_times == [float(x) for x in z["p0_service_samples"]]
    assert sink.events_received == int(z["p1_entity_stats"][0][1]["c0"]) and ps.link_ties == 0


@pytest.mark.parametrize("name", ["tandem_heavy", "fan_in", "two_sinks", "chain", "profile_source"])
def test_linked_volume_cases_on_the_device(name):
    """The volume cases of tests/test_linked_volume.py through the real LinkedRun: the thread engine's linked runs with
    inboxes of tens to hundreds of events per window and recorder rings of thousands of items publish exactly the
    unwrapped oracle run."""
    import test_linked_volume as V
    ps, _ = V.build(name)
    summ = ps.run()
    want, delivered, lost, ends = V.truth(ps._linked, seed=ps._seed, end_ns=ps._end_ns)
    assert ps.link_ties == 0 and np.array_equal(ps.last_delivered, delivered) and np.array_equal(ps.last_lost, lost)
    V.check_published(ps, summ, want, delivered, ends)


def test_linked_volume_ensemble_on_the_device():
    """run_ensemble(16) of the 500 req/s tandem: every replica's rings, unrolled, equal its unwrapped oracle run."""
    import test_linked_volume as V
    ps, _ = V.build("tandem_heavy")
    n = 16
    ens, delivered, lost = ps.run_ensemble(n)
    want, wd, wl, _ = V.truth(ps._linked, seed=ps._seed, end_ns=ps._end_ns, n_replicas=n)
    assert np.array_equal(delivered, wd) and np.array_equal(lost, wl)
    V.check_ensemble(ps._linked, ens, want, n)


def test_random_linked_models_on_the_device():
    """The 72 random linked ParallelSimulations (tests/random_models.random_linked_model; oracle == reference on all of
    them, tests/test_random_linked.py): 6 replicas each on the device against the oracle.  A replica in which a delivered
    event tied with another on time AND index is flagged (HS_ST_LINK_TIE; only the grid models can) and is left out."""
    import random_models as RM
    flagged = compared = 0
    for seed in range(RM.LINKED_SEEDS):
        lm, end_s, what = RM.random_linked_model(seed)
        end_ns, nP, n = int(end_s * 1e9), lm.n_partitions, 6
        caps = [dict(record_cap=512, sample_cap=64, service_cap=64) for _ in range(nP)]
        run = LinkedRun(lm)
        try:
            # queue_ring: the reference's queues are unbounded; some of the random models run overloaded for a while
            outs, (delivered, lost, over) = run.run(seed=1000 + seed, end_ns=end_ns, n_replicas=n, caps=caps, queue_ring=2048)
        finally:
            run.close()
        ps = [O.make_params(seed=1000 + seed, end_ns=end_ns, n_replicas=n, rid_base=q, rid_stride=nP + 1, **caps[q]) for q in range(nP)]
        want, wd, wl, _ = O.oracle_run_linked(lm, ps, end_ns=end_ns, cseed=1000 + seed)
        assert not over.any(), what
        tie = np.zeros(n, bool)
        for o in outs:
            tie |= (o["summaries"]["status"] & A.HS_ST_LINK_TIE) != 0
        assert "grid" in what or not tie.any(), what
        flagged += int(tie.sum())
        for r in np.nonzero(~tie)[0]:
            compared += 1
            assert (int(delivered[r]), int(lost[r])) == (int(wd[r]), int(wl[r])), (what, r)
            for q in range(nP):
                g, w = outs[q]["summaries"][r], want[q]["summaries"][r]
                for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
                    assert int(g[f]) == int(w[f]), (what, q, int(r), f, int(g[f]), int(w[f]))
                assert int(g["status"]) & ~A.HS_ST_LINK_TIE == int(w["status"]), (what, q, int(r))
                assert outs[q]["entity_stats"][r].tobytes() == want[q]["entity_stats"][r].tobytes(), (what, q, int(r))
                assert outs[q]["records"][r].tobytes() == want[q]["records"][r].tobytes(), (what, q, int(r))
                if want[q].get("sketches") is not None:
                    assert outs[q]["sketches"][r].tobytes() == want[q]["sketches"][r].tobytes(), (what, q, int(r))
    assert compared > 300 and flagged < 120, (compared, flagged)
