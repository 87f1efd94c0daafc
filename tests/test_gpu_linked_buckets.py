"""Time buckets and their p50 / p99 in the partitions of a linked run, on the device: the thread engine's sixteen
LINKED bucket instantiations (HASH x HEAPTOP x FAULTS, with and without percentiles) against the samples of a
record-mode LinkedRun of the same seeds, bucketed on the host; records that do not change with percentiles; per-cell
totals; the records after every window; sample-capacity growth; the refusals; ParallelSimulation.run_ensemble with
trackers and a Probe against Data.bucket of what ParallelSimulation.run() writes back; and run_ensemble on the mirror
scripts of the reference fixtures (tests/golden/lbucket_*.npz) against the reference's own Data.bucket lists on
replica 0 and the oracle on all 41 replicas."""
import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import linked_fault_models as LF
from happysim_b200 import _abi as A, buckets as B, engine, results
from happysim_b200.instrumentation import _percentile_sorted
from happysim_b200.linked import LinkedModel, LinkedRun, LinkSpec

pytestmark = pytest.mark.gpu

WF_HASH, WF_PROFILE, WF_HEAPTOP, WF_LINKED, WF_FAULTS, WF_BUCKETS, WF_BUCKET_PCT = 1, 4, 8, 16, 32, 64, 128
CAP = 256


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def _tandem(a_sink=True, faults=False):
    """A: Source(80/s) -> Server -> [50 ms link] -> B.s1 and, with ``a_sink``, Source(25/s) -> Server -> A.sink.
    B: s1 (c=2) -> B.lat, a depth Probe on s1 every 0.1 s, and Source(20/s) -> s2 -> B.tp.  With ``faults`` a crash and
    a pause on each side; B's faults hit its servers only: a request a crashed Sink drops still has its event record,
    and results.demultiplex would credit the next sample to it."""
    a = hs.ModelBuilder()
    src = a.source("A.src", rate=80.0)
    s1 = a.server("A.s1", mean_service_s=0.008)
    rem = a.remote("B.s1@A", link=0, dest_entity=0)
    a.set_target(src, s1); a.set_target(s1, rem)
    if a_sink:
        s2 = a.server("A.s2", mean_service_s=0.02)
        a.set_target(a.source("A.src2", rate=25.0), s2); a.set_target(s2, a.sink("A.sink"))
    ma = a.build(); ma.outbox_cap = 256
    b = hs.ModelBuilder()
    bs1 = b.server("B.s1", concurrency=2, mean_service_s=0.015)
    b.set_target(bs1, b.sink("B.lat"))
    b.probe("B.probe", target=bs1, metric="depth", interval_s=0.1)
    bs2 = b.server("B.s2", mean_service_s=0.03)
    b.set_target(b.source("B.src", rate=20.0), bs2); b.set_target(bs2, b.sink("B.tp"))
    mb = b.build(); mb.inbox_cap = 256
    assert mb.names[0] == "B.s1"
    lm = LinkedModel([ma, mb], ["A", "B"], [[LinkSpec(1, A.HS_SVC_EXPONENTIAL, 0.05, 0.0, 0)], []], window_s=0.05)
    if not faults:
        return lm
    return LF.linked_with_faults(lm, [[("crash", "A.s1", 0.7, 1.1, False), ("pause", "A.sink" if a_sink else "A.s1", 1.6, 1.9, False)],
                                      [("crash", "B.s1", 0.4, 0.9, False), ("pause", "B.s2", 1.2, 1.5, False)]])


def _bucket_run(lm, n, seed, end_ns, w, nb, cap, flags):
    """(outputs, last launch of every partition) of a bucketed LinkedRun"""
    run = LinkedRun(lm)
    try:
        outs, counts = run.run(seed=seed, end_ns=end_ns, n_replicas=n, flags=flags, buckets=(w, nb), bucket_sample_cap=cap)
        infos = [e.last_launch() for e in run.engines]
    finally:
        run.close()
    assert not counts[2].any()
    return outs, infos


def _record_run(lm, n, seed, end_ns, flags, cap=4096):
    run = LinkedRun(lm)
    try:
        outs, _ = run.run(seed=seed, end_ns=end_ns, n_replicas=n, flags=flags,
                          caps=dict(record_cap=4 * cap, sample_cap=cap, service_cap=cap))
    finally:
        run.close()
    for o in outs:
        assert (o["summaries"]["n_sink_samples"] <= cap).all() and (o["summaries"]["events_processed"] <= 4 * cap).all()
    return outs


def _check_records(model, rec, got, past, pct, w, nb, replicas):
    """the records (and percentiles) of every replica in ``replicas`` against its record-mode samples"""
    rows = B.rows(model)
    for r in replicas:
        per_sink, _ = results.demultiplex(model, rec, r)
        for b, ent in enumerate(rows):
            sm = per_sink[ent]
            t = np.asarray(sm["completion_ns"] if sm is not None else [], np.int64)
            v = np.asarray(sm["latency_s"] if sm is not None else [], np.float64)
            k = B.bucket_index(t, w)
            slot = np.minimum(k, nb)
            g = got[r, b]
            assert (np.bincount(slot, minlength=nb + 1) == g["count"]).all(), (r, b)
            sums = B.replica_sums(g)
            cuts = np.flatnonzero(np.diff(slot)) + 1             # a row's samples come in time order
            for ks, vs in zip(np.split(slot, cuts), np.split(v, cuts)):
                if not len(ks):
                    continue
                s, vals = int(ks[0]), [float(x) for x in vs]
                assert _bits(sums[s]) == _bits(sum(vals)) and _bits(g["max"][s]) == _bits(max(vals)), (r, b, s)
                if s == nb:
                    assert int(past[r, b]) == int(k[-1]), (r, b)
                if pct is not None:
                    srt = sorted(vals)
                    want = [_percentile_sorted(srt, 0.50), _percentile_sorted(srt, 0.99)]
                    assert _bits(pct[r, b, s]).tolist() == _bits(want).tolist(), (r, b, s)


@pytest.mark.parametrize("faults", [0, 1])
@pytest.mark.parametrize("hash_", [0, 1])
@pytest.mark.parametrize("n", [2048, 16384])
def test_linked_bucket_kernels_match_record_mode(n, hash_, faults):
    """each of the sixteen LINKED bucket kernels (this parametrization x percentiles on / off) is the one that ran, and
    its records equal those derived from a record-mode run of the same seeds; without percentiles the records, past-end
    indices and totals are the same bytes; the sinkless partition keeps its kernel without buckets"""
    lm = _tandem(a_sink=False, faults=bool(faults))
    seed, end_ns, w, nb = 17, int(2.5e9), 0.1, 26
    outs, infos = _bucket_run(lm, n, seed, end_ns, w, nb, CAP, hash_)
    plain, infos0 = _bucket_run(lm, n, seed, end_ns, w, nb, 0, hash_)
    rec = _record_run(lm, n, seed, end_ns, hash_)
    fl = WF_BUCKETS | WF_PROFILE | WF_LINKED | hash_ | (WF_FAULTS if faults else 0) | (WF_HEAPTOP if n == 16384 else 0)
    assert infos[1]["engine"] == 3 and infos[1]["kernel"] == "thread", infos[1]
    assert infos[1]["flags"] == fl | WF_BUCKET_PCT and infos0[1]["flags"] == fl, (infos[1], infos0[1])
    assert not infos[0]["flags"] & WF_BUCKETS and "buckets" not in outs[0], infos[0]        # A has no bucketed row
    assert infos[0]["flags"] == infos0[0]["flags"]
    o, p = outs[1], plain[1]
    for k in ("buckets", "bucket_past_end", "bucket_totals"):
        assert o[k].tobytes() == p[k].tobytes(), k
    assert "bucket_percentiles" not in p and o["bucket_sample_cap"] == CAP
    for q in range(2):
        s, ws = outs[q]["summaries"], rec[q]["summaries"]
        assert (s["events_processed"] == ws["events_processed"]).all() and (s["order_hash"] == ws["order_hash"]).all(), q
        assert (s["n_sink_samples"] == ws["n_sink_samples"]).all() and not (s["status"] & ~np.uint32(A.HS_ST_LINK_TIE)).any(), q
    assert int(o["buckets"]["count"].sum()) == int(rec[1]["summaries"]["n_sink_samples"].sum())
    assert o["bucket_totals"].tobytes() == B.cell_totals_reference(o["buckets"], 1).tobytes()
    assert o["bucket_percentile_totals"].tobytes() == \
        B.cell_percentile_totals_reference(o["buckets"], o["bucket_percentiles"], 1).tobytes()
    reps = range(n) if n <= 2048 else range(0, n, 61)
    _check_records(lm.models[1], rec[1], o["buckets"], o["bucket_past_end"], o["bucket_percentiles"], w, nb, reps)


def test_records_after_every_window():
    """after each window the records of every bucketed partition count the partition's Sink and Probe samples so far
    (the accumulators are stored at each window end), and the final records equal LinkedRun's"""
    lm = _tandem(a_sink=True)
    seed, end_ns, w, nb, n = 3, int(1.2e9), 0.25, 5, 64
    run = LinkedRun(lm)
    try:
        nP = lm.n_partitions
        coord = engine.Coordinator(0, n, lm.n_streams, seed=seed, rid_base=nP, rid_stride=nP + 1, stream=run._stream_ptr)
        for e in run.engines:
            e.set_buckets(w, nb)
            e.set_bucket_percentiles(CAP)
        ends = lm.window_ends(end_ns)
        for k, wend in enumerate(ends):
            for q, e in enumerate(run.engines):
                e.run(engine.make_params(seed=seed, end_ns=wend, n_replicas=n, rid_base=q, rid_stride=nP + 1, engine=3,
                                         resume=1 if k else 0, flags=A.HS_RUN_LINKED))
            arr, dst = lm.link_descs(0)
            coord.exchange(run.engines[0], arr, [run.engines[d] for d in dst])
            for q, e in enumerate(run.engines):
                got, _ = e.read_buckets(nb)
                smp = e.read_outputs()["summaries"]["n_sink_samples"]
                assert (got["count"].sum(axis=(1, 2)) == smp).all(), (k, q)
        last = [e.read_buckets(nb)[0] for e in run.engines]
        coord.close()
        for e in run.engines:
            e.set_bucket_percentiles(0)
            e.set_buckets(0.0, 0)
    finally:
        run.close()
    outs, _ = _bucket_run(lm, n, seed, end_ns, w, nb, CAP, 0)
    for q in range(2):
        assert outs[q]["buckets"].tobytes() == last[q].tobytes(), q


# ---- the refusals -----------------------------------------------------------------------------------------------

def test_refusals():
    lm = _tandem()
    e = engine.Engine(0)
    try:
        e.upload(lm.models[1], partition=True)
        e.set_buckets(0.5, 8)
        with pytest.raises(engine.EngineError, match="recorder rings"):
            e.run(engine.make_params(seed=1, end_ns=10**9, n_replicas=4, engine=3, sample_cap=64, flags=A.HS_RUN_LINKED))
        e.run(engine.make_params(seed=1, end_ns=10**9, n_replicas=4, engine=3, flags=A.HS_RUN_LINKED))
        assert e.last_launch()["flags"] & (WF_BUCKETS | WF_LINKED) == WF_BUCKETS | WF_LINKED
        e.upload(lm.models[1])                              # not a partition upload
        with pytest.raises(engine.EngineError, match="linked"):
            e.run(engine.make_params(seed=1, end_ns=10**9, n_replicas=4, engine=3, flags=A.HS_RUN_LINKED))
    finally:
        e.set_buckets(0.0, 0)
        e.close()


# ---- ParallelSimulation ------------------------------------------------------------------------------------------

def _mirror(faults=False):
    """A: Source -> Server -> [link] -> B.s1 -> LatencyTracker, and Source -> Server -> A.sink.  B: a depth Probe on s1,
    Source -> s2 -> ThroughputTracker.  With ``faults`` a crash and a pause in A."""
    lat, tp = hs.LatencyTracker("B.lat"), hs.ThroughputTracker("B.tp")
    b1 = hs.Server("B.s1", concurrency=2, service_time=hs.ExponentialLatency(0.015), downstream=lat)
    b2 = hs.Server("B.s2", service_time=hs.ExponentialLatency(0.03), downstream=tp)
    probe, data = hs.Probe.on(b1, "depth", interval=0.1)
    bsrc = hs.Source.poisson(rate=20.0, target=b2, name="B.src")
    asink = hs.Sink("A.sink")
    a1 = hs.Server("A.s1", service_time=hs.ExponentialLatency(0.008), downstream=b1)
    a2 = hs.Server("A.s2", service_time=hs.ExponentialLatency(0.02), downstream=asink)
    srcs = [hs.Source.poisson(rate=80.0, target=a1, name="A.src"), hs.Source.poisson(rate=25.0, target=a2, name="A.src2")]
    fs = None
    if faults:
        fs = hs.FaultSchedule()
        fs.add(hs.CrashNode("A.s1", at=0.7, restart_at=1.1))
        fs.add(hs.PauseNode("A.sink", start=1.6, end=1.9))
    parts = [hs.SimulationPartition("A", entities=[a1, a2, asink], sources=srcs, fault_schedule=fs),
             hs.SimulationPartition("B", entities=[b1, b2, lat, tp], sources=[bsrc], probes=[probe])]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=hs.ConstantLatency(0.05))
    ps = hs.ParallelSimulation(parts, duration=3.0, links=[link], seed=9)
    return ps, {"A": [asink], "B": [lat, tp, probe, data]}


@pytest.mark.parametrize("faults", [False, True])
def test_run_ensemble_matches_data_bucket_of_run(faults):
    """bucketed_data of every Sink, tracker and Probe of replica 0 equals Data.bucket(w) of what run() writes back onto
    the script's objects, bit for bit; every replica's records equal a record-mode LinkedRun's"""
    w, nb, n = 0.25, 13, 41
    ps, objs = _mirror(faults)
    outs, delivered, lost = ps.run_ensemble(n, buckets=(w, nb), bucket_percentiles=True)
    for name, o in outs.items():
        assert o["bucket_count"] == nb and o["bucket_width_s"] == w and o["bucket_totals"].shape[0] == 1
        assert len(o["bucket_objects"]) == len(o["bucket_rows"]) == o["buckets"].shape[1]
    ps2, objs2 = _mirror(faults)
    ps2.run()
    for name in objs:
        for obj, obj2 in zip(objs[name], objs2[name]):
            if isinstance(obj2, hs.Sink):                       # a Sink keeps its samples in two lists
                src = hs.Data()
                src._samples = [(float(int(t.nanoseconds)) / 1_000_000_000, v) for t, v in zip(obj2.completion_times, obj2.latencies_s)]
            else:
                src = obj2 if isinstance(obj2, hs.Data) else obj2.data_sink if hasattr(obj2, "data_sink") else obj2.data
            want = src.bucket(w)
            got = B.bucketed_data(outs[name], obj, 0)
            for f in ("times", "counts", "sums", "means", "maxes"):
                assert getattr(got, f)() == getattr(want, f)(), (name, f, obj)
            assert _bits(got.p50s()).tolist() == _bits(want.p50s()).tolist(), (name, obj)
            assert _bits(got.p99s()).tolist() == _bits(want.p99s()).tolist(), (name, obj)
    lm = ps._linked
    rec = _record_run(lm, n, ps._seed, ps._end_ns, 0)
    for q, name in enumerate(lm.names):
        o = outs[name]
        _check_records(lm.models[q], rec[q], o["buckets"], o["bucket_past_end"], o["bucket_percentiles"], w, nb, range(n))


def test_sample_cap_grows():
    """a too-small bucket_sample_cap is grown and gives the bytes of a run started with the larger capacity"""
    w, nb = 1.0, 4
    ps, _ = _mirror()
    outs, _, _ = ps.run_ensemble(64, buckets=(w, nb), bucket_percentiles=True, bucket_sample_cap=2)
    cap = outs["B"]["bucket_sample_cap"]
    assert cap > 2 and cap == max(B.sample_cap_needed(o["buckets"]) for o in outs.values())
    ps2, _ = _mirror()
    again, _, _ = ps2.run_ensemble(64, buckets=(w, nb), bucket_percentiles=True, bucket_sample_cap=cap)
    for name in outs:
        for k in ("buckets", "bucket_past_end", "bucket_percentiles", "bucket_percentile_totals", "bucket_totals"):
            assert outs[name][k].tobytes() == again[name][k].tobytes(), (name, k)
        assert not (outs[name]["summaries"]["status"] & A.HS_ST_BUCKET_OVERFLOW).any()


def test_tandem_heavy_100s_at_16384_replicas():
    """tandem_heavy (500 req/s) for 100 s at 16 384 replicas with 1 000 buckets and percentiles: the recorder rings of
    this run would need about 5 MB per partition-replica.  Bucket counts equal the Sink's sample counts, and 8 replicas
    re-run in record mode at their own replica_index_base give the same records."""
    lm, kw, z = G.load_linked("linked_tandem_heavy")
    n, end_ns, w, nb = 16384, 100 * 10**9, 0.1, 1001
    outs, infos = _bucket_run(lm, n, kw["seed"], end_ns, w, nb, 128, 0)
    o = outs[1]
    assert infos[1]["flags"] == WF_BUCKETS | WF_BUCKET_PCT | WF_PROFILE | WF_LINKED | WF_HEAPTOP, infos[1]
    for q in range(2):
        assert not (outs[q]["summaries"]["status"] & ~np.uint32(A.HS_ST_LINK_TIE)).any(), q
    sink = lm.models[1].ids_of(A.HS_ENT_SINK)[0]
    assert (o["buckets"]["count"].sum(axis=(1, 2)) == outs[1]["entity_stats"][:, sink]["c0"]).all()
    assert int(o["buckets"]["count"].sum()) > n * 45000
    for base in (0, 8191, 16376):
        run = LinkedRun(lm)
        try:
            rec, _ = run.run(seed=kw["seed"], end_ns=end_ns, n_replicas=8, replica_index_base=base, flags=0,
                             caps=dict(record_cap=0, sample_cap=65536, service_cap=65536))
        finally:
            run.close()
        sub = o["buckets"][base:base + 8]
        _check_records(lm.models[1], rec[1], sub, o["bucket_past_end"][base:base + 8],
                       o["bucket_percentiles"][base:base + 8], w, nb, range(8))


# ---- the reference fixtures (tests/golden/gen_linked_bucket_golden.py) ----------------------------------------------

import linked_bucket_models as LB  # noqa: E402
import layered_oracle_lib as LO  # noqa: E402
import oracle_lib as O  # noqa: E402


@pytest.mark.parametrize("name", list(LB.CASES))
def test_run_ensemble_equals_the_reference_and_the_oracle(name):
    """ParallelSimulation.run_ensemble(41, buckets=, bucket_percentiles=True) of the mirror script: bucketed_data of every
    tracker, Sink and Probe equals the reference's own Data.bucket lists on replica 0 (counts exact, floats bitwise), and
    every replica's records, past-end indices and percentiles equal the oracle's samples of the same seeds, bucketed on
    the host"""
    lm, kw, z = LB.load(name)
    n = 41
    ps = LB.CASES[name][0]()
    outs, delivered, lost = ps.run_ensemble(n, buckets=(LB.W, LB.NB), bucket_percentiles=True)
    nP = lm.n_partitions
    params = [O.make_params(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=n, rid_base=q, rid_stride=nP + 1,
                            record_cap=8192, sample_cap=4096, service_cap=4096) for q in range(nP)]
    run = LO.run_linked if any(m.ids_of(A.HS_ENT_FAULT) for m in lm.models) else O.oracle_run_linked
    want, wd, wl, _ = run(lm, params, end_ns=kw["end_ns"], cseed=kw["seed"])
    assert (delivered == wd).all() and (lost == wl).all()
    rows = 0
    for q, pname in enumerate(lm.names):
        o = outs[pname]
        if not B.rows(lm.models[q]):
            assert "buckets" not in o
            continue
        assert (o["summaries"]["events_processed"] == want[q]["summaries"]["events_processed"]).all(), q
        for b, obj in enumerate(o["bucket_objects"]):
            assert LB.same(LB.lists(B.bucketed_data(o, obj, 0)), LB.fixture_lists(z, q, b)), (q, b)
            rows += 1
        host = LB.host_out(lm.models[q], ps._linked.objects[q], want[q], range(n))
        g, h = o["buckets"], host["buckets"]
        assert (g["count"] == h["count"]).all(), q
        has = g["count"] > 0
        assert (_bits(B.replica_sums(g))[has] == _bits(h["sum"])[has]).all() and (_bits(g["max"])[has] == _bits(h["max"])[has]).all(), q
        assert (_bits(o["bucket_percentiles"])[has] == _bits(host["bucket_percentiles"])[has]).all(), q
        late = has[:, :, LB.NB]
        assert (o["bucket_past_end"][late] == host["bucket_past_end"][late]).all(), q
    assert rows == (3 if name == "lbucket_three_way" else 4)
