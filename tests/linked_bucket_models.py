"""Linked ParallelSimulations whose partitions feed LatencyTrackers, ThroughputTrackers, Sinks and Probes: the mirror
scripts behind tests/golden/lbucket_*.npz (gen_linked_bucket_golden.py), the fixtures' loader, and the host
restatement of the device's time buckets over a replica's recorded samples.  Test infrastructure.

The fixtures are named lbucket_*, not linked_* / lfault_*: their Probe rows need the partitions' rate-profile tables,
which golden_lib.load_linked (and with it the tests that take every linked_* / lfault_* fixture) does not load."""
from __future__ import annotations

import numpy as np

import happysim_b200 as hs
from happysim_b200 import _abi as A, buckets as B, results
from happysim_b200.instrumentation import _percentile_sorted

W, NB = 0.25, 13                     # 13 buckets of 0.25 s cover the 3 s runs (the end time falls in bucket 12)
FIELDS = ("times", "counts", "means", "sums", "maxes", "p50s", "p99s")


def tracker_tandem(faults=False):
    """A: Source(60/s) -> Server -> [50 ms link] -> B.s1, and Source(25/s) -> Server -> A.sink (a Sink of its own).
    B: s1 (c=2) -> LatencyTracker, a depth Probe on s1 every 0.1 s, Source(20/s) -> s2 -> ThroughputTracker.
    With ``faults`` A's schedule crashes its linked Server and pauses its Sink."""
    lat, tp = hs.LatencyTracker("B.lat"), hs.ThroughputTracker("B.tp")
    b1 = hs.Server("B.s1", concurrency=2, service_time=hs.ExponentialLatency(0.015), downstream=lat)
    b2 = hs.Server("B.s2", service_time=hs.ExponentialLatency(0.03), downstream=tp)
    probe, data = hs.Probe.on(b1, "depth", interval=0.1)
    asink = hs.Sink("A.sink")
    a1 = hs.Server("A.s1", service_time=hs.ExponentialLatency(0.01), downstream=b1)
    a2 = hs.Server("A.s2", service_time=hs.ExponentialLatency(0.02), downstream=asink)
    srcs = [hs.Source.poisson(rate=60.0, target=a1, name="A.src"), hs.Source.poisson(rate=25.0, target=a2, name="A.src2")]
    fs = None
    if faults:
        fs = hs.FaultSchedule()
        for cls, name, t0, t1, _ in SCHEDULES["tracker_tandem_faults"][0]:
            fs.add(hs.CrashNode(name, at=t0, restart_at=t1) if cls == "crash" else hs.PauseNode(name, start=t0, end=t1))
    parts = [hs.SimulationPartition("A", entities=[a1, a2, asink], sources=srcs, fault_schedule=fs),
             hs.SimulationPartition("B", entities=[b1, b2, lat, tp], sources=[hs.Source.poisson(rate=20.0, target=b2, name="B.src")],
                                    probes=[probe])]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=hs.ConstantLatency(0.05))
    return hs.ParallelSimulation(parts, duration=3.0, links=[link], seed=SEEDS["tracker_tandem"])


def three_way():
    """A: Source(50/s) -> Server -> [40 ms link] -> B.s1 -> [exponential 60 ms link] -> C.s1 -> LatencyTracker, with a
    depth Probe on C.s1; B: Source(30/s) -> s2 -> Sink.  A buckets nothing; B and C do."""
    lat = hs.LatencyTracker("C.lat")
    c1 = hs.Server("C.s1", concurrency=2, service_time=hs.ExponentialLatency(0.02), downstream=lat)
    probe, data = hs.Probe.on(c1, "depth", interval=0.2)
    bsink = hs.Sink("B.sink")
    b1 = hs.Server("B.s1", service_time=hs.ExponentialLatency(0.008), downstream=c1)
    b2 = hs.Server("B.s2", service_time=hs.ExponentialLatency(0.025), downstream=bsink)
    a1 = hs.Server("A.s1", service_time=hs.ExponentialLatency(0.01), downstream=b1)
    parts = [hs.SimulationPartition("A", entities=[a1], sources=[hs.Source.poisson(rate=50.0, target=a1, name="A.src")]),
             hs.SimulationPartition("B", entities=[b1, b2, bsink], sources=[hs.Source.poisson(rate=30.0, target=b2, name="B.src")]),
             hs.SimulationPartition("C", entities=[c1, lat], probes=[probe])]
    links = [hs.PartitionLink("A", "B", min_latency=0.04, latency=hs.ConstantLatency(0.04)),
             hs.PartitionLink("B", "C", min_latency=0.04, latency=hs.ExponentialLatency(0.06))]
    return hs.ParallelSimulation(parts, duration=3.0, links=links, seed=SEEDS["three_way"])


SEEDS = {"tracker_tandem": 23, "three_way": 31}
# per partition: (class, entity name, t0_s, t1_s, cancelled), as tests/linked_fault_models.py takes them
SCHEDULES = {"tracker_tandem_faults": [[("crash", "A.s1", 0.7, 1.1, False), ("pause", "A.sink", 1.6, 1.9, False)], []]}
# fixture name -> (mirror script, per-partition schedules or None)
CASES = {"lbucket_tracker_tandem": (lambda: tracker_tandem(), None),
         "lbucket_three_way": (three_way, None),
         "lbucket_tracker_tandem_faults": (lambda: tracker_tandem(faults=True), SCHEDULES["tracker_tandem_faults"])}


def load(name):
    """golden_lib.load_linked of an lbucket_* fixture, with every partition's rate profiles (its Probes' ticks)"""
    import golden_lib as G
    lm, kw, z = G.load_linked(name)
    for q, m in enumerate(lm.models):
        if len(z[f"p{q}_profiles"]):
            m.profiles = z[f"p{q}_profiles"]
        if len(z[f"p{q}_profile_table"]):
            m.profile_table = z[f"p{q}_profile_table"]
    return lm, kw, z


def host_buckets(model, out, r: int, w: float = W, nb: int = NB):
    """The device's bucket records of replica ``r`` restated from its recorded samples (``out``: record-mode outputs of
    one partition): (BUCKET_DTYPE [rows, nb + 1] with sum() in ``sum`` and ``comp`` = 0, past-end indices [rows],
    percentiles [rows, nb + 1, 2])."""
    rows = B.rows(model)
    rec = np.zeros((len(rows), nb + 1), A.BUCKET_DTYPE)
    past = np.zeros(len(rows), np.int64)
    pct = np.zeros((len(rows), nb + 1, 2))
    per_sink, _ = results.demultiplex(model, out, r)
    for b, ent in enumerate(rows):
        sm = per_sink[ent]
        if sm is None or not len(sm):
            continue
        k = B.bucket_index(np.asarray(sm["completion_ns"], np.int64), w)
        for s in np.unique(np.minimum(k, nb)):
            sel = np.minimum(k, nb) == s
            vals = [float(x) for x in np.asarray(sm["latency_s"])[sel]]
            rec[b, s]["count"], rec[b, s]["sum"], rec[b, s]["max"] = len(vals), sum(vals), max(vals)
            srt = sorted(vals)
            pct[b, s] = (_percentile_sorted(srt, 0.50), _percentile_sorted(srt, 0.99))
            if s == nb:
                past[b] = int(k[sel][0])
    return rec, past, pct


def host_out(model, objects, out, replicas, w: float = W, nb: int = NB):
    """a bucketed run_ensemble output dict (the keys bucketed_data reads) restated from record-mode outputs"""
    recs = [host_buckets(model, out, r, w, nb) for r in replicas]
    return {"buckets": np.stack([x[0] for x in recs]), "bucket_past_end": np.stack([x[1] for x in recs]),
            "bucket_percentiles": np.stack([x[2] for x in recs]), "bucket_width_s": w, "bucket_count": nb,
            "bucket_rows": B.rows(model), "bucket_objects": B.row_objects(model, objects)}


def lists(bd) -> dict:
    """the seven lists of a BucketedData"""
    return {f: list(getattr(bd, f)()) for f in FIELDS}


def fixture_lists(z, q: int, b: int) -> dict:
    """the reference's Data.bucket(W) lists of bucketed row b of partition q, as the fixture stores them"""
    return {f: z[f"p{q}_bucket{b}_{f}"].tolist() for f in FIELDS}


def same(got: dict, want: dict) -> bool:
    """counts exact, floats bitwise"""
    for f in FIELDS:
        a, e = np.asarray(got[f], np.float64), np.asarray(want[f], np.float64)
        if a.shape != e.shape or a.view(np.uint64).tolist() != e.view(np.uint64).tolist():
            return False
    return True
