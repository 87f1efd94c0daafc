"""Time buckets of a linked ParallelSimulation, host side: the argument checks of run_ensemble(buckets=...), which come
before any device is touched, and the one function that fills the bucket keys of an ensemble's output dict."""
import numpy as np
import pytest

import happysim_b200 as hs
from happysim_b200 import _abi as A, buckets as B
from happysim_b200.lowering import UnsupportedModelError


def _linked(duration=3.0):
    lat, tp = hs.LatencyTracker("B.lat"), hs.ThroughputTracker("B.tp")
    b1 = hs.Server("B.s1", concurrency=2, service_time=hs.ExponentialLatency(0.015), downstream=lat)
    b2 = hs.Server("B.s2", service_time=hs.ExponentialLatency(0.03), downstream=tp)
    probe, data = hs.Probe.on(b1, "depth", interval=0.1)
    a1 = hs.Server("A.s1", service_time=hs.ExponentialLatency(0.008), downstream=b1)
    parts = [hs.SimulationPartition("A", entities=[a1], sources=[hs.Source.poisson(rate=80.0, target=a1, name="A.src")]),
             hs.SimulationPartition("B", entities=[b1, b2, lat, tp], probes=[probe],
                                    sources=[hs.Source.poisson(rate=20.0, target=b2, name="B.src")])]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=hs.ConstantLatency(0.05))
    return hs.ParallelSimulation(parts, duration=duration, links=[link], seed=9), (lat, tp, probe, data)


@pytest.mark.parametrize("kw, match", [
    (dict(buckets=(0.1, 30)), "end before the end time"),              # 30 x 0.1 s = 3 s: the end time is in bucket 30
    (dict(buckets=(0.0, 40)), "finite number of seconds"),
    (dict(buckets=(0.1, 2.5)), "must be an int"),
    (dict(buckets=0.1), r"\(width_s, n\)"),
    (dict(bucket_percentiles=True), "needs buckets"),
    (dict(buckets=(0.1, 31), bucket_percentiles=True, bucket_sample_cap=0), "bucket_sample_cap"),
])
def test_argument_errors_come_before_the_device(kw, match, monkeypatch):
    ps, _ = _linked()

    def no_device(*a, **k):
        raise AssertionError("the device was reached")
    monkeypatch.setattr(ps, "_run_linked", no_device)
    with pytest.raises(ValueError, match=match):
        ps.run_ensemble(8, **kw)


def test_arguments_reach_the_linked_run(monkeypatch):
    """checked (width, n) and the capacity (0 without percentiles) go to the window loop"""
    ps, _ = _linked()
    seen = []
    monkeypatch.setattr(ps, "_run_linked", lambda *a: seen.append(a) or ([{}, {}], 0, 0, 0.0, 0))
    ps.run_ensemble(8, 16, buckets=(0.1, 31), bucket_percentiles=True, bucket_sample_cap=32)
    ps.run_ensemble(8, buckets=(np.float32(0.5), np.int64(7)))
    ps.run_ensemble(8)
    assert seen == [(8, 16, (0.1, 31), 32), (8, 0, (0.5, 7), 0), (8, 0, None, 0)]


def test_run_ensemble_without_links_still_refuses():
    ps = hs.ParallelSimulation([hs.SimulationPartition("A", entities=[hs.Sink("s")])], duration=1.0)
    with pytest.raises(UnsupportedModelError):
        ps.run_ensemble(4, buckets=(0.5, 4))


class _FakeEngine:
    """the bucket readers of engine.Engine over fixed arrays"""

    def __init__(self, nr, rows, n):
        self.rec = np.zeros((nr, rows, n + 1), A.BUCKET_DTYPE)
        self.rec["count"][:, :, 0] = np.arange(nr * rows).reshape(nr, rows) + 1
        self.rec["sum"][:, :, 0] = 0.5 * self.rec["count"][:, :, 0]
        self.rec["max"][:, :, 0] = 0.5
        self.past = np.zeros((nr, rows), np.int64)
        self.pct = np.full((nr, rows, n + 1, 2), 0.25)

    def read_buckets(self, n):
        return self.rec, self.past

    def read_bucket_totals(self, n_cells, rows, n):
        return B.cell_totals_reference(self.rec, n_cells)

    def read_bucket_percentiles(self, n):
        return self.pct

    def read_bucket_percentile_totals(self, n_cells, rows, n):
        return B.cell_percentile_totals_reference(self.rec, self.pct, n_cells)


def test_read_outputs_gives_the_keys_bucketed_data_reads():
    """the partition B of the linked model: its rows are the two trackers and the Probe, in entity order, and
    bucketed_data finds each of them through the keys read_outputs fills"""
    ps, (lat, tp, probe, data) = _linked()
    lm = ps._linked
    m, objs = lm.models[1], lm.objects[1]
    assert len(B.rows(m)) == 3
    eng = _FakeEngine(4, 3, 31)
    plain = B.read_outputs(eng, (0.1, 31), 0, m, objs)
    assert set(plain) == {"buckets", "bucket_past_end", "bucket_totals", "bucket_width_s", "bucket_count", "bucket_rows",
                          "bucket_objects"}
    out = B.read_outputs(eng, (0.1, 31), 16, m, objs)
    assert set(out) - set(plain) == {"bucket_percentiles", "bucket_percentile_totals", "bucket_sample_cap"}
    assert out["bucket_sample_cap"] == 16 and out["bucket_totals"].shape == (1, 3, 32)
    assert out["bucket_rows"] == B.rows(m)
    assert {id(o) for o in out["bucket_objects"]} == {id(lat), id(tp), id(probe)}
    for b, o in enumerate(out["bucket_objects"]):
        got = B.bucketed_data(out, o, 2)
        c = int(eng.rec["count"][2, b, 0])
        assert got.counts() == [c] and got.times() == [0.0]
        assert got.p50s() == [1.0 if o is tp else 0.25]
    assert B.bucketed_data(out, data, 1).counts() == B.bucketed_data(out, probe, 1).counts()


# ---- the reference fixtures (tests/golden/gen_linked_bucket_golden.py) ----------------------------------------------

import golden_lib as G  # noqa: E402
import linked_bucket_models as LB  # noqa: E402
import layered_oracle_lib as LO  # noqa: E402
import oracle_lib as O  # noqa: E402


def _oracle(name, n=1):
    """the oracle (the linked fault oracle for a fixture with FAULT rows) on a fixture: (LinkedModel, npz, outputs)"""
    lm, kw, z = LB.load(name)
    nP = lm.n_partitions
    ps = [O.make_params(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=n, rid_base=q, rid_stride=nP + 1,
                        **G.linked_caps(z, q)) for q in range(nP)]
    run = LO.run_linked if any(m.ids_of(A.HS_ENT_FAULT) for m in lm.models) else O.oracle_run_linked
    outs, delivered, lost, ends = run(lm, ps, end_ns=kw["end_ns"], cseed=kw["seed"])
    assert len(ends) == int(z["total_windows"]) and int(delivered[0]) == int(z["cross_events"])
    return lm, z, outs


@pytest.mark.parametrize("name", list(LB.CASES))
def test_oracle_reproduces_the_bucket_fixture(name):
    """every record, sample and statistic of every partition, as the reference recorded them"""
    lm, z, outs = _oracle(name)
    for q in range(lm.n_partitions):
        G.check_linked_partition(z, q, outs[q])


@pytest.mark.parametrize("name", list(LB.CASES))
def test_mirror_lowers_to_the_fixture_and_oracle_buckets_equal_data_bucket(name):
    """the mirror script lowers to the fixture's models; the oracle's samples of each row, bucketed on the host, give
    bucketed_data equal to the reference's own Data.bucket lists (counts exact, floats bitwise)"""
    lm, z, outs = _oracle(name)
    ps = LB.CASES[name][0]()
    assert float(z["bucket_w"]) == LB.W and int(z["bucket_n"]) == LB.NB
    n_rows = 0
    for q in range(lm.n_partitions):
        assert ps._linked.models[q].entities.tobytes() == lm.models[q].entities.tobytes(), q
        out = LB.host_out(lm.models[q], ps._linked.objects[q], outs[q], [0])
        for b, obj in enumerate(out["bucket_objects"]):
            want = LB.fixture_lists(z, q, b)
            assert sum(want["counts"]) > 5, (q, b)
            assert LB.same(LB.lists(B.bucketed_data(out, obj, 0)), want), (q, b)
            n_rows += 1
    assert n_rows == {"lbucket_three_way": 3}.get(name, 4)


def test_the_references_own_objects_lower_to_the_tracker_fixture():
    G.import_reference()
    from happysimulator.components.common import Sink
    from happysimulator.components.server.server import Server
    from happysimulator.distributions.constant import ConstantLatency
    from happysimulator.distributions.exponential import ExponentialLatency
    from happysimulator.instrumentation.collectors import LatencyTracker, ThroughputTracker
    from happysimulator.instrumentation.probe import Probe
    from happysimulator.load.source import Source
    from happysimulator.parallel.link import PartitionLink
    from happysimulator.parallel.partition import SimulationPartition
    lat, tp = LatencyTracker("B.lat"), ThroughputTracker("B.tp")
    b1 = Server("B.s1", concurrency=2, service_time=ExponentialLatency(0.015), downstream=lat)
    b2 = Server("B.s2", service_time=ExponentialLatency(0.03), downstream=tp)
    probe, _ = Probe.on(b1, "depth", interval=0.1)
    asink = Sink("A.sink")
    a1 = Server("A.s1", service_time=ExponentialLatency(0.01), downstream=b1)
    a2 = Server("A.s2", service_time=ExponentialLatency(0.02), downstream=asink)
    hidden = lambda *ss: [x for s in ss for x in (s, s.queue, s.driver, s.worker)]
    parts = [SimulationPartition(name="A", entities=hidden(a1, a2) + [asink],
                                 sources=[Source.poisson(rate=60.0, target=a1, name="A.src"),
                                          Source.poisson(rate=25.0, target=a2, name="A.src2")]),
             SimulationPartition(name="B", entities=hidden(b1, b2) + [lat, tp], probes=[probe],
                                 sources=[Source.poisson(rate=20.0, target=b2, name="B.src")])]
    link = PartitionLink(source_partition="A", dest_partition="B", min_latency=0.05, latency=ConstantLatency(0.05))
    ps = hs.ParallelSimulation(parts, duration=3.0, links=[link], seed=23)
    lm, kw, z = LB.load("lbucket_tracker_tandem")
    for q in range(2):
        assert ps._linked.models[q].entities.tobytes() == lm.models[q].entities.tobytes(), q
