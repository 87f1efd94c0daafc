"""Time buckets (hs_set_buckets, Simulation.run_ensemble(buckets=)) on the host: the bucket index restated against
``math.floor(t / w)`` of the reference's Data.bucket, the argument checks, the C-ABI layouts, the row mapping, the
BucketedData a replica's records give, and the numpy restatement of the device's cell reduction."""
import ctypes as C
import math
import os
import random

import numpy as np
import pytest

import happysim_b200 as hs
from happysim_b200 import _abi as A, buckets as B
from happysim_b200.instrumentation import Data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _T:
    def __init__(self, ns):
        self.ns = ns

    def to_seconds(self):
        return self.ns / 1_000_000_000


def _ref_index(ns, w):
    return math.floor(_T(ns).to_seconds() / w)


@pytest.mark.parametrize("w", [0.1, 0.3, 1e-3, 7.5])
def test_bucket_index_matches_math_floor(w):
    rng = random.Random(int(w * 1e6))
    ns = [rng.randrange(0, 10**13) for _ in range(4000)]
    # exact multiples of the width, their neighbours, and times whose ns / 1e9 rounds onto a boundary
    for k in range(0, 2000):
        b = int(round(k * w * 1e9))
        ns += [b - 1, b, b + 1]
    ns = [x for x in ns if x >= 0]
    got = B.bucket_index(np.array(ns, np.int64), w)
    want = [_ref_index(x, w) for x in ns]
    assert got.tolist() == want
    assert [B.bucket_index(x, w) for x in ns[:500]] == want[:500]


def test_bucket_index_is_not_integer_arithmetic():
    # 0.3 / 0.1 == 2.9999999999999996: the sample at 300 ms lies in bucket 2, not 3
    assert B.bucket_index(300_000_000, 0.1) == 2 == math.floor(0.3 / 0.1)
    assert 300_000_000 // 100_000_000 == 3
    assert B.bucket_index(np.array([300_000_000]), 0.1).tolist() == [2]


def test_check_spec():
    assert B.check_spec((0.1, 11), 10**9) == (0.1, 11)
    assert B.check_spec((1, 2), 10**9) == (1.0, 2)
    for bad in [None, 0.1, (0.1,), (0.1, 2, 3), (0.0, 10), (-1.0, 10), (float("inf"), 10), (float("nan"), 10),
                (0.1, 0), (0.1, -3), (0.1, 2.0), (0.1, True), (0.1, (1 << 24) + 1)]:
        with pytest.raises(ValueError):
            B.check_spec(bad, 10**9)
    with pytest.raises(ValueError, match="end time"):
        B.check_spec((0.1, 10), 10**9)          # 1.0 / 0.1 == 10.0: the end time falls in bucket 10
    with pytest.raises(ValueError, match="end time"):
        B.check_spec((1.0, 59), 60 * 10**9)


def test_abi_layouts():
    assert A.HS_ABI_VERSION == 7
    assert A.BUCKET_DTYPE.itemsize == 32 and A.BUCKET_TOTAL_DTYPE.itemsize == 48
    assert A.BUCKET_DTYPE.names == ("count", "sum", "comp", "max")
    assert A.BUCKET_TOTAL_DTYPE.names == ("replicas", "count", "sum", "mean_sum", "mean_sq_sum", "max")
    hdr = open(os.path.join(ROOT, "include", "hs_b200.h")).read()
    assert "#define HS_ABI_VERSION 7u" in hdr
    for name in ("hs_set_buckets", "hs_read_buckets", "hs_read_bucket_totals"):
        assert f"int {name}(" in hdr
        assert name in hs.engine.EXPORTED_SYMBOLS


def test_rows_and_objects():
    m = hs.mm1()
    assert B.rows(m) == m.ids_of(A.HS_ENT_SINK)
    srv = hs.Server("srv", service_time=hs.ExponentialLatency(0.05))
    lat = hs.LatencyTracker("lat")
    srv.downstream = lat
    probe, data = hs.Probe.on(srv, "depth", interval=0.5)
    sim = hs.Simulation(sources=[hs.Source.poisson(rate=5.0, target=srv, name="src")], entities=[srv, lat],
                        probes=[probe], end_time=hs.Instant.from_seconds(3.0))
    rows = B.rows(sim.model)
    objs = B.row_objects(sim.model, sim.objects)
    assert len(rows) == 2 and objs[0] is lat and objs[1] is probe
    out = {"bucket_objects": objs}
    assert B._row_of(out, data) == 1 and B._row_of(out, lat) == 0
    with pytest.raises(KeyError):
        B._row_of(out, srv)


def _records_from_samples(samples, w, n):
    """the records the device keeps for one row: per bucket count, Neumaier pair, max"""
    rec = np.zeros(n + 1, A.BUCKET_DTYPE)
    past = 0
    for t, v in samples:
        k = B.bucket_index(t, w)
        s = k if k < n else n
        if k >= n:
            past = k
        r = rec[s]
        r["max"] = v if (r["count"] == 0 or v > r["max"]) else r["max"]
        r["count"] += 1
        # hs_neumaier_add
        sm, c = float(r["sum"]), float(r["comp"])
        t2 = sm + v
        c += (sm - t2) + v if abs(sm) >= abs(v) else (v - t2) + sm
        r["sum"], r["comp"] = t2, c
    return rec, past


@pytest.mark.parametrize("tracker", [False, True])
def test_bucketed_data_equals_data_bucket(tracker):
    rng = random.Random(5)
    w, n = 0.1, 12
    t = sorted(rng.randrange(0, 1_150_000_000) for _ in range(500)) + [1_300_000_000]   # the last one past bucket n
    vals = [rng.expovariate(3.0) * (10 ** rng.randrange(-3, 4)) for _ in t]
    rec, past = _records_from_samples(list(zip(t, vals)), w, n)
    obj = hs.ThroughputTracker("tp") if tracker else hs.LatencyTracker("lat")
    out = {"bucket_objects": [obj], "bucket_width_s": w, "bucket_count": n,
           "buckets": rec[None, None, :], "bucket_past_end": np.array([[past]], np.int64)}
    got = B.bucketed_data(out, obj, 0)
    d = Data()
    d._samples = [(x / 1_000_000_000, 1.0 if tracker else v) for x, v in zip(t, vals)]
    want = d.bucket(w)
    assert got.times() == want.times() and got.counts() == want.counts()
    assert got.sums() == want.sums() and got.means() == want.means() and got.maxes() == want.maxes()
    assert all(math.isnan(x) for x in got.p50s() + got.p99s())
    assert want.times()[-1] == 13 * w


def test_cell_reduction_reference():
    rng = np.random.default_rng(3)
    nr, rows, nb = 1000, 2, 7
    b = np.zeros((nr, rows, nb + 1), A.BUCKET_DTYPE)
    b["count"] = rng.integers(0, 4, size=b.shape)
    b["sum"] = np.where(b["count"] > 0, rng.random(b.shape) * b["count"], 0.0)
    b["comp"] = np.where(rng.random(b.shape) < 0.2, rng.random(b.shape) * 1e-17, 0.0)
    b["max"] = rng.random(b.shape)
    for rpc, n_cells, base in [(1, 1, 0), (100, 10, 0), (37, 4, 5), (1000, 1, 0)]:
        got = B.cell_totals_reference(b, n_cells, replica_index_base=base, replicas_per_cell=rpc)
        cell = ((base + np.arange(nr)) // rpc) % n_cells
        for c in range(n_cells):
            sel = b[cell == c]
            has = sel["count"] > 0
            assert (got[c]["replicas"] == has.sum(0)).all()
            assert (got[c]["count"] == sel["count"].sum(0)).all()
            s = B.replica_sums(sel)
            m = np.where(has, s / np.maximum(sel["count"], 1), 0.0)
            for f, x in (("sum", np.where(has, s, 0.0)), ("mean_sum", m), ("mean_sq_sum", m * m)):
                exact = np.array([[math.fsum(x[:, i, j]) for j in range(nb + 1)] for i in range(rows)])
                bound = 2 * len(sel) * np.finfo(float).eps * np.abs(x).sum(0) + 1e-300
                assert (np.abs(got[c][f] - exact) <= bound).all(), f
            mx = np.where(has, sel["max"], -np.inf).max(0)
            assert (got[c]["max"] == mx).all()
    # fixed order: the same input gives the same bits
    a1 = B.cell_totals_reference(b, 3, replicas_per_cell=50)
    a2 = B.cell_totals_reference(b.copy(), 3, replicas_per_cell=50)
    assert a1.tobytes() == a2.tobytes()


def test_cell_reduction_slices_follow_cells_not_runs():
    """a plain ensemble (replicas_per_cell = 1, one cell) is sliced 256 replicas at a time, as one cell of 1 000
    replicas is: the same order, the same bits"""
    rng = np.random.default_rng(8)
    b = np.zeros((1000, 1, 5), A.BUCKET_DTYPE)
    b["count"] = rng.integers(1, 4, size=b.shape)
    b["sum"] = rng.random(b.shape) * 1e3 ** rng.integers(-2, 3, size=b.shape)
    b["max"] = rng.random(b.shape)
    plain = B.cell_totals_reference(b, 1, replicas_per_cell=1)
    one_cell = B.cell_totals_reference(b, 1, replicas_per_cell=1000)
    assert plain.tobytes() == one_cell.tobytes()
    # two cells interleaved run by run: each cell's slices only ever hold that cell's replicas
    two = B.cell_totals_reference(b, 2, replicas_per_cell=10)
    cell = (np.arange(1000) // 10) % 2
    for c in range(2):
        assert (two[c]["count"] == b[cell == c]["count"].sum(0)).all()


def test_throughput_tracker_subclass_is_counted_as_ones():
    class MyTracker(hs.ThroughputTracker):
        pass
    t = [100_000_000, 150_000_000, 450_000_000]
    rec, past = _records_from_samples([(x, 0.25) for x in t], 0.2, 4)
    obj = MyTracker("mine")
    out = {"bucket_objects": [obj], "bucket_width_s": 0.2, "bucket_count": 4,
           "buckets": rec[None, None, :], "bucket_past_end": np.array([[past]], np.int64)}
    got = B.bucketed_data(out, obj, 0)
    assert got.sums() == [2.0, 1.0] and got.maxes() == [1.0, 1.0] and got.means() == [1.0, 1.0]
