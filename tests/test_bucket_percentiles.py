"""Bucket percentiles (hs_set_bucket_percentiles, run_ensemble(bucket_percentiles=True)) on the host: the kernels'
selection and interpolation (hs_percentile.h, through its ctypes twin) against the reference's
``_percentile_sorted(sorted(vals), p)``, the numpy restatement of the device's per-cell percentile reduction, the
BucketedData a replica's percentile records give, the argument checks and the C-ABI layout."""
import math
import os
import random

import numpy as np
import pytest

import bucket_pct_lib as P
import golden_lib as G
import happysim_b200 as hs
from happysim_b200 import _abi as A, buckets as B
from happysim_b200.instrumentation import Data, _percentile_sorted

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _records_from_samples(samples, w, n):
    """the records the device keeps for one row: per bucket count, Neumaier pair, max (as tests/test_buckets.py)"""
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
        sm, c = float(r["sum"]), float(r["comp"])
        t2 = sm + v
        c += (sm - t2) + v if abs(sm) >= abs(v) else (v - t2) + sm
        r["sum"], r["comp"] = t2, c
    return rec, past


def _want(v):
    s = sorted(float(x) for x in v)
    return _percentile_sorted(s, 0.50), _percentile_sorted(s, 0.99)


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64).tolist()


def _multisets(seed):
    """thousands of multisets: every size up to 300, larger ones up to 10^4, heavy duplicates, values whose
    interpolation rounds, integer-valued Probe-like values, sorted and reversed runs"""
    rng = random.Random(seed)
    out = []
    for n in list(range(1, 301)) + [rng.randrange(301, 10_001) for _ in range(60)] + [10_000]:
        kind = rng.randrange(6)
        if kind == 0:
            v = [rng.expovariate(20.0) for _ in range(n)]                        # latencies
        elif kind == 1:
            v = [float(rng.randrange(0, 4)) for _ in range(n)]                   # heavy duplicates
        elif kind == 2:
            v = [float(rng.randrange(0, 200)) for _ in range(n)]                 # queue depths, counts
        elif kind == 3:
            v = [rng.random() * 10 ** rng.randrange(-9, 9) for _ in range(n)]    # interpolation across magnitudes
        elif kind == 4:
            v = sorted(rng.expovariate(1.0) for _ in range(n))
            if rng.random() < 0.5:
                v.reverse()
        else:
            base = [rng.expovariate(3.0) for _ in range(rng.randrange(1, 4))]
            v = [rng.choice(base) for _ in range(n)]                             # a few distinct values, repeated
        out.append(v)
    out += [[0.0], [0.0, 0.0], [1e-300, 5e-324, 0.0], [0.1, 0.2, 0.3], [1.0] * 101, [2.0 ** 60, 1.0, 3.0]]
    return out


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_twin_equals_percentile_sorted(seed):
    sets = _multisets(seed)
    got = P.percentiles(sets)
    want = np.array([_want(v) for v in sets])
    assert len(sets) > 350
    assert _bits(got) == _bits(want)


def test_twin_covers_rounding_interpolation():
    """sizes and values where 1.0 - frac and the final sum round: the explicit rounding keeps every bit"""
    rng = random.Random(11)
    sets = []
    for n in (3, 7, 13, 51, 99, 101, 151, 1000, 1001, 9999):
        for _ in range(40):
            sets.append([rng.uniform(0.0, 1.0) * 10 ** rng.randrange(-3, 4) for _ in range(n)])
    got = P.percentiles(sets)
    want = np.array([_want(v) for v in sets])
    assert _bits(got) == _bits(want)


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
def test_twin_equals_reference_data_bucket():
    """the reference's own Data.bucket(w).p50s() / p99s() over samples whose buckets are the multisets"""
    ref = G.import_reference()
    from happysimulator.instrumentation.data import Data as RefData
    sets = _multisets(7)[::3]
    d = RefData()
    w = 1.0
    for k, v in enumerate(sets):
        for i, x in enumerate(v):
            d._samples.append((k * w + (i + 0.5) / (len(v) + 1) * w, float(x)))
    b = d.bucket(w)
    assert b.counts() == [len(v) for v in sets]
    got = P.percentiles(sets)
    assert _bits(got[:, 0]) == _bits(b.p50s()) and _bits(got[:, 1]) == _bits(b.p99s())
    assert ref is not None


def _random_pct_records(rng, nr, rows, nb):
    b = np.zeros((nr, rows, nb + 1), A.BUCKET_DTYPE)
    b["count"] = rng.integers(0, 3, size=b.shape)
    pct = rng.random(b.shape + (2,)) * 10.0 ** rng.integers(-3, 3, size=b.shape + (2,))
    pct = np.where(b["count"][..., None] > 0, pct, 0.0)
    return b, pct


def test_cell_percentile_reduction_reference_equals_a_loop():
    rng = np.random.default_rng(4)
    nr, rows, nb = 700, 2, 5
    b, pct = _random_pct_records(rng, nr, rows, nb)
    for rpc, n_cells, base in [(1, 1, 0), (100, 4, 0), (37, 3, 5), (700, 1, 0)]:
        got = B.cell_percentile_totals_reference(b, pct, n_cells, replica_index_base=base, replicas_per_cell=rpc)
        assert got.dtype == A.BUCKET_PCT_TOTAL_DTYPE and got.shape == (n_cells, rows, nb + 1)
        cell = [((base + r) // rpc) % n_cells for r in range(nr)]
        for c in range(n_cells):
            for i in range(rows):
                for j in range(nb + 1):
                    # the device's order: slices of <= 256 consecutive replicas of the cell, then the slices
                    parts, r = [], 0
                    while r < nr:
                        c0, end = cell[r], r + 1
                        while end < min(r + 256, nr) and cell[end] == c0:
                            end += 1
                        if c0 == c:
                            s = [0.0, 0.0, 0.0, 0.0]
                            for q in range(r, end):
                                if b[q, i, j]["count"] > 0:
                                    x, y = float(pct[q, i, j, 0]), float(pct[q, i, j, 1])
                                    s = [s[0] + x, s[1] + x * x, s[2] + y, s[3] + y * y]
                            parts.append(s)
                        r = end
                    tot = [0.0, 0.0, 0.0, 0.0]
                    for s in parts:
                        tot = [a + z for a, z in zip(tot, s)]
                    assert _bits([got[c, i, j][f] for f in A.BUCKET_PCT_TOTAL_DTYPE.names]) == _bits(tot)


def test_cell_totals_reference_unchanged_by_the_shared_slicing():
    """the shared slice generator gives cell_totals_reference the slices it had: a plain ensemble and one cell of
    all replicas agree bit for bit"""
    rng = np.random.default_rng(8)
    b = np.zeros((1000, 1, 5), A.BUCKET_DTYPE)
    b["count"] = rng.integers(1, 4, size=b.shape)
    b["sum"] = rng.random(b.shape)
    b["max"] = rng.random(b.shape)
    assert (B.cell_totals_reference(b, 1).tobytes() == B.cell_totals_reference(b, 1, replicas_per_cell=1000).tobytes())
    assert [s for s in B._cell_slices(600, 2, 0, 100)] == [(0, 0, 100), (1, 100, 200), (0, 200, 300), (1, 300, 400),
                                                         (0, 400, 500), (1, 500, 600)]
    assert [s for s in B._cell_slices(600, 1, 0, 1)] == [(0, 0, 256), (0, 256, 512), (0, 512, 600)]


def _out_for(obj, samples, w, n, with_pct):
    rec, past = _records_from_samples(samples, w, n)
    out = {"bucket_objects": [obj], "bucket_width_s": w, "bucket_count": n,
           "buckets": rec[None, None, :], "bucket_past_end": np.array([[past]], np.int64)}
    if with_pct:
        groups = {}
        for t, v in samples:
            k = B.bucket_index(t, w)
            groups.setdefault(min(k, n), []).append(v)
        pct = np.zeros((1, 1, n + 1, 2))
        for s, vals in groups.items():
            pct[0, 0, s] = P.percentiles([vals])[0]
        out["bucket_percentiles"] = pct
    return out


@pytest.mark.parametrize("kind", ["latency", "throughput", "probe"])
def test_bucketed_data_with_and_without_percentiles(kind):
    rng = random.Random(9)
    w, n = 0.1, 12
    t = sorted(rng.randrange(0, 1_150_000_000) for _ in range(700)) + [1_300_000_000]
    if kind == "probe":
        vals = [float(rng.randrange(0, 30)) for _ in t]
        obj = hs.LatencyTracker("depth-like")
    else:
        vals = [rng.expovariate(3.0) for _ in t]
        obj = hs.ThroughputTracker("tp") if kind == "throughput" else hs.LatencyTracker("lat")
    samples = list(zip(t, vals))
    d = Data()
    d._samples = [(x / 1_000_000_000, 1.0 if kind == "throughput" else v) for x, v in samples]
    want = d.bucket(w)

    plain = B.bucketed_data(_out_for(obj, samples, w, n, False), obj, 0)
    assert all(math.isnan(x) for x in plain.p50s() + plain.p99s())
    assert plain.counts() == want.counts()

    got = B.bucketed_data(_out_for(obj, samples, w, n, True), obj, 0)
    assert got.times() == want.times() and got.counts() == want.counts() and got.sums() == want.sums()
    assert _bits(got.p50s()) == _bits(want.p50s()) and _bits(got.p99s()) == _bits(want.p99s())
    if kind == "throughput":
        assert got.p50s() == [1.0] * len(want.times()) == got.p99s()


def test_bucketed_data_overflowed_bucket_is_nan():
    obj = hs.LatencyTracker("lat")
    samples = [(100_000_000, 0.5), (150_000_000, 0.25), (350_000_000, 1.0)]
    out = _out_for(obj, samples, 0.2, 4, True)
    out["bucket_percentiles"][0, 0, 0] = np.nan
    got = B.bucketed_data(out, obj, 0)
    assert math.isnan(got.p50s()[0]) and math.isnan(got.p99s()[0]) and got.p50s()[1] == 1.0


def test_sample_cap_checks():
    spec = (0.1, 10)
    assert B.check_sample_cap(64, spec) == 64 and B.check_sample_cap(np.int64(1), spec) == 1
    for bad in [0, -1, 1.5, True, None, (1 << 24) + 1]:
        with pytest.raises(ValueError):
            B.check_sample_cap(bad, spec)
    with pytest.raises(ValueError, match="needs buckets"):
        B.check_sample_cap(64, None)
    rec = np.zeros((3, 1, 5), A.BUCKET_DTYPE)
    rec["count"][1, 0, 2] = 65
    assert B.sample_cap_needed(rec) == 128
    rec["count"][1, 0, 2] = 64
    assert B.sample_cap_needed(rec) == 64
    rec["count"][:] = 0
    assert B.sample_cap_needed(rec) == 1


def test_abi():
    assert A.HS_ST_BUCKET_OVERFLOW == 512 and A.BUCKET_PCT_TOTAL_DTYPE.itemsize == 32
    assert A.BUCKET_PCT_TOTAL_DTYPE.names == ("p50_sum", "p50_sq_sum", "p99_sum", "p99_sq_sum")
    hdr = open(os.path.join(ROOT, "include", "hs_b200.h")).read()
    assert "#define HS_ST_BUCKET_OVERFLOW 512u" in hdr
    for fn in ("hs_set_bucket_percentiles", "hs_read_bucket_percentiles", "hs_read_bucket_percentile_totals"):
        assert fn in hdr
