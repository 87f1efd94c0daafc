"""Data / BucketedData mirrors against the reference's own classes (when the checkout is present)
and against hand-checked values."""
import os
import random

import numpy as np

import golden_lib as G
import happysim_b200 as hs


def test_data_aggregations_hand_checked():
    d = hs.Data()
    d._samples = [(0.1, 1.0), (0.6, 3.0), (1.2, 2.0), (2.9, 10.0)]
    assert d.count() == 4 and d.sum() == 16.0 and d.mean() == 4.0 and d.min() == 1.0 and d.max() == 10.0
    assert d.percentile(0.0) == 1.0 and d.percentile(1.0) == 10.0 and d.percentile(0.5) == 2.5
    b = d.bucket(1.0)
    assert b.times() == [0.0, 1.0, 2.0] and b.counts() == [2, 1, 1] and b.sums() == [4.0, 2.0, 10.0]
    assert d.between(0.5, 2.0).raw_values() == [3.0, 2.0]
    assert d.rate(1.0).raw_values() == [2.0, 1.0, 1.0]
    assert hs.Data().mean() == 0.0 and hs.Data().percentile(0.9) == 0.0 and not hs.Data()


DATA_PERCENTILES = (0.0, 0.5, 0.9, 0.99, 1.0)
HELPER_SIZES = (0, 1, 2, 3, 7, 100, 1001)


def data_samples():
    rnd = random.Random(3)
    return sorted((rnd.random() * 30, rnd.expovariate(2.0)) for _ in range(2000))


def helper_cases():
    rnd = random.Random(1)
    cases = []
    for n in HELPER_SIZES:
        v = sorted(rnd.random() * 10 for _ in range(n))
        cases += [(v, p) for p in (-1, 0, 1e-9, 0.25, 0.5, 0.99, 0.999, 1, 2, rnd.random(), rnd.random())]
    return cases


def _reference_answers():
    """What the reference's Data class and _percentile_sorted answered for these inputs
    (tests/golden/gen_instrumentation_golden.py)."""
    return np.load(os.path.join(G.GOLDEN_DIR, "instrumentation_data.npz"))


def test_data_matches_the_reference_class():
    want = _reference_answers()
    a = hs.Data()
    a._samples = data_samples()
    assert [a.mean(), a.min(), a.max(), a.count(), a.sum(), a.std()] == want["stats"].tolist()
    assert [a.percentile(p) for p in DATA_PERCENTILES] == want["percentiles"].tolist()
    got = a.bucket(2.5).to_dict()
    assert sorted(got) == sorted(k[len("bucket_"):] for k in want.files if k.startswith("bucket_"))
    for k, v in got.items():
        assert [float(x) for x in v] == want["bucket_" + k].tolist(), k
    assert [list(r) for r in a.rate(5.0).values] == want["rate"].tolist()


def test_percentile_helper_equals_the_reference_helper_float_for_float():
    from happysim_b200.instrumentation import _percentile_sorted as mine
    cases = helper_cases()
    want = _reference_answers()["helper"].tolist()
    assert len(cases) == len(want)
    for (v, p), w in zip(cases, want):
        assert mine(v, p) == w, (len(v), p)
