"""Node faults on the seeded random models (tests/random_models.py: random_model, random_model_v2, each with the random
fault plan of random_fault_case) on the device, every replica against the fault oracle (tests/fault_oracle.c), which
tests/test_faults.py pins against the unmodified reference on the same models.

(a) every model on the auto, warp and thread engines, replica word 0 also against the reference's fixture
    (tests/golden/random_fault_models.npz); the models with a random key table (no reference counterpart) against the
    oracle only;
(b) a few models whose plans crash a counter, a sketch, a load balancer, a CachingServer, a multi-slot / LIFO / bounded
    server and a source, with a cancelled fault among them, at every thread-engine geometry (the wide kernel, the
    phase-locked dispatch at 1 to 32 replicas per warp with and without the shared heap top) and on the warp engine
    with staged second replicas;
(c) windowed runs cut around the first fault that fires, at a cancelled fault's pop and at end - 1, against the uncut run;
(d) time buckets and their percentiles of faulted models against the samples of a record-mode run.

A replica whose in-run event tied a fault event on (time, sort index) is flagged HS_ST_FAULT_TIE; past such a tie the
engines do not restate heapq's layout order (DESIGN.md).  The flagged set must equal the oracle's, every other replica is
compared in full, and a run where more than MAX_TIE_FRACTION of the replicas are flagged fails, so that the comparison
cannot quietly empty itself.  The number of tied replicas is reported as the test property ``fault_ties``."""
import numpy as np
import pytest

import fault_oracle_lib as FO
from happysim_b200 import _abi as A, buckets as B, engine, lowering
from random_models import FAULT_SEEDS_V1, FAULT_SEEDS_V2, random_fault_case, with_faults
from test_faults import check_random_fault_reference
from test_gpu_bucket_percentiles import CAP, _bucket_run, _check_pct, _record_run
from test_gpu_buckets import _check_replicas
from test_gpu_launch_geometry import CAPS, FLAGS, GEOMETRY, RING, assert_same, check_thread_geometry, compare

pytestmark = pytest.mark.gpu

WF_PROFILE, WF_HEAPTOP, WF_FAULTS, WF_BUCKETS, WF_BUCKET_PCT = 4, 8, 32, 64, 128     # HS_WF_* of csrc/hs_warp_engine.cuh
KEYS = ("summaries", "entity_stats", "records", "sink_samples", "service_samples", "histograms", "sketches")
MAX_TIE_FRACTION = 0.05
# rings that hold a whole run of every model (the oracle's longest replica processes about 15 000 events)
WHOLE = dict(record_cap=16384, sample_cap=4096, service_cap=4096)

ALL_CASES = [(1, s) for s in range(max(FAULT_SEEDS_V1) + 1)] + [(2, s) for s in FAULT_SEEDS_V2]


def _id(c):
    return f"v{c[0]}-{c[1]}"


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def faulted(version, seed, scale=1.0):
    """-> (the model with its FAULT rows, end_ns, run seed)"""
    model, end_s, plan, cancel, run_seed, _, _ = random_fault_case(version, seed, scale)
    return with_faults(model, plan, cancel), int(end_s * 1e9), run_seed


def compare_tie_aware(got, want, keys=KEYS):
    """The fault-tie flags of every replica equal the oracle's; the unflagged replicas equal it bit for bit in ``keys``.
    Returns the number of flagged replicas."""
    tg = (got["summaries"]["status"] & A.HS_ST_FAULT_TIE) != 0
    tw = (want["summaries"]["status"] & A.HS_ST_FAULT_TIE) != 0
    assert np.array_equal(tg, tw), f"fault-tie flags: device {np.flatnonzero(tg)[:8]}, oracle {np.flatnonzero(tw)[:8]}"
    assert tw.mean() <= MAX_TIE_FRACTION, f"{int(tw.sum())} of {len(tw)} replicas tied with a fault event"
    if tw.any():
        keep = np.flatnonzero(~tw)
        got = {k: None if got.get(k) is None else np.ascontiguousarray(got[k][keep]) for k in keys}
        want = {k: None if want.get(k) is None else np.ascontiguousarray(want[k][keep]) for k in keys}
    assert_same(got, want, keys=[k for k in keys if want.get(k) is not None])
    return int(tw.sum())


# ---- (a) every model, every general engine -------------------------------------------------------------------------

@pytest.mark.parametrize("case", ALL_CASES, ids=_id)
def test_every_engine_matches_the_fault_oracle(eng, case, record_property):
    version, seed = case
    fm, end_ns, run_seed = faulted(version, seed)
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=5, rid_stride=1, **WHOLE)
    want = FO.run(fm, engine.make_params(**kw))
    assert int(want["summaries"]["events_processed"].max()) < WHOLE["record_cap"]
    with_ref = version == 2 or seed in FAULT_SEEDS_V1
    eng.upload(fm)
    ties = 0
    for e in (0, 1, 3):                  # auto: the thread engine (faults are not lane-eligible)
        eng.run(engine.make_params(engine=e, **kw))
        li = eng.last_launch()
        assert li["engine"] == (1 if e == 1 else 3) and li["flags"] & WF_FAULTS, (e, li)
        got = eng.read_outputs()
        ties += compare_tie_aware(got, want)
        if with_ref:
            check_random_fault_reference(fm, version, seed, got, r=0)
    record_property("fault_ties", ties)


# ---- (b) every thread-engine geometry --------------------------------------------------------------------------------

# Plans drawn on a quarter of each model's horizon; test_geometry_seeds_crash_every_kind checks what they cover.
GEO_SCALE = 0.25
GEOMETRY_CASES = [(1, 8), (1, 18), (1, 21), (1, 35), (2, 4), (2, 11)]


def crashed_kinds(fm):
    """what the model's FAULT rows do: the kinds of entity a crash or pause event that is not cancelled reaches
    ('server_special': a multi-slot, LIFO or bounded server), and 'cancelled' if an event is cancelled"""
    E = fm.entities
    out = set()
    names = {A.HS_ENT_COUNTER: "counter", A.HS_ENT_SKETCH: "sketch", A.HS_ENT_LB: "lb", A.HS_ENT_CACHE_SERVER: "cache",
             A.HS_ENT_SOURCE: "source", A.HS_ENT_SINK: "sink", A.HS_ENT_SERVER: "server"}
    for i in fm.ids_of(A.HS_ENT_FAULT):
        if E["i2"][i]:
            out.add("cancelled")
        elif E["i1"][i]:
            t = int(E["target"][i])
            k = names[int(E["kind"][t])]
            if k == "server" and (E["i0"][t] > 1 or E["i1"][t] == A.HS_Q_LIFO or E["l0"][t] >= 0):
                k = "server_special"
            out.add(k)
    return out


def test_geometry_seeds_crash_every_kind():
    got = set().union(*(crashed_kinds(faulted(v, s, GEO_SCALE)[0]) for v, s in GEOMETRY_CASES))
    assert {"counter", "sketch", "lb", "cache", "server_special", "source", "cancelled"} <= got, got


@pytest.mark.parametrize("row", sorted(GEOMETRY) + ["warp"])
@pytest.mark.parametrize("case", GEOMETRY_CASES, ids=_id)
def test_every_geometry_matches_the_fault_oracle(eng, sm, case, row, record_property):
    """``row`` of test_gpu_launch_geometry.GEOMETRY on the thread engine; "warp": the warp engine at the rpw32 size,
    where its persistent warps stage second replicas"""
    version, seed = case
    fm, end_ns, run_seed = faulted(version, seed, GEO_SCALE)
    n = GEOMETRY["rpw32" if row == "warp" else row][0](sm)
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=n, flags=FLAGS, queue_ring=RING, **CAPS)
    eng.upload(fm)
    eng.run(engine.make_params(engine=1 if row == "warp" else 3, **kw))
    li = eng.last_launch()
    assert li["flags"] & WF_FAULTS, li
    if row == "warp":
        assert (li["engine"], li["kernel"]) == (1, "warp") and n > li["grid"] * li["block"] // 32, li
    else:
        check_thread_geometry(li, row, n)
    got = eng.read_outputs()
    assert not (got["summaries"]["status"] & A.HS_ST_QUEUE_OVERFLOW).any(), "queue ring too small for this model"
    want = FO.run(fm, engine.make_params(**kw))
    assert np.median(want["summaries"]["events_processed"]) > CAPS["record_cap"]       # the rings wrap
    ties = compare_tie_aware(got, want)
    if not ties:
        compare(eng, fm, got, want)      # and the device's merged sketch image
    record_property("fault_ties", ties)


# ---- (c) windows cut at fault instants ---------------------------------------------------------------------------------

def fault_cuts(fm, end_ns):
    """t - 1, t and t + 1 ns of the first fault event that fires, the time of the first cancelled one, end - 1"""
    E = fm.entities
    fr = fm.ids_of(A.HS_ENT_FAULT)
    fired = [int(E["l0"][i]) for i in fr if not E["i2"][i] and int(E["l0"][i]) <= end_ns]
    cancelled = [int(E["l0"][i]) for i in fr if E["i2"][i]]
    cuts = [end_ns - 1]
    if fired:
        t = min(fired)
        cuts += [t - 1, t, t + 1]
    if cancelled:
        cuts.append(min(cancelled))
    return sorted({c for c in cuts if 0 <= c < end_ns})


@pytest.mark.parametrize("eng_id", [1, 3])
@pytest.mark.parametrize("case", ALL_CASES[::2], ids=_id)
def test_windows_cut_at_fault_instants(eng, case, eng_id):
    version, seed = case
    fm, end_ns, run_seed = faulted(version, seed)
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=32, rid_stride=1, engine=eng_id, **WHOLE)
    eng.upload(fm)
    eng.run(engine.make_params(**kw))
    whole = eng.read_outputs()
    cuts = fault_cuts(fm, end_ns)
    assert len(cuts) >= 1
    for cut in cuts:
        eng.run(engine.make_params(window_end_ns=cut, **kw))
        eng.run(engine.make_params(resume=1, **kw))
        got = eng.read_outputs()
        for k in KEYS:
            if whole[k] is not None:
                assert got[k].tobytes() == whole[k].tobytes(), (cut, k)


# ---- (d) time buckets ----------------------------------------------------------------------------------------------------

BUCKET_CASES = [(1, 0), (1, 2), (1, 8), (1, 16), (1, 23), (1, 29), (1, 62), (2, 1)]      # each has a Sink or a Probe


@pytest.mark.parametrize("pct", [0, 1])
@pytest.mark.parametrize("geometry", ["thread_wide", "thread_heaptop"])
@pytest.mark.parametrize("case", BUCKET_CASES, ids=_id)
def test_buckets_of_faulted_models(eng, sm, case, geometry, pct):
    """bucket records against Data.bucket(w) of a record-mode run's samples; p50 / p99 against _percentile_sorted"""
    version, seed = case
    fm, end_ns, run_seed = faulted(version, seed)
    assert {A.HS_ENT_SINK, A.HS_ENT_PROBE} & set(fm.entities["kind"].tolist())
    n_rep = 64 if geometry == "thread_wide" else GEOMETRY["rpw2"][0](sm)
    end_s = end_ns / 1e9
    w = 0.1
    n = int(end_s / w) + 2
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=n_rep, rid_stride=1, engine=3, flags=0)
    eng.upload(fm)
    got, past, pq, info, st = _bucket_run(eng, kw, w, n, CAP if pct else 0)
    fl = WF_FAULTS | WF_BUCKETS | WF_PROFILE | (WF_HEAPTOP if geometry == "thread_heaptop" else 0) | (WF_BUCKET_PCT if pct else 0)
    assert info["flags"] == fl and info["kernel"] == ("thread_wide" if geometry == "thread_wide" else "thread"), info
    assert not (st & A.HS_ST_BUCKET_OVERFLOW).any()
    smp = int(lowering.source_rate_bound(fm) * end_s * 1.5) + 256
    rec = _record_run(eng, kw, smp, smp * 16 if len(B.rows(fm)) > 1 else 0)
    picked = range(0, n_rep, 1 if n_rep <= 64 else 7)
    assert _check_replicas(fm, rec, got, past, w, n, replicas=picked) > len(picked)
    if pct:
        assert _check_pct(fm, rec, got, pq, w, n, picked) > len(picked)
