"""Bucket percentiles on the device (hs_set_bucket_percentiles, run_ensemble(bucket_percentiles=True)): every replica's
p50 and p99 of every bucket against the reference's _percentile_sorted(sorted(vals), p) of the same replica's complete
sample list, taken from a record-mode run of the same seeds on the same engine, bit for bit.  Every run asserts through
Engine.last_launch() the percentile instantiation it meant to reach: the lane engine's six (general, profile and M/M/1
chains, with and without the order hash), the warp engine's four and the thread engine's twelve (wide, plain and
HEAPTOP, with and without faults and hash), and that its bucket records are byte-identical to the same run without
percentiles.  Also: runs cut into windows mid-bucket, the sample-capacity overflow, the per-cell totals of a sweep,
trackers and a Probe through the Python API, configs[1] at full size, and the refusals."""
import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
from happysim_b200 import _abi as A, buckets as B, engine, results
from happysim_b200.api import EnsembleStatusError
from happysim_b200.instrumentation import _percentile_sorted

pytestmark = pytest.mark.gpu

LF_HASH, LF_PROFILE, LF_SIMPLE, LF_BUCKETS, LF_BUCKET_PCT = 1, 4, 8, 16, 32
WF_HASH, WF_PROFILE, WF_HEAPTOP, WF_FAULTS, WF_BUCKETS, WF_BUCKET_PCT = 1, 4, 8, 32, 64, 128
CAP = 512


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def _record_run(eng, kw, sample_cap, record_cap):
    eng.set_bucket_percentiles(0)
    eng.set_buckets(0.0, 0)
    eng.run(engine.make_params(sample_cap=sample_cap, record_cap=record_cap, **kw))
    out = eng.read_outputs()
    assert (out["summaries"]["n_sink_samples"] <= sample_cap).all(), "the sample ring must hold every sample"
    return out


def _bucket_run(eng, kw, w, n, cap):
    """(records, past-end indices, percentiles or None, launch info, status) of one bucketed run"""
    eng.set_buckets(w, n)
    eng.set_bucket_percentiles(cap)
    try:
        eng.run(engine.make_params(**kw))
        info = eng.last_launch()
        got, past = eng.read_buckets(n)
        pct = eng.read_bucket_percentiles(n) if cap else None
        st = eng.read_outputs()["summaries"]["status"].copy()
    finally:
        eng.set_bucket_percentiles(0)
        eng.set_buckets(0.0, 0)
    return got, past, pct, info, st


def _check_pct(model, rec_out, got, pct, w, n, replicas, rec_base=0):
    """pct[r] == _percentile_sorted of every bucket of replica r's samples (replica r - rec_base of the record-mode
    output), bitwise; returns the number of buckets checked"""
    rows = B.rows(model)
    checked = 0
    for r in replicas:
        per_sink, _ = results.demultiplex(model, rec_out, r - rec_base)
        for b, ent in enumerate(rows):
            sm = per_sink[ent]
            t = np.asarray(sm["completion_ns"] if sm is not None else [], np.int64)
            v = np.asarray(sm["latency_s"] if sm is not None else [], np.float64)
            slot = np.minimum(B.bucket_index(t, w), n)
            assert (np.bincount(slot, minlength=n + 1) == got[r, b]["count"]).all(), (r, b)
            cuts = np.flatnonzero(np.diff(slot)) + 1
            for ks, vs in zip(np.split(slot, cuts), np.split(v, cuts)):
                if not len(ks):
                    continue
                s = sorted(float(x) for x in vs)
                want = [_percentile_sorted(s, 0.50), _percentile_sorted(s, 0.99)]
                assert _bits(pct[r, b, ks[0]]).tolist() == _bits(want).tolist(), (r, b, ks[0], pct[r, b, ks[0]], want)
                checked += 1
    return checked


def _roundtrip(eng, model, kw, w, n, *, sample_cap, record_cap=0, replicas=None):
    """a percentile run, its records against the same run without percentiles, its percentiles against record mode"""
    eng.upload(model)
    got, past, pct, info, st = _bucket_run(eng, kw, w, n, CAP)
    assert not (st & A.HS_ST_BUCKET_OVERFLOW).any()
    plain, past0, _, info0, st0 = _bucket_run(eng, kw, w, n, 0)
    assert got.tobytes() == plain.tobytes() and past.tobytes() == past0.tobytes() and st.tobytes() == st0.tobytes()
    assert info0["flags"] == info["flags"] & ~(LF_BUCKET_PCT if info["engine"] == 2 else WF_BUCKET_PCT)
    rec = _record_run(eng, kw, sample_cap, record_cap)
    reps = replicas if replicas is not None else range(kw["n_replicas"])
    return _check_pct(model, rec, got, pct, w, n, reps), info


# ---- the lane engine: its six percentile kernels ------------------------------------------------------------------

@pytest.mark.parametrize("hash_", [0, 1])
@pytest.mark.parametrize("case", ["simple", "general", "profile"])
def test_lane_kernels(eng, case, hash_):
    if case == "simple":
        model, kw, fl = hs.mm1(), dict(seed=7, end_ns=30 * 10**9), LF_SIMPLE
    elif case == "general":
        model, kw, z = G.load("philox_mmc4"); kw.pop("rid_base"); fl = 0
    else:
        model, kw, z = G.load("philox_spike_poisson_mm1"); kw.pop("rid_base"); fl = LF_PROFILE
    end_s = kw["end_ns"] / 1e9
    w = 0.25 if case != "general" else 0.1
    n = int(end_s / w) + 2
    kw = dict(kw, n_replicas=1317, rid_stride=1, engine=2, flags=hash_)
    checked, info = _roundtrip(eng, model, kw, w, n, sample_cap=int(end_s * 60) + 256)
    assert info["engine"] == 2 and info["flags"] == LF_BUCKETS | LF_BUCKET_PCT | fl | hash_, info
    assert checked > 1317 * 5


# ---- the thread and warp engines ------------------------------------------------------------------------------------

def _fixture(name):
    model, kw, z = G.load(name)
    kw.pop("rid_base")
    return model, kw


GENERAL = {"probe": lambda: _fixture("philox_probe_mm1"), "fault": lambda: _fixture("fault_tandem_probe_crash_middle")}


@pytest.mark.parametrize("hash_", [0, 1])
@pytest.mark.parametrize("geometry", [("thread_wide", 1024), ("thread", 2048), ("thread_heaptop", 16384), ("warp", 1024)])
@pytest.mark.parametrize("case", ["probe", "fault"])
def test_general_kernels(eng, case, geometry, hash_):
    kind, n_rep = geometry
    model, kw = GENERAL[case]()
    if n_rep >= 2048:
        kw = dict(kw, end_ns=min(kw["end_ns"], 5 * 10**9))
    end_s = kw["end_ns"] / 1e9
    w = 0.1
    n = int(end_s / w) + 2
    faults = bool(model.ids_of(A.HS_ENT_FAULT))
    kw = dict(kw, n_replicas=n_rep, rid_stride=1, engine=1 if kind == "warp" else 3, flags=hash_)
    smp = int(hs.lowering.source_rate_bound(model) * end_s * 1.5) + 256
    multi = len(B.rows(model)) > 1
    picked = range(0, n_rep, 1 if n_rep <= 2048 else 7)
    checked, info = _roundtrip(eng, model, kw, w, n, sample_cap=smp, record_cap=smp * 16 if multi else 0, replicas=picked)
    fl = WF_BUCKETS | WF_BUCKET_PCT | WF_PROFILE | hash_ | (WF_FAULTS if faults else 0) | \
        (WF_HEAPTOP if kind == "thread_heaptop" else 0)
    assert info["flags"] == fl, info
    assert info["kernel"] == ("warp" if kind == "warp" else "thread_wide" if kind == "thread_wide" else "thread"), info
    assert checked > len(picked)


# ---- windows, overflow, totals --------------------------------------------------------------------------------------

@pytest.mark.parametrize("e", [2, 3, 1])
def test_windows_cut_mid_bucket(eng, e):
    model = hs.mm1(8.0, 0.1) if e == 2 else hs.lb_round_robin(8, 64.0)
    kw = dict(seed=11, end_ns=6 * 10**9, n_replicas=512, rid_stride=1, engine=e)
    w, n = 0.4, 16
    eng.upload(model)
    whole, past0, pct0, _, _ = _bucket_run(eng, kw, w, n, CAP)
    eng.set_buckets(w, n)
    eng.set_bucket_percentiles(CAP)
    try:
        for j, cut in enumerate([0.55e9, 1.3e9, 2.0e9, 4.77e9, -1]):
            eng.run(engine.make_params(window_end_ns=int(cut), resume=int(j > 0), **kw))
        got, past = eng.read_buckets(n)
        pct = eng.read_bucket_percentiles(n)
        with pytest.raises(engine.EngineError, match="sample capacity"):
            eng.set_bucket_percentiles(CAP * 2)
            eng.run(engine.make_params(window_end_ns=-1, resume=1, **kw))
    finally:
        eng.set_bucket_percentiles(0)
        eng.set_buckets(0.0, 0)
    assert got.tobytes() == whole.tobytes() and past.tobytes() == past0.tobytes()
    assert pct.tobytes() == pct0.tobytes()


def test_overflow_status_and_growth(eng):
    """a capacity below a bucket's count: NaN and HS_ST_BUCKET_OVERFLOW for that replica, exact counts; run_ensemble
    grows the capacity and returns what an adequate one gives; a windowed run raises, naming the capacity"""
    model = hs.mm1(40.0, 0.02)
    kw = dict(seed=5, end_ns=3 * 10**9, n_replicas=256, rid_stride=1, engine=2)
    w, n = 0.5, 7
    eng.upload(model)
    got, _, pct, _, st = _bucket_run(eng, kw, w, n, 8)
    over = got["count"] > 8
    assert over.any()
    assert ((st & A.HS_ST_BUCKET_OVERFLOW) != 0).tolist() == over.any(axis=(1, 2)).tolist()
    assert np.isnan(pct[over]).all() and not np.isnan(pct[~over]).any()
    full, _, pct_full, _, st_full = _bucket_run(eng, kw, w, n, 64)
    assert full.tobytes() == got.tobytes() and not (st_full & A.HS_ST_BUCKET_OVERFLOW).any()
    assert pct[~over].tobytes() == pct_full[~over].tobytes()

    srv = hs.Server("srv", service_time=hs.ExponentialLatency(0.02)); snk = hs.Sink("snk"); srv.downstream = snk
    sim = hs.Simulation(sources=[hs.Source.poisson(rate=40.0, target=srv, name="src")], entities=[srv, snk],
                        end_time=hs.Instant.from_seconds(3.0), seed=5)
    out = sim.run_ensemble(256, rid_stride=1, buckets=(w, n), bucket_percentiles=True, bucket_sample_cap=4)
    need = B.sample_cap_needed(out["buckets"])
    assert out["bucket_sample_cap"] == need > 4 and not (out["status"] & A.HS_ST_BUCKET_OVERFLOW).any()
    ok = sim.run_ensemble(256, rid_stride=1, buckets=(w, n), bucket_percentiles=True, bucket_sample_cap=4 * need)
    assert out["bucket_percentiles"].tobytes() == ok["bucket_percentiles"].tobytes()
    assert out["buckets"].tobytes() == ok["buckets"].tobytes()
    with pytest.raises(EnsembleStatusError, match="bucket_sample_cap="):
        sim.run_ensemble(256, rid_stride=1, buckets=(w, n), bucket_percentiles=True, bucket_sample_cap=4,
                         window_end_s=1.7)
    ign = sim.run_ensemble(256, rid_stride=1, buckets=(w, n), bucket_percentiles=True, bucket_sample_cap=4,
                           on_overflow="ignore")
    assert (ign["status"] & A.HS_ST_BUCKET_OVERFLOW).any() and np.isnan(ign["bucket_percentiles"]).any()


def test_cell_totals_of_a_sweep(eng):
    """the M/M/c sweep's per-cell percentile totals: the numpy restatement bit for bit, the same bits on a repeat run and
    on the thread engine; the record totals are those of the run without percentiles"""
    model = hs.mmc_sweep(cs=range(1, 5), rhos=(0.5, 0.9))
    n_cells = model.n_cells
    rpc = 300
    kw = dict(seed=21, end_ns=4 * 10**9, n_replicas=n_cells * rpc, replicas_per_cell=rpc, rid_stride=1)
    w, n = 0.25, 17
    eng.upload(model)
    outs = []
    for e, cap in ((2, CAP), (2, CAP), (3, CAP), (2, 0)):
        eng.set_buckets(w, n)
        eng.set_bucket_percentiles(cap)
        try:
            eng.run(engine.make_params(engine=e, **kw))
            got, _ = eng.read_buckets(n)
            tot = eng.read_bucket_totals(n_cells, got.shape[1], n)
            pct = eng.read_bucket_percentiles(n) if cap else None
            ptot = eng.read_bucket_percentile_totals(n_cells, got.shape[1], n) if cap else None
        finally:
            eng.set_bucket_percentiles(0)
            eng.set_buckets(0.0, 0)
        outs.append((got, tot, pct, ptot))
    got, tot, pct, ptot = outs[0]
    want = B.cell_percentile_totals_reference(got, pct, n_cells, replicas_per_cell=rpc)
    assert ptot.tobytes() == want.tobytes()
    assert (ptot["p99_sum"] >= ptot["p50_sum"]).all() and (ptot["p50_sum"] > 0).any()
    for o in outs[1:3]:
        assert o[0].tobytes() == got.tobytes() and o[2].tobytes() == pct.tobytes() and o[3].tobytes() == ptot.tobytes()
    assert outs[3][0].tobytes() == got.tobytes() and outs[3][1].tobytes() == tot.tobytes()
    assert tot.tobytes() == B.cell_totals_reference(got, n_cells, replicas_per_cell=rpc).tobytes()


# ---- the Python API ------------------------------------------------------------------------------------------------

def test_api_trackers_and_probe():
    """trackers, a ThroughputTracker and a Probe: bucketed_data's p50s / p99s equal Data.bucket(w) of what a
    record-mode run writes back"""
    def build():
        lat, tp = hs.LatencyTracker("lat"), hs.ThroughputTracker("tp")
        s1 = hs.Server("s1", service_time=hs.ExponentialLatency(0.08)); s1.downstream = lat
        s2 = hs.Server("s2", service_time=hs.ExponentialLatency(0.05)); s2.downstream = tp
        lb = hs.LoadBalancer("lb", backends=[s1, s2], strategy=hs.RoundRobin())
        probe, data = hs.Probe.on(s1, "depth", interval=0.1)
        src = hs.Source.poisson(rate=18.0, target=lb, name="src")
        sim = hs.Simulation(sources=[src], entities=[lb, s1, s2, lat, tp], probes=[probe],
                            end_time=hs.Instant.from_seconds(8.0), seed=5)
        return sim, (lat, tp, probe, data)
    w, n = 0.5, 17
    sim, objs = build()
    out = sim.run_ensemble(256, rid_stride=1, buckets=(w, n), bucket_percentiles=True)
    assert out["bucket_percentiles"].shape == (256, 3, n + 1, 2) and out["bucket_sample_cap"] == 64
    assert out["bucket_percentile_totals"].shape == (1, 3, n + 1)
    sim2, objs2 = build()
    rec = sim2.run_ensemble(256, rid_stride=1, sample_cap=2048, record_cap=16384)
    for r in range(0, 256, 17):
        results.write_back(sim2.model, sim2.objects, rec, r, hs.Instant)
        for o, o2 in zip(objs, objs2):
            want = (o2 if isinstance(o2, hs.Data) else o2.data_sink if hasattr(o2, "data_sink") else o2.data).bucket(w)
            got = B.bucketed_data(out, o, r)
            for f in ("times", "counts", "sums", "means", "maxes"):
                assert getattr(got, f)() == getattr(want, f)(), (r, f, o)
            assert _bits(got.p50s()).tolist() == _bits(want.p50s()).tolist(), (r, o)
            assert _bits(got.p99s()).tolist() == _bits(want.p99s()).tolist(), (r, o)
    assert all(x == 1.0 for x in B.bucketed_data(out, objs[1], 3).p99s())
    # without the option nothing changes: NaN percentiles, the same records
    plain = build()[0].run_ensemble(256, rid_stride=1, buckets=(w, n))
    assert "bucket_percentiles" not in plain and plain["buckets"].tobytes() == out["buckets"].tobytes()
    assert plain["bucket_totals"].tobytes() == out["bucket_totals"].tobytes()


def test_run_replicas_passes_percentiles_through():
    def build():
        return hs.Simulation(sources=[hs.Source.poisson(rate=8.0, target=srv, name="src")], entities=[srv, snk],
                             end_time=hs.Instant.from_seconds(5.0))
    srv = hs.Server("srv", service_time=hs.ExponentialLatency(0.1)); snk = hs.Sink("snk"); srv.downstream = snk
    res = hs.ParallelRunner().run_replicas(build, 64, base_seed=7, buckets=(0.5, 11), bucket_percentiles=True,
                                           bucket_sample_cap=32)
    got = res.raw["bucket_percentiles"]
    assert got.shape == (64, 1, 12, 2) and res.raw["bucket_sample_cap"] == 32
    want = build().run_ensemble(64, seed=7, seed_stride=1, rid_stride=0, buckets=(0.5, 11), bucket_percentiles=True,
                                bucket_sample_cap=32)
    assert got.tobytes() == want["bucket_percentiles"].tobytes()


def test_configs1_at_full_size(eng):
    """configs[1] (65 536 M/M/1 replicas, 100 s, w = 1 s) on the lane engine's M/M/1 percentile kernel; 64 replicas
    checked against record mode"""
    model = hs.mm1(8.0, 0.1)
    w, n = 1.0, 101
    kw = dict(seed=1234, end_ns=100 * 10**9, rid_stride=1, flags=1)
    eng.upload(model)
    got, past, pct, info, st = _bucket_run(eng, dict(kw, n_replicas=65536), w, n, 64)
    assert info["engine"] == 2 and info["flags"] == LF_BUCKETS | LF_BUCKET_PCT | LF_SIMPLE | LF_HASH
    assert not (st & A.HS_ST_BUCKET_OVERFLOW).any()
    eng.set_buckets(w, n)
    eng.set_bucket_percentiles(64)
    try:
        eng.run(engine.make_params(**dict(kw, n_replicas=65536)))
        ptot = eng.read_bucket_percentile_totals(1, 1, n)
    finally:
        eng.set_bucket_percentiles(0)
        eng.set_buckets(0.0, 0)
    assert ptot.tobytes() == B.cell_percentile_totals_reference(got, pct, 1).tobytes()
    pick = list(range(65536 - 64, 65536))
    rec = _record_run(eng, dict(kw, n_replicas=64, replica_index_base=pick[0]), sample_cap=1200, record_cap=0)
    assert _check_pct(model, rec, got, pct, w, n, pick, rec_base=pick[0]) > 64 * 90    # about 100 buckets each


def test_refusals(eng):
    eng.upload(hs.mm1())
    kw = dict(seed=1, end_ns=10**9, n_replicas=64)
    try:
        eng.set_bucket_percentiles(64)
        with pytest.raises(engine.EngineError, match="need time buckets"):
            eng.run(engine.make_params(**kw))
        eng.set_buckets(0.1, 11)
        eng.run(engine.make_params(window_end_ns=5 * 10**8, **kw))
        eng.set_bucket_percentiles(32)
        with pytest.raises(engine.EngineError, match="sample capacity"):
            eng.run(engine.make_params(resume=1, **kw))
        eng.set_bucket_percentiles(1 << 20)                              # 65 536 x 2^20 x 8 B of value buffers
        with pytest.raises(engine.EngineError, match="GB"):
            eng.run(engine.make_params(**dict(kw, n_replicas=65536, end_ns=10**9)))
    finally:
        eng.set_bucket_percentiles(0)
        eng.set_buckets(0.0, 0)
    sim = hs.Simulation(sources=[], entities=[], end_time=hs.Instant.from_seconds(1.0), _lowered=(hs.mm1(), [], hs.Instant))
    with pytest.raises(ValueError, match="needs buckets"):
        sim.run_ensemble(4, bucket_percentiles=True)
