"""Time buckets on the device (hs_set_buckets, Simulation.run_ensemble(buckets=)): every replica's buckets against
Data.bucket(w) of the same replica's complete sample list, taken from a record-mode run of the same seeds on the same
engine (counts exact, sums and maxes bitwise).  Every run asserts through Engine.last_launch() the bucket
instantiation it meant to reach: the lane engine's six (general, profile and M/M/1 chains, with and without the order
hash), the warp engine's four and the thread engine's twelve (wide, plain and HEAPTOP, with and without faults and
hash).  Also: runs cut into windows mid-bucket, a constant-rate grid whose samples sit on bucket boundaries, a fault
schedule, trackers and a Probe through the Python API, a sample of configs[1] at full size and the per-cell totals."""
import math

import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
from happysim_b200 import _abi as A, buckets as B, engine, results

pytestmark = pytest.mark.gpu

LF_HASH, LF_PROFILE, LF_SIMPLE, LF_BUCKETS = 1, 4, 8, 16
WF_HASH, WF_HEAPTOP, WF_FAULTS, WF_BUCKETS, WF_PROFILE = 1, 8, 32, 64, 4


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


def _record_run(eng, kw, sample_cap, record_cap):
    eng.set_buckets(0.0, 0)
    eng.run(engine.make_params(sample_cap=sample_cap, record_cap=record_cap, **kw))
    out = eng.read_outputs()
    assert (out["summaries"]["n_sink_samples"] <= sample_cap).all(), "the sample ring must hold every sample"
    assert (out["summaries"]["events_processed"] <= max(record_cap, 1)).all() or record_cap == 0
    return out


def _bucket_run(eng, kw, w, n):
    eng.set_buckets(w, n)
    try:
        eng.run(engine.make_params(**kw))
        info = eng.last_launch()
        got, past = eng.read_buckets(n)
    finally:
        eng.set_buckets(0.0, 0)
    return got, past, info


def _check_replicas(model, rec_out, got, past, w, n, replicas=None, rec_base=0):
    """got[r] == the records Data.bucket(w) implies for replica r's samples, replica r - rec_base of the record-mode
    output"""
    rows = B.rows(model)
    assert got.shape[1] == len(rows)
    sums = B.replica_sums(got)
    n_checked = 0
    for r in (replicas if replicas is not None else range(got.shape[0])):
        per_sink, _ = results.demultiplex(model, rec_out, r - rec_base)
        for b, ent in enumerate(rows):
            sm = per_sink[ent]
            t = np.asarray(sm["completion_ns"] if sm is not None else [], np.int64)
            v = np.asarray(sm["latency_s"] if sm is not None else [], np.float64)
            k = B.bucket_index(t, w)
            slot = np.minimum(k, n)
            assert (np.bincount(slot, minlength=n + 1) == got[r, b]["count"]).all(), (r, b)
            if len(t) and k[-1] >= n:
                assert past[r, b] == k[-1] and (k[k >= n] == k[-1]).all()
            cuts = np.flatnonzero(np.diff(slot)) + 1
            for ks, vs in zip(np.split(slot, cuts), np.split(v, cuts)):
                if not len(ks):
                    continue
                vals = [float(x) for x in vs]
                assert sums[r, b, ks[0]] == sum(vals), (r, b, ks[0])
                assert got[r, b, ks[0]]["max"] == max(vals), (r, b, ks[0])
            n_checked += len(t)
    return n_checked


def _roundtrip(eng, model, kw, w, n, *, sample_cap, record_cap=0, expect_engine, expect_flags):
    eng.upload(model)
    got, past, info = _bucket_run(eng, kw, w, n)
    assert info["engine"] == expect_engine and info["flags"] == expect_flags, info
    rec = _record_run(eng, kw, sample_cap, record_cap)
    assert rec["summaries"]["events_processed"].tolist() == eng.read_outputs()["summaries"]["events_processed"].tolist()
    return _check_replicas(model, rec, got, past, w, n), got, info


# ---- the lane engine: its six bucket kernels ----------------------------------------------------------------------

@pytest.mark.parametrize("hash_", [0, 1])
@pytest.mark.parametrize("case", ["simple", "general", "profile", "spike"])
def test_lane_kernels(eng, case, hash_):
    if case == "simple":
        model, kw, fl = hs.mm1(), dict(seed=7, end_ns=30 * 10**9), LF_SIMPLE
    elif case == "general":
        model, kw, z = G.load("philox_mmc4"); kw.pop("rid_base"); fl = 0
    elif case == "profile":
        model, kw, z = G.load("philox_ramp_poisson_mm1"); kw.pop("rid_base"); fl = LF_PROFILE
    else:
        model, kw, z = G.load("philox_spike_poisson_mm1"); kw.pop("rid_base"); fl = LF_PROFILE
    end_s = kw["end_ns"] / 1e9
    w = 0.25 if case != "general" else 0.1
    n = int(end_s / w) + 2
    kw = dict(kw, n_replicas=1317, rid_stride=1, engine=2, flags=hash_)
    checked, got, info = _roundtrip(eng, model, kw, w, n, sample_cap=int(end_s * 60) + 256,
                                    expect_engine=2, expect_flags=LF_BUCKETS | fl | hash_)
    assert checked > 1317 * 10


# ---- the thread and warp engines ------------------------------------------------------------------------------------

def _farm():
    return hs.lb_round_robin(n_servers=16, rate=256.0), dict(seed=3, end_ns=3 * 10**9)


def _fixture(name):
    model, kw, z = G.load(name)
    kw.pop("rid_base")
    return model, kw


GENERAL = {"farm": _farm, "tandem": lambda: _fixture("philox_tandem"), "probe": lambda: _fixture("philox_probe_mm1"),
           "fault": lambda: _fixture("fault_tandem_probe_crash_middle")}


@pytest.mark.parametrize("hash_", [0, 1])
@pytest.mark.parametrize("geometry", [("thread_wide", 1024), ("thread", 2048), ("thread_heaptop", 16384), ("warp", 1024)])
@pytest.mark.parametrize("case", ["farm", "tandem", "probe", "fault"])
def test_general_kernels(eng, case, geometry, hash_):
    kind, n_rep = geometry
    model, kw = GENERAL[case]()
    end_s = kw["end_ns"] / 1e9
    if n_rep >= 2048:
        kw = dict(kw, end_ns=min(kw["end_ns"], 5 * 10**9)); end_s = kw["end_ns"] / 1e9
    w = 0.1
    n = int(end_s / w) + 2
    faults = bool(model.ids_of(A.HS_ENT_FAULT))
    kw = dict(kw, n_replicas=n_rep, rid_stride=1, engine=1 if kind == "warp" else 3, flags=hash_)
    fl = WF_BUCKETS | WF_PROFILE | hash_ | (WF_FAULTS if faults else 0) | (WF_HEAPTOP if kind == "thread_heaptop" else 0)
    eng.upload(model)
    got, past, info = _bucket_run(eng, kw, w, n)
    assert info["flags"] == fl, info
    assert info["kernel"] == ("warp" if kind == "warp" else "thread_wide" if kind == "thread_wide" else "thread"), info
    smp = int(hs.lowering.source_rate_bound(model) * end_s * 1.5) + 256
    multi = len(B.rows(model)) > 1
    rec = _record_run(eng, kw, sample_cap=smp, record_cap=smp * 16 if multi else 0)
    picked = range(0, n_rep, 1 if n_rep <= 2048 else 7)
    assert _check_replicas(model, rec, got, past, w, n, replicas=picked) > len(picked)


def test_fault_empties_buckets(eng):
    """a crashed sink records nothing: the buckets of the crash window are empty in every replica"""
    model, kw = _fixture("fault_mm1_pause_sink")
    flt = model.ids_of(A.HS_ENT_FAULT)
    t0, t1 = sorted(int(model.entities["l0"][i]) for i in flt)[:2]
    w = 0.05
    n = int(kw["end_ns"] / 1e9 / w) + 2
    kw = dict(kw, n_replicas=2048, rid_stride=1)
    eng.upload(model)
    got, past, info = _bucket_run(eng, kw, w, n)
    assert info["flags"] & WF_FAULTS and info["flags"] & WF_BUCKETS
    lo, hi = B.bucket_index(t0, w) + 1, B.bucket_index(t1, w)
    assert hi > lo and got["count"][:, 0, lo:hi].sum() == 0
    assert got["count"][:, 0, :lo].sum() > 0 and got["count"][:, 0, hi + 1:].sum() > 0
    rec = _record_run(eng, kw, sample_cap=4096, record_cap=0)
    _check_replicas(model, rec, got, past, w, n)


def test_grid_samples_on_bucket_boundaries(eng):
    """constant arrivals every 100 ms, constant 100 ms service: every completion lies on a multiple of w = 0.1"""
    model = hs.mm1(rate=10.0, mean_service_s=0.1, poisson=False, exponential=False)
    kw = dict(seed=1, end_ns=20 * 10**9, n_replicas=64, rid_stride=1)
    w, n = 0.1, 202
    for e, kern in ((2, "lane"), (3, "thread_wide"), (1, "warp")):
        eng.upload(model)
        got, past, info = _bucket_run(eng, dict(kw, engine=e), w, n)
        assert info["kernel"] == kern
        rec = _record_run(eng, dict(kw, engine=e), sample_cap=512, record_cap=0)
        t = rec["sink_samples"][0]["completion_ns"][: int(rec["summaries"]["n_sink_samples"][0])]
        assert (t % 100_000_000 == 0).all() and (B.bucket_index(t, w) != t // 100_000_000).any()
        _check_replicas(model, rec, got, past, w, n)


@pytest.mark.parametrize("e", [2, 3, 1])
def test_windows_cut_mid_bucket(eng, e):
    model = hs.mm1(8.0, 0.1) if e == 2 else hs.lb_round_robin(8, 64.0)
    kw = dict(seed=11, end_ns=6 * 10**9, n_replicas=512, rid_stride=1, engine=e)
    w, n = 0.4, 16
    eng.upload(model)
    whole, past0, _ = _bucket_run(eng, kw, w, n)
    eng.set_buckets(w, n)
    try:
        for j, cut in enumerate([0.55e9, 1.3e9, 2.0e9, 4.77e9, -1]):
            eng.run(engine.make_params(window_end_ns=int(cut), resume=int(j > 0), **kw))
            # after every pause the records hold every sample so far: the current buckets were stored at the pause
            mid, _ = eng.read_buckets(n)
            assert (mid["count"].sum(axis=(1, 2)) == eng.read_outputs()["summaries"]["n_sink_samples"]).all(), cut
        got, past = eng.read_buckets(n)
        with pytest.raises(engine.EngineError, match="bucket"):
            eng.set_buckets(w, n + 1)
            eng.run(engine.make_params(window_end_ns=-1, resume=1, **kw))
    finally:
        eng.set_buckets(0.0, 0)
    assert got.tobytes() == whole.tobytes() and past.tobytes() == past0.tobytes()


def test_refusals(eng):
    eng.upload(hs.mm1())
    kw = dict(seed=1, end_ns=10**9, n_replicas=64)
    try:
        eng.set_buckets(0.1, 11)
        with pytest.raises(engine.EngineError, match="recorder"):
            eng.run(engine.make_params(sample_cap=16, **kw))
        eng.set_buckets(0.1, 10)
        with pytest.raises(engine.EngineError, match="end time"):
            eng.run(engine.make_params(**kw))
        with pytest.raises(engine.EngineError):
            eng.set_buckets(-1.0, 10)
        eng.set_buckets(0.1, 11)
        with pytest.raises(engine.EngineError, match="linked"):          # a window of a linked partition
            eng.run(engine.make_params(flags=A.HS_RUN_LINKED, **kw))
        eng.set_buckets(1e-6, 1 << 24)                                    # 65 536 x (2^24 + 1) x 32 B: more than the device has
        with pytest.raises(engine.EngineError, match="GB"):
            eng.run(engine.make_params(**dict(kw, n_replicas=65536)))
    finally:
        eng.set_buckets(0.0, 0)
    sim = hs.Simulation(sources=[], entities=[], end_time=hs.Instant.from_seconds(1.0), _lowered=(hs.mm1(), [], hs.Instant))
    with pytest.raises(ValueError):
        sim.run_ensemble(4, buckets=(0.1, 5))


def test_api_trackers_and_probe():
    """Simulation.run_ensemble(buckets=) on a farm whose backends feed a LatencyTracker and a ThroughputTracker, with a
    Probe on a server: buckets.bucketed_data(out, obj, r) equals Data.bucket(w) of what a record-mode run writes back"""
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
    out = sim.run_ensemble(256, rid_stride=1, buckets=(w, n))
    assert len(out["bucket_rows"]) == 3
    sim2, objs2 = build()
    rec = sim2.run_ensemble(256, rid_stride=1, sample_cap=2048, record_cap=16384)
    for r in range(0, 256, 17):
        results.write_back(sim2.model, sim2.objects, rec, r, hs.Instant)
        for o, o2 in zip(objs, objs2):
            want = (o2 if isinstance(o2, hs.Data) else o2.data_sink if hasattr(o2, "data_sink") else o2.data).bucket(w)
            got = B.bucketed_data(out, o, r)
            for f in ("times", "counts", "sums", "means", "maxes"):
                assert getattr(got, f)() == getattr(want, f)(), (r, f, o)
            assert all(math.isnan(x) for x in got.p50s())


def test_run_replicas_passes_buckets_through():
    """ParallelRunner.run_replicas(..., buckets=) is run_ensemble(..., buckets=) with seeds base_seed + i"""
    def build():
        return hs.Simulation(sources=[hs.Source.poisson(rate=8.0, target=srv, name="src")], entities=[srv, snk],
                             end_time=hs.Instant.from_seconds(5.0))
    srv = hs.Server("srv", service_time=hs.ExponentialLatency(0.1)); snk = hs.Sink("snk"); srv.downstream = snk
    res = hs.ParallelRunner().run_replicas(build, 64, base_seed=7, buckets=(0.5, 11))
    got = res.raw["buckets"]
    assert got.shape == (64, 1, 12) and res.raw["bucket_objects"] == [snk]
    want = build().run_ensemble(64, seed=7, seed_stride=1, rid_stride=0, buckets=(0.5, 11))
    assert got.tobytes() == want["buckets"].tobytes() and int(got["count"].sum()) > 64 * 20


def test_configs1_sample_at_full_size(eng):
    """configs[1] (65 536 M/M/1 replicas) bucketed on the lane engine's M/M/1 kernel; 64 replicas checked"""
    model = hs.mm1(8.0, 0.1)
    w, n = 1.0, 101
    kw = dict(seed=1234, end_ns=100 * 10**9, rid_stride=1)
    eng.upload(model)
    got, past, info = _bucket_run(eng, dict(kw, n_replicas=65536), w, n)
    assert info["engine"] == 2 and info["flags"] == LF_BUCKETS | LF_SIMPLE | LF_HASH
    # the plain ensemble's totals (one cell, slices of 256 replicas): the documented order bit for bit
    tot = eng.read_bucket_totals(1, 1, n)
    assert tot.tobytes() == B.cell_totals_reference(got, 1).tobytes()
    assert (tot[0]["count"] == got["count"].sum(0)).all()
    pick = list(range(65536 - 64, 65536))
    rec = _record_run(eng, dict(kw, n_replicas=64, replica_index_base=pick[0]), sample_cap=1200, record_cap=0)
    assert _check_replicas(model, rec, got, past, w, n, replicas=pick, rec_base=pick[0]) > 64 * 600


def test_cell_totals_of_a_sweep(eng):
    """the M/M/c sweep's per-cell totals: the numpy restatement of the documented order bit for bit, counts and maxes
    against the per-replica records, the same bits on a repeat run and on another engine"""
    model = hs.mmc_sweep(cs=range(1, 5), rhos=(0.5, 0.9))
    n_cells = model.n_cells
    rpc = 300
    kw = dict(seed=21, end_ns=4 * 10**9, n_replicas=n_cells * rpc, replicas_per_cell=rpc, rid_stride=1)
    w, n = 0.25, 17
    eng.upload(model)
    outs = []
    for e in (2, 2, 3):
        eng.set_buckets(w, n)
        try:
            eng.run(engine.make_params(engine=e, **kw))
            got, _ = eng.read_buckets(n)
            tot = eng.read_bucket_totals(n_cells, got.shape[1], n)
        finally:
            eng.set_buckets(0.0, 0)
        outs.append((got, tot))
    got, tot = outs[0]
    want = B.cell_totals_reference(got, n_cells, replicas_per_cell=rpc)
    assert tot.tobytes() == want.tobytes()
    cell = np.arange(kw["n_replicas"]) // rpc
    for c in range(n_cells):
        sel = got[cell == c]
        assert (tot[c]["count"] == sel["count"].sum(0)).all()
        assert (tot[c]["replicas"] == (sel["count"] > 0).sum(0)).all()
        mx = np.where(sel["count"] > 0, sel["max"], -np.inf).max(0)
        assert (tot[c]["max"] == mx).all()
        s = B.replica_sums(sel)
        exact = np.array([[math.fsum(s[:, i, j][sel["count"][:, i, j] > 0]) for j in range(n + 1)] for i in range(s.shape[1])])
        assert (np.abs(tot[c]["sum"] - exact) <= 2 * rpc * np.finfo(float).eps * np.abs(exact) + 1e-300).all()
    assert outs[1][1].tobytes() == tot.tobytes()
    assert outs[2][0].tobytes() == got.tobytes() and outs[2][1].tobytes() == tot.tobytes()
