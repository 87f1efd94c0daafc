"""Node faults without a GPU: the C-ABI's validation of FAULT rows, the lowering of the reference's and the mirror's
FaultSchedule to identical rows, and the errors the reference raises."""
import ctypes as C

import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
from happysim_b200 import _abi as A, engine, lowering


def _validate(model):
    L = engine.load_library()
    return L.hs_model_validate(C.byref(model.desc()))


def _mm1_with(rows):
    m = hs.mm1()
    m.entities = np.array(list(m.entities.tolist()) + rows, dtype=A.ENTITY_DTYPE)
    m.names = list(m.names) + [f"f{i}" for i in range(len(rows))]
    return m


def test_validate_accepts_a_fault_row():
    assert _validate(_mm1_with([(A.HS_ENT_FAULT, 1, 0, 1, 0, 1, 10**9, 0.0, 0.0)])) == 0


@pytest.mark.parametrize("row", [
    (A.HS_ENT_FAULT, 7, 0, 1, 0, 1, 10**9, 0.0, 0.0),          # target out of range
    (A.HS_ENT_FAULT, -1, 0, 1, 0, 1, 10**9, 0.0, 0.0),
    (A.HS_ENT_FAULT, 3, 0, 1, 0, 1, 10**9, 0.0, 0.0),          # targets a FAULT row (itself)
    (A.HS_ENT_FAULT, 1, 0, 1, 0, 1, -1, 0.0, 0.0),             # negative time
    (A.HS_ENT_FAULT, 1, 0, 2, 0, 1, 10**9, 0.0, 0.0),          # bad action
])
def test_validate_rejects_bad_fault_rows(row):
    assert _validate(_mm1_with([row])) == A.HS_ERR_INVALID


def test_validate_rejects_a_fault_on_a_probe_measure_row():
    b = hs.ModelBuilder()
    src = b.source(rate=4.0); srv = b.server(); snk = b.sink()
    b.set_target(src, srv); b.set_target(srv, snk)
    _, pid = b.probe(target=srv, metric="depth", interval_s=0.5)
    b.fault(target=pid, time_ns=10**9, crash=True, sort_index=2)
    assert _validate(b.build()) == A.HS_ERR_INVALID


def test_validate_rejects_faults_with_remote_rows_and_rows_after_faults():
    b = hs.ModelBuilder()
    src = b.source(rate=4.0); srv = b.server()
    rem = b.remote(link=0, dest_entity=0)
    b.set_target(src, srv); b.set_target(srv, rem)
    b.fault(target=srv, time_ns=10**9, crash=True, sort_index=1)
    m = b.build(); m.outbox_cap = 16
    assert _validate(m) == A.HS_ERR_INVALID
    m = _mm1_with([(A.HS_ENT_FAULT, 1, 0, 1, 0, 1, 10**9, 0.0, 0.0), (A.HS_ENT_SINK, -1, 0, 0, 0, 0, -1, 0.0, 0.0)])
    assert _validate(m) == A.HS_ERR_INVALID


def _mirror_sim(schedule):
    sink = hs.Sink()
    srv = hs.Server("Server", service_time=hs.ExponentialLatency(0.1), downstream=sink)
    src = hs.Source.poisson(rate=8.0, target=srv, name="Source")
    return hs.Simulation(sources=[src], entities=[srv, sink], end_time=hs.Instant.from_seconds(10.0),
                         fault_schedule=schedule)


def test_mirror_lowering_matches_the_fixture_rows():
    """The mirror's schedule lowers to the FAULT rows the reference's generated events gave (times, indices)."""
    fs = hs.api.FaultSchedule()
    fs.add(hs.api.CrashNode("Server", at=3.0, restart_at=6.5))
    sim = _mirror_sim(fs)
    model, _, z = G.load("fault_mm1_crash_restart")
    fr = model.ids_of(A.HS_ENT_FAULT)
    assert sim.model.entities[sim.model.ids_of(A.HS_ENT_FAULT)].tobytes() == model.entities[fr].tobytes()


def test_unknown_name_raises_key_error():
    fs = hs.api.FaultSchedule()
    fs.add(hs.api.CrashNode("nope", at=1.0))
    with pytest.raises(KeyError):
        _mirror_sim(fs)


def test_other_fault_classes_are_unsupported():
    class MyFault:
        entity_name = "Server"

        def generate_events(self, ctx):
            return []
    fs = hs.api.FaultSchedule()
    fs.add(MyFault())
    with pytest.raises(lowering.UnsupportedModelError, match="MyFault"):
        _mirror_sim(fs)


def test_cancellation_is_read_at_run_time():
    fs = hs.api.FaultSchedule()
    h = fs.add(hs.api.CrashNode("Server", at=3.0, restart_at=6.5))
    sim = _mirror_sim(fs)
    h.cancel()
    lowering.refresh_fault_cancellation(sim.model)
    assert (sim.model.entities["i2"][sim.model.ids_of(A.HS_ENT_FAULT)] == 1).all()
    assert fs.stats.faults_cancelled == 1 and fs.stats.faults_scheduled == 1


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
def test_reference_schedule_lowers_like_the_mirror():
    ref = G.import_reference()
    from happysimulator import faults as F
    fs = F.FaultSchedule()
    fs.add(F.CrashNode("Server", at=3.0, restart_at=6.5))
    fs.add(F.PauseNode("Sink", start=1.0, end=2.0))
    mfs = hs.api.FaultSchedule()
    mfs.add(hs.api.CrashNode("Server", at=3.0, restart_at=6.5))
    mfs.add(hs.api.PauseNode("Sink", start=1.0, end=2.0))
    sim = _mirror_sim(mfs)
    rsink = ref.Sink("Sink")
    rsrv = ref.Server("Server", service_time=ref.ExponentialLatency(0.1), downstream=rsink)
    rsrc = ref.Source.poisson(rate=8.0, target=rsrv, name="Source")
    rsim = ref.Simulation(sources=[rsrc], entities=[rsrv, rsink], end_time=ref.Instant.from_seconds(10.0), fault_schedule=fs)
    rm, _ = lowering.lower(rsim._sources, rsim._entities, fault_schedule=fs)
    a, b = rm.entities[rm.ids_of(A.HS_ENT_FAULT)], sim.model.entities[sim.model.ids_of(A.HS_ENT_FAULT)]
    assert a.tobytes() == b.tobytes()


# ---- the fault oracle (tests/layered_oracle.c) against the reference ----------------------------------------------------
import layered_oracle_lib as LO  # noqa: E402


def _check_ref(ref, got, r=0):
    s, ws = got["summaries"][r], ref["summaries"][0]
    for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
        assert int(s[f]) == int(ws[f]), (f, int(s[f]), int(ws[f]))
    assert got["entity_stats"][r].tobytes() == ref["entity_stats"][0].tobytes(), "entity statistics differ"
    for k in ("records", "sink_samples", "service_samples"):
        n = len(ref[k])
        assert got[k][r][:n].tobytes() == ref[k][:n].tobytes(), f"{k} differ"


@pytest.mark.parametrize("name", G.case_names("fault_"))
def test_fault_oracle_reproduces_reference_fixture(name):
    model, kw, z = G.load(name)
    got = LO.run(model, engine.make_params(n_replicas=1, **G.caps(z), **kw))
    G.check_against(z, got)
    tie = bool(int(got["summaries"]["status"][0]) & A.HS_ST_FAULT_TIE)
    assert tie == name.startswith("fault_tie"), "HS_ST_FAULT_TIE exactly where the reference tied"
    # the reference's own final flags and the events_cancelled its summary reported
    fr = model.ids_of(A.HS_ENT_FAULT)
    assert int(got["entity_stats"][0][fr]["c1"].sum()) == int(z["events_cancelled"])


from random_models import (FAULT_SEEDS_V1, FAULT_SEEDS_V2, fault_schedule, random_fault_case,  # noqa: E402
                           with_faults)

RANDOM_SEEDS = FAULT_SEEDS_V1


def _gen_fault_golden():
    import os
    import sys
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    if d not in sys.path:
        sys.path.insert(0, d)
    import gen_fault_golden as GF
    return GF


def reference_case_kw(version, seed, rid):
    """(model, plan builder for gen_fault_golden.run_case, its kwargs, plan, cancel) of a random faulted model
    (tests/random_models.py:random_fault_case) on replica word ``rid``"""
    model, end_s, plan, cancel, run_seed, _, ex = random_fault_case(version, seed)
    kw = dict(seed=run_seed, rid=rid, end_s=end_s, cancel=cancel, expect_tie="any")
    if version == 1:
        kw.update(sketch_seeds=ex["sketch_seeds"], zipf_s=ex["zipf_s"])
    else:
        kw.update(chash_vnodes=ex["chash_vnodes"], profile_objects=ex["profile_objects"])
    return model, (lambda by, F: fault_schedule(plan, F)), kw, plan, cancel


def _oracle_vs_reference(version, seed):
    GF = _gen_fault_golden()
    model, build, kw, plan, cancel = reference_case_kw(version, seed, seed % 5)
    fm, ref, meta = GF.run_case(model, build, kw)
    assert with_faults(model, plan, cancel).entities.tobytes() == fm.entities.tobytes()
    got = LO.run(fm, engine.make_params(n_replicas=1, seed=kw["seed"], rid_base=seed % 5, end_ns=int(kw["end_s"] * 1e9),
                                        record_cap=len(ref["records"]) + 1, sample_cap=len(ref["sink_samples"]) + 1,
                                        service_cap=len(ref["service_samples"]) + 1))
    _check_ref(ref, got)
    if "sketches" in ref:
        a, b = got["sketches"][:1], ref["sketches"].reshape(1, -1)
        if version == 1:            # TDigest rows carry dead slots (leftovers of merges): compare the live state
            a, b = fm.canonical_sketches(a), fm.canonical_sketches(b)
        assert a.tobytes() == b.tobytes(), "sketch / cache states differ"


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
@pytest.mark.parametrize("seed", RANDOM_SEEDS)
def test_fault_oracle_matches_reference_on_random_models(seed):
    """Seeded random models (tests/random_models.py) with random node-fault schedules: the fault oracle against the
    unmodified reference, run here with the Philox plug-ins."""
    _oracle_vs_reference(1, seed)


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
@pytest.mark.parametrize("seed", FAULT_SEEDS_V2)
def test_fault_oracle_matches_reference_on_random_v2_models(seed):
    """The same for random_model_v2: step profiles (the reference runs the user's StepProfile object) and CachingServer
    farms behind round-robin and consistent-hash load balancers, with their TTL cache states."""
    _oracle_vs_reference(2, seed)


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
@pytest.mark.parametrize("version,seed", [(1, s) for s in FAULT_SEEDS_V1] + [(2, s) for s in FAULT_SEEDS_V2])
def test_with_faults_lowers_like_the_reference_schedule(version, seed):
    """random_models.with_faults (no reference needed, so the GPU tests can use it) gives the rows lowering.fault_events
    gives the reference's own FaultSchedule once its Simulation is built: targets, times, bootstrap sort indices (after
    the sources' and the probes' first ticks), cancelled flags, byte for byte."""
    GF = _gen_fault_golden()
    model, build, kw, plan, cancel = reference_case_kw(version, seed, 0)
    fm = GF.build_case(model, build, kw)[-1]
    got = with_faults(model, plan, cancel)
    assert got.entities.tobytes() == fm.entities.tobytes()
    assert got.n_entities > model.n_entities


# ---- tests/golden/random_fault_models.npz: the reference on the same faulted models, replica word 0 -----------------
import os  # noqa: E402

_RF_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "random_fault_models.npz")
RF = np.load(_RF_PATH) if os.path.exists(_RF_PATH) else None     # None while gen_random_fault_golden.py runs


def random_fault_reference(version, seed):
    """(summary row, entity statistics with the FAULT rows' fired / cancelled counts, sketch or cache state bytes
    (canonical for random_model's sketches), events_cancelled) the reference produced on replica word 0"""
    p = f"v{version}s{seed}_"
    return RF[p + "summary"][0], RF[p + "stats"][0], RF[p + "sketches"], int(RF[p + "cancelled"])


def check_random_fault_reference(fm, version, seed, out, r=0):
    ws, wstats, wsk, cancelled = random_fault_reference(version, seed)
    s = out["summaries"][r]
    for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
        assert int(s[f]) == int(ws[f]), (version, seed, f, int(s[f]), int(ws[f]))
    assert out["entity_stats"][r].tobytes() == wstats.tobytes(), (version, seed, "entity statistics")
    fr = fm.ids_of(A.HS_ENT_FAULT)
    assert int(out["entity_stats"][r][fr]["c1"].sum()) == cancelled
    if len(wsk):
        sk = fm.canonical_sketches(out["sketches"])[r] if version == 1 else out["sketches"][r]
        assert sk.tobytes() == wsk.tobytes(), (version, seed, "sketch / cache states")


def test_random_fault_fixture_covers_every_seed():
    assert RF["seeds_v1"].tolist() == FAULT_SEEDS_V1 and RF["seeds_v2"].tolist() == FAULT_SEEDS_V2


@pytest.mark.parametrize("version,seed", [(1, s) for s in FAULT_SEEDS_V1] + [(2, s) for s in FAULT_SEEDS_V2])
def test_fault_oracle_reproduces_random_fault_fixture(version, seed):
    model, end_s, plan, cancel, run_seed, what, _ = random_fault_case(version, seed)
    fm = with_faults(model, plan, cancel)
    got = LO.run(fm, engine.make_params(n_replicas=1, seed=run_seed, end_ns=int(end_s * 1e9)))
    check_random_fault_reference(fm, version, seed, got)


# ---- results.demultiplex: samples of several collectors when a crashed sink drops requests --------------------------
def _multi_collector_cases():
    out = []
    for version, seeds in ((1, range(max(FAULT_SEEDS_V1) + 1)), (2, FAULT_SEEDS_V2)):
        for seed in seeds:
            model, end_s, plan, cancel, run_seed, _, _ = random_fault_case(version, seed)
            if len(model.ids_of(A.HS_ENT_SINK)) + len(model.ids_of(A.HS_ENT_PROBE)) > 1:
                out.append((version, seed))
    return out


def _dropped_by_replay(fm, rec):
    """the REQ_SINK records popped while their sink was crashed, replaying the FAULT records one by one"""
    E = fm.entities
    crashed, out = {}, np.zeros(len(rec), bool)
    for j, (k, e) in enumerate(zip(rec["kind"].tolist(), rec["entity"].tolist())):
        if k == A.HS_EV_FAULT:
            crashed[int(E["target"][e])] = int(E["i1"][e])
        elif k == A.HS_EV_REQ_SINK:
            out[j] = bool(crashed.get(e, 0))
    return out


@pytest.mark.parametrize("version,seed", _multi_collector_cases())
def test_demultiplex_leaves_out_requests_a_crashed_sink_dropped(version, seed):
    """With several Sinks / Probes, results.demultiplex tells their samples apart by the REQ_SINK / PROBE event records.
    A request that reaches a crashed sink is recorded and counted but leaves no sample (Event.invoke drops it), so it
    must not take the next sample: every collector gets as many samples as its statistics count, and every Sink the
    completion times of exactly its own surviving requests."""
    from happysim_b200 import results
    model, end_s, plan, cancel, run_seed, what, _ = random_fault_case(version, seed)
    fm = with_faults(model, plan, cancel)
    out = LO.run(fm, engine.make_params(seed=run_seed, end_ns=int(end_s * 1e9), n_replicas=8, rid_stride=1,
                                        record_cap=16384, sample_cap=4096, service_cap=4096))
    assert int(out["summaries"]["events_processed"].max()) < 16384
    collectors = fm.ids_of(A.HS_ENT_SINK) + fm.ids_of(A.HS_ENT_PROBE)
    for r in range(8):
        per_sink, _ = results.demultiplex(fm, out, r)
        rec = out["records"][r][: int(out["summaries"]["events_processed"][r])]
        dropped = _dropped_by_replay(fm, rec)
        for i in collectors:
            got = per_sink[i] if per_sink[i] is not None else np.zeros(0, out["sink_samples"].dtype)
            assert len(got) == int(out["entity_stats"][r][i]["c0"]), (what, r, fm.names[i])
            if int(fm.entities["kind"][i]) == A.HS_ENT_SINK:
                mine = (rec["kind"] == A.HS_EV_REQ_SINK) & (rec["entity"] == i) & ~dropped
                assert got["completion_ns"].tolist() == rec["time_ns"][mine].tolist(), (what, r, fm.names[i])


def test_some_multi_collector_models_drop_requests_at_a_crashed_sink():
    n = 0
    for version, seed in _multi_collector_cases():
        model, end_s, plan, cancel, run_seed, _, _ = random_fault_case(version, seed)
        fm = with_faults(model, plan, cancel)
        out = LO.run(fm, engine.make_params(seed=run_seed, end_ns=int(end_s * 1e9), n_replicas=1, record_cap=16384))
        n += int(_dropped_by_replay(fm, out["records"][0][: int(out["summaries"]["events_processed"][0])]).sum())
    assert n > 0
