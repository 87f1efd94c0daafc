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


# ---- the fault oracle (tests/fault_oracle.c) against the reference ----------------------------------------------------
import fault_oracle_lib as FO  # noqa: E402


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
    got = FO.run(model, engine.make_params(n_replicas=1, **G.caps(z), **kw))
    G.check_against(z, got)
    tie = bool(int(got["summaries"]["status"][0]) & A.HS_ST_FAULT_TIE)
    assert tie == name.startswith("fault_tie"), "HS_ST_FAULT_TIE exactly where the reference tied"
    # the reference's own final flags and the events_cancelled its summary reported
    fr = model.ids_of(A.HS_ENT_FAULT)
    assert int(got["entity_stats"][0][fr]["c1"].sum()) == int(z["events_cancelled"])


def _random_seeds(n=60):
    """the first n seeds of tests/random_models.py whose model the reference harness can build (no random key table)"""
    from random_models import random_model
    out, s = [], 0
    while len(out) < n:
        if not random_model(s, with_extras=True)[3]["random_key_table"]:
            out.append(s)
        s += 1
    return out


RANDOM_SEEDS = _random_seeds()


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
@pytest.mark.parametrize("seed", RANDOM_SEEDS)
def test_fault_oracle_matches_reference_on_random_models(seed):
    """Seeded random models (tests/random_models.py) with random node-fault schedules: the fault oracle against the
    unmodified reference, run here with the Philox plug-ins."""
    import os
    import random
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import gen_fault_golden as GF
    from random_models import random_model
    model, end_s, _, ex = random_model(seed, with_extras=True)
    end_s = min(float(end_s), 6.0)
    rng = random.Random(1000 + seed)
    ents = model.entities
    names = [n for i, n in enumerate(model.names) if int(ents["kind"][i]) != A.HS_ENT_PROBE and not (
        int(ents["kind"][i]) == A.HS_ENT_SOURCE and int(ents["kind"][int(ents["target"][i])]) == A.HS_ENT_PROBE)]
    plan = []
    for _ in range(rng.randint(1, 4)):
        nm = rng.choice(names)
        a = round(rng.uniform(0.0, end_s), 3)
        kind = rng.choice(["crash", "crash_restart", "pause"])
        b = round(a + rng.uniform(0.01, end_s / 2), 3)
        plan.append((kind, nm, a, b))
    cancel = [k for k in range(len(plan)) if rng.random() < 0.2]

    def build(by, F):
        s = F.FaultSchedule()
        for kind, nm, a, b in plan:
            s.add(F.CrashNode(nm, at=a) if kind == "crash" else F.CrashNode(nm, at=a, restart_at=b) if kind == "crash_restart"
                  else F.PauseNode(nm, start=a, end=b))
        return s
    kw = dict(seed=seed, rid=seed % 5, end_s=end_s, cancel=cancel, expect_tie="any", sketch_seeds=ex["sketch_seeds"],
              zipf_s=ex["zipf_s"])
    fm, ref, meta = GF.run_case(model, build, kw)
    got = FO.run(fm, engine.make_params(n_replicas=1, seed=seed, rid_base=seed % 5, end_ns=int(end_s * 1e9),
                                        record_cap=len(ref["records"]) + 1, sample_cap=len(ref["sink_samples"]) + 1,
                                        service_cap=len(ref["service_samples"]) + 1))
    _check_ref(ref, got)
