"""The layout rules of tests/model_size_lib.py against hand-computed values, the large models of
tests/test_gpu_model_sizes.py on the oracle, and the oracle against the reference's own runs of the marked models
(tests/golden/size_*.npz, tests/golden/gen_model_size_golden.py).  No device needed."""
import os

import numpy as np
import pytest

import golden_lib as G
import high_water_lib as HW
import model_size_lib as L
import oracle_lib as O
from happysim_b200 import _abi as A, engine

# name: (model, rows, S, warp-engine warps or None when refused, tables in shared memory, bytes per warp)
# Hand-computed from general_setup / launch_warp: per warp 16 + 128 + 96 ne + ceil16(46 S) + 24 x 48 bytes, tables
# 48 ne + 4 ne + 4 backends bytes, warps min(8, 102 400 // per warp) while they fit 231 424 bytes.
TABLE = {
    "farm64": (lambda: L.farm(64), 67, 160, 6, True, 15088),
    "farm128": (lambda: L.farm(128), 131, 288, 3, True, 27120),
    "farm256": (lambda: L.farm(256), 259, 544, 2, True, 51184),
    "farm512": (lambda: L.farm(512), 515, 1056, 1, True, 99312),
    "farm1024": (lambda: L.farm(1024), 1027, 2080, 1, False, 195568),
    "sinks2300": (lambda: L.sink_fan(2300, 1.0), 2302, 32, 1, False, 223760),
    "c4965": (lambda: L.wide_server(4965, 1.0, 1.0), 3, 4992, 1, True, 231216),
    "c4966": (lambda: L.wide_server(4966, 1.0, 1.0), 3, 5024, None, None, 232688),
}


@pytest.mark.parametrize("name", sorted(TABLE))
def test_warp_layout_rule_matches_hand_computed_values(name):
    mk, ne, S, warps, smem_tables, per_warp = TABLE[name]
    model = mk()
    geo = L.warp_geometry(model)
    assert (model.n_entities, HW.fel_slots(model), geo["per_warp"]) == (ne, S, per_warp)
    if warps is None:
        assert geo["refused"]
    else:
        assert (geo["refused"], geo["warps"], geo["model_bytes"] > 0) == (False, warps, smem_tables)
        assert geo["smem"] <= L.WARP_SMEM_MAX


def test_thread_slot_and_entity_rules():
    assert HW.fel_slots(L.slot_server()) == 36544
    assert HW.fel_slots(L.slot_server(L.MAX_SLOT_C)) == 65504 <= L.SLOT_LIMIT
    assert HW.fel_slots(L.slot_server(L.MAX_SLOT_C + 1)) == 65536 > L.SLOT_LIMIT
    assert L.max_counter_fan().n_entities == L.ENTITY_LIMIT
    assert [L.fixed_slots(L.counter_fan(k, 1.0)) for k in (30, 31)] == [True, False]       # ne = S = 32, then 33
    assert L.fixed_slots(L.farm(64)) and not L.fixed_slots(L.slot_server()) and not L.fixed_slots(L.big_sketches())


def test_validation_takes_65535_rows_and_refuses_65536():
    engine.validate_model(L.max_counter_fan())
    with pytest.raises(engine.EngineError, match=r"n_entities must be 1\.\.65535"):
        engine.validate_model(L.counter_fan(L.N_FAN_COUNTERS + 1, 1.0, probe_on=L.N_FAN_COUNTERS))


def test_slot_server_holds_more_than_2_15_pending_continuations():
    """The coverage the GPU cases claim: most replicas of the slot server (the seed of the GPU file's first case)
    reach more than 32 768 pending future events, and the bounded queue keeps every queue within the ring."""
    model = L.slot_server()
    out, hw = HW.run(model, O.make_params(seed=72, end_ns=L.SLOT_END_NS, n_replicas=24, queue_ring=1024))
    assert (hw["future"] > 1 << 15).mean() > 0.7 and hw["future"].max() <= HW.fel_slots(model)
    assert hw["queue"].max() <= 1024 and not out["summaries"]["status"].any()


FIXTURES = sorted(L.fixture_models())


@pytest.fixture(scope="module")
def fixture_models():
    return L.fixture_models()


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_matches_the_reference_at_model_size(fixture_models, name):
    model, end_ns, _ = fixture_models[name]
    z = np.load(os.path.join(G.GOLDEN_DIR, f"size_{name}.npz"))
    seed, z_end = (int(v) for v in z["meta"])
    assert (seed, z_end) == (L.FIXTURE_SEED, end_ns)
    ws = z["summaries"][0]
    n_ev, n_smp = int(ws["events_processed"]), int(ws["n_sink_samples"])
    got = O.oracle_run(model, O.make_params(seed=seed, end_ns=end_ns, n_replicas=1, record_cap=n_ev + 1,
                                            sample_cap=n_smp + 1))
    s = got["summaries"][0]
    for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
        assert int(s[f]) == int(ws[f]), (f, int(s[f]), int(ws[f]))
    assert got["entity_stats"][0].tobytes() == z["entity_stats"][0].tobytes(), "entity statistics differ"
    tail = z["records_tail"]
    assert got["records"][0][n_ev - len(tail): n_ev].tobytes() == tail.tobytes(), "event records differ"
    tail = z["samples_tail"]
    assert got["sink_samples"][0][n_smp - len(tail): n_smp].tobytes() == tail.tobytes(), "Sink samples differ"
    if name == "slot_server":
        assert int(ws["heap_left"]) > 1 << 15
    if name == "counter_fan":
        assert (z["entity_stats"][0][1:1 + L.N_FAN_COUNTERS]["c0"] > 0).all()
        assert int(z["records_tail"]["entity"].max()) <= L.ENTITY_LIMIT - 1
        assert A.HS_ENT_PROBE == int(model.entities["kind"][L.ENTITY_LIMIT - 2])
