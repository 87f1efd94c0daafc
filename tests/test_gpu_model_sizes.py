"""The general engines at the model sizes that change their layout, every replica against the oracle.

Ensemble size is covered by tests/test_gpu_launch_geometry.py; this file covers the other axis, the size of one model:

  warp engine    A replica block per warp in shared memory.  Its size sets the warps per CTA (8 down to 1), whether
                 the model tables are copied into shared memory or read from global memory, and whether the model is
                 refused (launch_warp, general_setup).  Rows from 3 warps down to the last accepted block (231 216 B),
                 each with a second replica staged by the persistent warps, fresh and cut into three windows.
  thread engine  Heap keys carry the payload slot in 16 bits, the free-slot stack and event records hold 16-bit ids:
                 a server with about 35 000 requests in service next to a short one whose continuations take and
                 give back slot ids above 2^15 (a heap 8 levels deep under a shared-memory top), the largest slot
                 count S = 65 504, 65 535 rows (every one of 65 531 Counters reached, a Probe on the last), and both
                 sides of the entity-owned payload-slot rule.
  state region   Sketches and TTL caches at the top of their ranges: HLL p = 16 (table-driven and hashed on the
                 device), a 2 719 x 7 Count-Min sketch, a Bloom filter of 2^20 + 1 bits, TopK k = 512, TDigest
                 compression 400, a reservoir of 5 000 and a CachingServer with 2^20 key slots (8 MB per replica).
  limits         One step under and one over each limit; after every refusal the same Engine runs the next model.

Every case compares every replica with the oracle bit for bit (summaries, entity statistics, event records, Sink and
service-time samples in rings small enough to wrap, latency histograms, sketch states and the merged sketch image) and
asserts through Engine.last_launch() the layout tests/model_size_lib.py restates, so a change to a sizing rule fails
here instead of silently moving the coverage.  Whether the thread engine used entity-owned payload slots is not
reported by hs_last_launch, and both layouts compute the same results: the two Counter fans sit on either side of the
rule as restated, and no output comparison can tell which layout ran.

Measured on an H100 80GB HBM3 (700 W power limit) with 8 host CPUs: the file runs in about 70 s, and the device's
memory in use peaked at 6 329 MiB (the device was otherwise idle; the module's one Engine keeps its largest buffers
until it closes).  The largest allocations are the thread-engine replica blocks of
the slot server at two replicas per warp (2 117 x 1.8 MB), the 65 535-row model (40 x 8.4 MB of state, 40 x 65 535
entity statistics and records that keep the whole run) and the state region (48 x 8.8 MB)."""
import numpy as np
import pytest

import model_size_lib as L
import oracle_lib as O
from happysim_b200 import _abi as A, engine
from high_water_lib import fel_slots
from test_gpu_launch_geometry import CAPS, FLAGS, GEOMETRY, check_thread_geometry, compare, run_in_windows

pytestmark = pytest.mark.gpu

RING = 32                  # queue rings: the farms' queues stay a few entries deep (a deeper one is flagged and fails)


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


def device_vs_oracle(eng, model, kw, eng_id):
    eng.upload(model)
    eng.run(engine.make_params(engine=eng_id, **kw))
    li = eng.last_launch()
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    compare(eng, model, eng.read_outputs(), want)
    return li, want


# ---- (a) warp engine layouts -------------------------------------------------------------------------------------------

# name: (model, horizon in ns, warps, tables in shared memory)
WARP_ROWS = {
    "farm128": (lambda: L.farm(128), 400_000_000, 3, True),
    "farm256": (lambda: L.farm(256), 300_000_000, 2, True),
    "farm512": (lambda: L.farm(512), 250_000_000, 1, True),
    "farm1024_rr": (lambda: L.farm(1024), 150_000_000, 1, False),
    "farm1024_configs3": (lambda: L.farm(1024, key_table=L.configs3_table(), rate=8192.0), 150_000_000, 1, False),
    "sinks2300": (lambda: L.sink_fan(2300, 20000.0), 200_000_000, 1, False),
    "c4965": (lambda: L.wide_server(4965, 3000.0, 1.0, exponential=True), 1_500_000_000, 1, True),
}


def check_warp_geometry(li, model, n, sm):
    geo = L.warp_geometry(model)
    assert not geo["refused"]
    assert (li["engine"], li["kernel"], li["block"], li["smem"]) == (1, "warp", geo["warps"] * 32, geo["smem"]), (li, geo)
    assert li["grid"] == L.warp_grid(geo, n, sm) and n > li["grid"] * geo["warps"], (li, geo, n)    # second replicas
    return geo


@pytest.mark.parametrize("mode", ["fresh", "windows"])
@pytest.mark.parametrize("name", sorted(WARP_ROWS))
def test_warp_engine_layout(eng, sm, name, mode):
    mk, end_ns, warps, smem_tables = WARP_ROWS[name]
    model = mk()
    geo = L.warp_geometry(model)
    assert (geo["warps"], geo["model_bytes"] > 0) == (warps, smem_tables), geo
    n = sm * geo["ctas_per_sm"] * warps + 3
    kw = dict(seed=71, end_ns=end_ns, n_replicas=n, flags=FLAGS, queue_ring=RING, **CAPS)
    if mode == "windows":          # the 1-warp rows move blocks of up to 231 216 B by TMA across mbarrier phases
        li, _ = run_in_windows(eng, model, kw, 1)
    else:
        li, want = device_vs_oracle(eng, model, kw, 1)
        assert np.median(want["summaries"]["events_processed"]) > CAPS["record_cap"]
    check_warp_geometry(li, model, n, sm)


# ---- (b) thread engine: slots above 2^15, the largest S, 65 535 rows ----------------------------------------------------

SLOT_RING = 1024           # = the slot server's queue capacity: a stalled replica drops instead of overflowing the ring


@pytest.mark.parametrize("row", ["wide", "rpw1", "rpw2"])
def test_thread_engine_slot_ids_above_2_15(eng, sm, row):
    """Most replicas hold more than 32 768 pending continuations (heap_left), and the short server's continuations
    are popped from slot ids above 2^15: the 16-bit slot ids of the heap keys and the free-slot stack.  At two replicas per warp the heap's top 21 keys sit in shared memory
    above 8 levels in HBM; that row runs cut into three windows (the paused prefix and the end against the oracle)."""
    model = L.slot_server()
    assert fel_slots(model) == 36544 and not L.fixed_slots(model)
    n = GEOMETRY[row][0](sm)
    kw = dict(seed=72, end_ns=L.SLOT_END_NS, n_replicas=n, flags=FLAGS, queue_ring=SLOT_RING, **CAPS)
    if row == "rpw2":
        li, _ = run_in_windows(eng, model, kw, 3)
    else:
        li, want = device_vs_oracle(eng, model, kw, 3)
        assert (want["summaries"]["heap_left"] > 1 << 15).mean() > 0.7
    check_thread_geometry(li, row, n)


def test_largest_slot_count_runs_after_the_next_is_refused(eng, sm):
    """c = 65 474 needs S = 65 536 slots: refused, naming the limit.  The same Engine then runs c = 65 473 (S = 65 504)
    with every slot of most replicas busy, the short server's continuations taking slot ids up to the top."""
    over = L.slot_server(L.MAX_SLOT_C + 1, service_s=33.0)
    assert fel_slots(over) == 65536
    eng.upload(over)
    with pytest.raises(engine.EngineError, match=r"65536 future-event slots \(limit 65535\)"):
        eng.run(engine.make_params(engine=3, seed=74, end_ns=L.MAX_SLOT_END_NS, n_replicas=64))
    model = L.slot_server(L.MAX_SLOT_C, service_s=33.0)
    assert fel_slots(model) == 65504
    kw = dict(seed=74, end_ns=L.MAX_SLOT_END_NS, n_replicas=64, flags=FLAGS, queue_ring=SLOT_RING, **CAPS)
    li, want = device_vs_oracle(eng, model, kw, 3)
    check_thread_geometry(li, "wide", 64)
    assert (want["summaries"]["heap_left"] > L.MAX_SLOT_C).mean() > 0.7           # every slot busy


def test_most_entities_run_after_one_more_is_refused(eng, sm):
    """65 536 rows are refused at upload; the same Engine then takes 65 535 rows (65 531 Counters, a Probe on the
    last): every Counter is reached, and the records, which keep the whole run here, hold entity ids up to 65 534."""
    too_many = L.counter_fan(L.N_FAN_COUNTERS + 1, L.FAN_RATE, probe_on=L.N_FAN_COUNTERS)
    assert too_many.n_entities == L.ENTITY_LIMIT + 1
    with pytest.raises(engine.EngineError, match=r"n_entities must be 1\.\.65535"):
        eng.upload(too_many)
    model = L.max_counter_fan()
    assert model.n_entities == L.ENTITY_LIMIT and not L.fixed_slots(model)
    n = 40
    kw = dict(seed=75, end_ns=L.FAN_END_NS, n_replicas=n, flags=FLAGS, record_cap=1 << 19, sample_cap=7, service_cap=5)
    li, want = device_vs_oracle(eng, model, kw, 3)
    check_thread_geometry(li, "wide", n)
    counters = want["entity_stats"][:, 1:1 + L.N_FAN_COUNTERS]["c0"]
    assert (counters > 0).all()
    assert (want["summaries"]["events_processed"] < kw["record_cap"]).all()
    assert int(want["records"]["entity"].max()) == L.ENTITY_LIMIT - 1


@pytest.mark.parametrize("n_counters", [30, 31])
def test_entity_owned_payload_slots_boundary(eng, sm, n_counters):
    """ne = S = 32 takes the entity-owned payload slots, ne = 33 > S the free-slot stack (not observable in the
    outputs or hs_last_launch: this pins the models to either side of the rule as restated)."""
    model = L.counter_fan(n_counters, 400.0)
    assert (model.n_entities, fel_slots(model), L.fixed_slots(model)) == (n_counters + 2, 32, n_counters == 30)
    n = GEOMETRY["rpw2"][0](sm)
    li, _ = device_vs_oracle(eng, model, dict(seed=76, end_ns=300_000_000, n_replicas=n, flags=FLAGS, **CAPS), 3)
    check_thread_geometry(li, "rpw2", n)


# ---- (c) the per-replica state region at the top of its ranges ----------------------------------------------------------

@pytest.mark.parametrize("eng_id", [1, 3])
def test_state_region_at_the_top_of_its_ranges(eng, sm, eng_id):
    model = L.big_sketches()
    assert model.sketch_layout()[2] > 8 << 20
    kw = dict(seed=77, end_ns=6 * 10**9, n_replicas=48, flags=FLAGS, queue_ring=RING, **CAPS)
    li, want = device_vs_oracle(eng, model, kw, eng_id)
    assert li["engine"] == eng_id, li
    if eng_id == 1:
        geo = L.warp_geometry(model)
        assert (li["block"], li["smem"]) == (geo["warps"] * 32, geo["smem"]), li
    st = want["entity_stats"][0]
    sk = model.ids_of(A.HS_ENT_SKETCH)
    views = model.sketch_views(want["sketches"])
    reservoir, topk = sk[-1], sk[-3]
    assert (want["entity_stats"][:, reservoir]["c1"] > 5000).all()          # the reservoir replaces items
    assert (views[topk][:, 0] == 512).all()                                 # TopK holds k = 512 counters
    assert st[model.ids_of(A.HS_ENT_CACHE_SERVER)[0]]["c2"] > 0


# ---- (d) limits ---------------------------------------------------------------------------------------------------------

def test_warp_engine_last_accepted_block_after_the_next_is_refused(eng, sm):
    over = L.wide_server(4966, 3000.0, 1.0, exponential=True)
    assert L.warp_geometry(over)["refused"]
    eng.upload(over)
    with pytest.raises(engine.EngineError, match="model too large for the warp engine"):
        eng.run(engine.make_params(engine=1, seed=78, end_ns=10**9, n_replicas=8))
    model = WARP_ROWS["c4965"][0]()
    assert L.warp_geometry(model)["per_warp"] == 231216
    n = sm + 3
    li, _ = device_vs_oracle(eng, model, dict(seed=78, end_ns=10**9, n_replicas=n, flags=FLAGS, **CAPS), 1)
    check_warp_geometry(li, model, n, sm)


@pytest.mark.parametrize("case", ["c64", "c65", "cells_1_65"])
def test_automatic_engine_choice_at_the_lane_limit(eng, case):
    """Engine 0 takes the lane engine up to concurrency 64 and the thread engine above, also when one sweep cell of
    the model passes 64."""
    if case == "cells_1_65":
        model = L.wide_server(1, 10.0, 0.1, exponential=True)
        model.cell_d0 = np.tile(model.entities["d0"].astype(np.float64), (2, 1))
        model.cell_i0 = np.tile(model.entities["i0"].astype(np.int32), (2, 1))
        model.cell_d0[:, 0] = (8.0, 600.0)
        model.cell_i0[:, 1] = (1, 65)
        extra = dict(replicas_per_cell=3)
    else:
        c = int(case[1:])
        model = L.wide_server(c, 9.0 * c, 0.1, exponential=True)
        extra = {}
    kw = dict(seed=79, end_ns=2 * 10**9, n_replicas=301, flags=FLAGS, **CAPS, **extra)
    li, _ = device_vs_oracle(eng, model, kw, 0)
    assert li["engine"] == (2 if case == "c64" else 3), li
