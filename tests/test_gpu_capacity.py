"""The device's fixed-size structures at their bounds, every replica against the oracle.

The reference's queues and event heap have no limit.  On the device each sits in a fixed-size structure, and a replica
that would outgrow one is flagged and stopped; up to the bound the run must equal the reference:

  queue rings        queue_ring = R slots per server            HS_ST_QUEUE_OVERFLOW  <=> a queue passes R entries
  now tier           HS_W_NCAP = 24 same-timestamp events       HS_ST_FEL_OVERFLOW    <=> more than 24 pending
  future-event slots general_setup's S (hs_engine.cu)           HS_ST_FEL_OVERFLOW    <=> more than S pending
  outbox / inbox     ParallelSimulation.link_buffer             HS_ST_LINK_OVERFLOW / the coordinator's overflow count

The instrumented oracle (tests/high_water_lib.py) gives every replica's high-water mark of each structure, and the
ensembles of tests/capacity_models.py put replicas at bound - 1, bound and bound + 1 (tests/test_high_water.py checks
that on the CPU).  Every case asserts which kernel it reached, that the flagged replicas are exactly those whose
high-water passes the bound, that every other replica equals the oracle bit for bit, and that a flagged replica's
event records, order hash and clock equal the oracle's run stopped after as many events."""

import numpy as np
import pytest

import capacity_models as CM
import happysim_b200 as hs
import high_water_lib as HW
import oracle_lib as O
from happysim_b200 import _abi as A, engine
from happysim_b200.linked import LinkedRun
from test_gpu_lane_parity import KEYS, assert_same
from test_gpu_launch_geometry import check_thread_geometry

pytestmark = pytest.mark.gpu

CAPS = dict(record_cap=40, sample_cap=6, service_cap=4)      # rings that wrap
FLAGS = A.HS_RUN_ORDER_HASH
LF_REC, LF_SIMPLE = 2, 8                                      # HS_LF_* of csrc/hs_lane_engine.cuh


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def device_run(eng, model, kw):
    eng.upload(model)
    eng.run(engine.make_params(**kw))
    return eng.read_outputs(), eng.last_launch()


def rows(out, idx):
    return {k: (None if out[k] is None else np.ascontiguousarray(out[k][idx])) for k in KEYS}


def assert_stopped_prefix(model, kw, got, idx):
    """Replicas ``idx`` stopped at a bound: their records, order hash, event count and clock equal the oracle's run
    of the same replica limited to the events the device processed."""
    n_ev = got["summaries"]["events_processed"]

    def one(r):
        p = O.make_params(**dict(kw, n_replicas=1, replica_index_base=kw.get("replica_index_base", 0) + int(r),
                                 max_events=int(n_ev[r])))
        w = O.oracle_run(model, p)
        g, s = got["summaries"][r], w["summaries"][0]
        assert (int(g["events_processed"]), int(g["final_time_ns"]), int(g["order_hash"])) == \
               (int(s["events_processed"]), int(s["final_time_ns"]), int(s["order_hash"])), f"replica {r}"
        if got["records"] is not None:
            assert got["records"][r].tobytes() == w["records"][0].tobytes(), f"replica {r}: records"
    O._pool_map(one, list(idx))


def check_bound(model, kw, got, high, cap, bit, *, stopped=True):
    """flagged (status & bit) <=> high > cap; the rest bit for bit; the flagged ones a prefix of the oracle's run"""
    want, _ = HW.run(model, O.make_params(**kw))
    flagged = (got["summaries"]["status"] & bit) != 0
    over = high > cap
    assert np.array_equal(flagged, over), (f"flagged {np.flatnonzero(flagged & ~over)[:8]} under the bound, "
                                           f"unflagged {np.flatnonzero(over & ~flagged)[:8]} over it")
    assert over.any() and (~over).any() and (high == cap).any()
    ok = np.flatnonzero(~flagged)
    assert_same(rows(got, ok), rows(want, ok))
    if stopped:
        assert_stopped_prefix(model, kw, got, np.flatnonzero(flagged))
    return flagged


# ---- queue rings -----------------------------------------------------------------------------------------------------

def ring_high(model, kw):
    """per replica the longest queue of any server"""
    _, hw = HW.run(model, O.make_params(**kw))
    return hw["queue"].max(axis=1)


@pytest.mark.parametrize("rec", [False, True], ids=["summary", "rec"])
@pytest.mark.parametrize("name", ["mm1", "mmc4_lifo"])
def test_lane_queue_ring(eng, name, rec):
    """SIMPLE M/M/1 (its fused chain must fall back to the generic enqueue at a full ring) and the general lane kernel
    with c = 4 and LIFO (a pop reads slot q_head + R - 1)."""
    model, kw = CM.ring_case(name)
    kw = dict(kw, engine=2, flags=FLAGS, **(CAPS if rec else {}))
    got, li = device_run(eng, model, kw)
    fl = (LF_REC if rec else 0) | (LF_SIMPLE if name == "mm1" else 0)
    assert (li["engine"], li["kernel"], li["flags"] & (LF_REC | LF_SIMPLE)) == (2, "lane", fl), li
    check_bound(model, kw, got, ring_high(model, kw), CM.RING, A.HS_ST_QUEUE_OVERFLOW)


@pytest.mark.parametrize("row", ["wide", "rpw2", "warp"])
def test_general_engines_queue_ring_tandem(eng, sm, row):
    """Three servers in a row: every server's ring reaches the bound in some replicas."""
    n = 8 * sm - 5 if row == "wide" else CM.N_RING
    model, kw = CM.ring_case("tandem3", n=n)
    kw = dict(kw, engine=1 if row == "warp" else 3, flags=FLAGS, **CAPS)
    got, li = device_run(eng, model, kw)
    if row == "warp":
        assert (li["engine"], li["kernel"]) == (1, "warp"), li
    else:
        check_thread_geometry(li, row, n)
    _, hw = HW.run(model, O.make_params(**kw))
    for i in (2, 3, 4):
        assert (hw["queue"][:, i] == CM.RING).any() and (hw["queue"][:, i] > CM.RING).any(), i
    check_bound(model, kw, got, hw["queue"].max(axis=1), CM.RING, A.HS_ST_QUEUE_OVERFLOW)


@pytest.mark.parametrize("eng_id", [2, 3, 1])
def test_bounded_queue_of_ring_capacity_drops_and_never_flags(eng, eng_id):
    model, kw = CM.ring_case("mm1_capacity")
    kw = dict(kw, engine=eng_id, flags=FLAGS, **CAPS)
    got, li = device_run(eng, model, kw)
    assert li["engine"] == eng_id, li
    want, hw = HW.run(model, O.make_params(**kw))
    assert (hw["queue"][:, 1] == CM.RING).sum() > 100 and (want["entity_stats"][:, 1]["c1"] > 0).any()
    assert not got["summaries"]["status"].any()
    assert_same(got, want)


@pytest.mark.parametrize("name", ["mm1", "mmc4_lifo"])
def test_lane_ring_cut_at_a_full_ring_resumes_exactly(eng, name):
    """Cut into windows where some replicas hold exactly R queued requests (the ring head and the next item are
    reloaded on resume): the windowed run equals the uncut one, flags included."""
    model, kw = CM.ring_case(name)
    kw = dict(kw, engine=2, flags=FLAGS, **CAPS)
    whole, _ = device_run(eng, model, kw)
    eng.run(engine.make_params(**dict(kw, window_end_ns=CM.ring_cut(kw))))
    eng.run(engine.make_params(**dict(kw, resume=1)))
    assert eng.last_launch()["kernel"] == "lane"
    cut = eng.read_outputs()
    assert_same(cut, whole)
    check_bound(model, kw, cut, ring_high(model, kw), CM.RING, A.HS_ST_QUEUE_OVERFLOW, stopped=False)


# ---- the now tier ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("row", ["wide", "rpw2", "warp"])
def test_now_tier(eng, sm, row):
    """Sweep cells with 1, 2, 3, 19, 20 and 21 sources on one rate: now-tier depths around 4 (the thread engine's
    shared-memory entries) and around 24.  The warp engine also moves a popped future event into the tier before
    handling it, so it needs a free entry then (now_pop: never 24 with at most 24 otherwise, tests/test_high_water.py)."""
    n = CM.now_replicas("wide" if row == "warp" else row, sm)
    model = CM.now_farm()
    kw = dict(CM.now_kw(n), engine=1 if row == "warp" else 3, flags=FLAGS, **CAPS)
    got, li = device_run(eng, model, kw)
    if row == "warp":
        assert (li["engine"], li["kernel"]) == (1, "warp"), li
    else:
        check_thread_geometry(li, row, n)
    _, hw = HW.run(model, O.make_params(**kw))
    assert {3, 4, 5, 23, 24, 25} <= set(hw["now"].tolist())
    high = np.where(hw["now_pop"] >= HW.HS_W_NCAP, HW.HS_W_NCAP + 1, hw["now"]) if row == "warp" else hw["now"]
    check_bound(model, kw, got, high, HW.HS_W_NCAP, A.HS_ST_FEL_OVERFLOW)


# ---- the future-event slots ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("eng_id", [3, 1])
def test_future_event_slots(eng, eng_id):
    model = CM.cache_load()
    S = HW.fel_slots(model)
    kw = dict(CM.FEL_KW, engine=eng_id, flags=FLAGS, **CAPS)
    got, li = device_run(eng, model, kw)
    assert li["engine"] == eng_id, li
    _, hw = HW.run(model, O.make_params(**kw))
    flagged = (got["summaries"]["status"] & A.HS_ST_FEL_OVERFLOW) != 0
    lo, hi = int(hw["future"][~flagged].max()), int(hw["future"][flagged].min())
    assert lo < hi, f"no single threshold: unflagged replicas reach {lo} pending future events, flagged ones start at {hi}"
    assert lo == S == hi - 1, (f"the device flags above {lo} (first flagged at {hi}) future events; general_setup's "
                               f"sizing rule as restated in high_water_lib.fel_slots gives S = {S}")
    check_bound(model, kw, got, hw["future"], S, A.HS_ST_FEL_OVERFLOW)


def test_simulation_run_raises_on_a_future_slot_overflow():
    model = CM.cache_load()
    _, hw = HW.run(model, O.make_params(**CM.FEL_KW))
    r = int(np.argmax(hw["future"]))
    assert hw["future"][r] > HW.fel_slots(model)
    cs = hs.CachingServer("CachingServer", cache_capacity=4001, cache_ttl_s=0.001, cache_read_latency_s=0.0001,
                          datastore_read_latency_s=0.05, processing_latency_s=0.011)
    src = hs.Source.poisson(rate=1000.0, event_provider=hs.SimpleEventProvider(cs, context_fn=hs.UniformKeyContext(4000)))
    sim = hs.Simulation(end_time=hs.Instant(CM.FEL_KW["end_ns"]), sources=[src], entities=[cs], seed=CM.FEL_KW["seed"],
                        replica=r)
    assert sim.model.entities.tobytes() == model.entities.tobytes()
    with pytest.raises(RuntimeError, match="overflow"):
        sim.run()
    assert cs.stats.requests_processed == 0 and cs.stats_accepted == 0         # no partial results reach the objects


# ---- linked partitions -----------------------------------------------------------------------------------------------

def test_link_outbox_and_inbox():
    lm = CM.linked_tandem()
    caps = dict(record_cap=60, sample_cap=8, service_cap=6)
    kw = CM.LINKED_KW
    run = LinkedRun(lm)
    try:
        outs, (delivered, lost, over) = run.run(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=kw["n_replicas"], caps=caps)
        assert all(e.last_launch()["engine"] == 3 for e in run.engines)
    finally:
        run.close()
    want, wd, wl, hw = HW.run_linked(lm, CM.linked_params(lm, **caps), end_ns=kw["end_ns"], cseed=kw["seed"])
    # the outbox: the oracle drops and flags as the device does, so every replica of A is compared
    flagged = (outs[0]["summaries"]["status"] & A.HS_ST_LINK_OVERFLOW) != 0
    assert np.array_equal(flagged, hw[0]["outbox"] > CM.OUTBOX_CAP) and flagged.any() and not flagged.all()
    assert_same(outs[0], want[0])
    # the inbox: an overflowing barrier drops what the oracle delivers
    inb = hw[1]["inbox"]
    assert np.array_equal(over > 0, inb > CM.INBOX_CAP) and (over > 0).any() and (inb == CM.INBOX_CAP).any()
    ok = np.flatnonzero(over == 0)
    assert np.array_equal(delivered[ok], wd[ok]) and not lost.any() and not wl.any()
    assert_same(rows(outs[1], ok), rows(want[1], ok))
    assert not (outs[1]["summaries"]["status"] & ~np.uint32(A.HS_ST_LINK_TIE)).any()


def test_parallel_simulation_raises_naming_link_buffer(monkeypatch):
    monkeypatch.setattr(hs.ParallelSimulation, "link_buffer", 2)      # read when the partitions are lowered
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=2, service_time=hs.ExponentialLatency(0.02), downstream=sink)
    sa = hs.Server("A.server", service_time=hs.ExponentialLatency(0.012), downstream=sb)
    src = hs.Source.poisson(rate=40.0, target=sa)
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src]), hs.SimulationPartition("B", entities=[sb, sink])]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=hs.ConstantLatency(0.05))
    ps = hs.ParallelSimulation(parts, duration=6.0, links=[link], seed=17)
    with pytest.raises(RuntimeError, match="link_buffer = 2"):
        ps.run()
