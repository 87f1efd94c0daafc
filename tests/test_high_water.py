"""The oracle's high-water marks (hs_oracle.c built with -DHS_ORACLE_HIGH_WATER, tests/high_water_lib.py) on the CPU:
hand-checkable values, a recount from the oracle's own event records, byte-for-byte equality with the default build,
and the ensembles of tests/test_gpu_capacity.py straddling the bounds they test."""
import numpy as np
import pytest

import capacity_models as CM
import happysim_b200 as hs
import high_water_lib as HW
import oracle_lib as O
import random_models as RM
from happysim_b200 import _abi as A

H100_SMS = 132               # the GPU file sizes its thread-engine launches by the SM count of an H100 SXM


def servers_of(model):
    k = model.entities["kind"]
    return [i for i in range(model.n_entities) if k[i] in (A.HS_ENT_SERVER, A.HS_ENT_CACHE_SERVER)]


def straddles(x, cap, what):
    have = set(np.asarray(x).tolist())
    assert {cap - 1, cap, cap + 1} <= have, f"{what}: no replica at one of {cap - 1}, {cap}, {cap + 1} (have {sorted(have)})"


# ---- hand-checkable values ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [1, 3, 4, 5, 24, 25])
def test_k_sources_at_one_rate_fill_the_now_tier_k_deep(k):
    """k constant-rate sources at one rate, straight into a Counter: at every common tick the k SourceEvents are popped
    one after another (each leaves its payload in the now tier and its next tick in the future), then the k payloads."""
    b = hs.ModelBuilder()
    cnt = b.counter()
    for i in range(k):
        b.source(f"S{i}", rate=4.0, poisson=False, target=cnt)
    m = b.build()
    out, hw = HW.run(m, O.make_params(end_ns=3 * 10**9, n_replicas=2))
    assert (hw["now"] == k).all() and (hw["now_pop"] == k - 1).all() and (hw["future"] == k).all()
    assert (out["entity_stats"][:, 0]["c0"] == 12 * k).all()


def test_dd1_queue_reaches_its_known_maximum():
    """D/D/1, arrivals every 100 ms into 250.0001 ms of service: the k-th enqueue (k >= 2) finds the requests that
    started service strictly before it gone, floor((k - 1) * 1e8 / 250000100) + 1 of them, so it makes the queue
    k - 1 - floor((k - 1) * 1e8 / 250000100) long (the arrival times drift from whole multiples of 100 ms by tens of
    nanoseconds, far from any tie); the last enqueue makes the longest."""
    m = hs.mm1(rate=10.0, mean_service_s=0.2500001, poisson=False, exponential=False)
    out, hw = HW.run(m, O.make_params(end_ns=20 * 10**9, n_replicas=1))
    K = int(out["entity_stats"][0, 1]["c0"])             # enqueues (the tick past the end leaves its request unqueued)
    assert K == 200
    want = max([1] + [k - 1 - (k - 1) * 10**8 // 250000100 for k in range(2, K + 1)])
    assert int(hw["queue"][0, 1]) == want == 120


def test_dd1_underloaded_queue_holds_one():
    m = hs.mm1(rate=10.0, mean_service_s=0.05, poisson=False, exponential=False)
    _, hw = HW.run(m, O.make_params(end_ns=5 * 10**9, n_replicas=1))
    assert int(hw["queue"][0, 1]) == 1 and int(hw["now"][0]) >= 1


def test_bounded_queue_never_exceeds_its_capacity():
    m, kw = CM.ring_case("mm1_capacity", n=512)
    out, hw = HW.run(m, O.make_params(**{k: v for k, v in kw.items() if k != "queue_ring"}))
    q = hw["queue"][:, 1]
    assert q.max() == CM.RING and (q == CM.RING).sum() > 100
    dropped = out["entity_stats"][:, 1]["c1"]
    assert (dropped > 0).any() and (q[dropped > 0] == CM.RING).all()


# ---- against the oracle's own records -----------------------------------------------------------------------------------

def recount_queues(model, records, n_events):
    """Per server, the longest queue right after an enqueue, replayed from the event records: ENQUEUE adds one
    unless a bounded queue is full (then it drops), POLL takes one if there is one."""
    e = model.entities
    cap = {i: (-1 if e["kind"][i] == A.HS_ENT_CACHE_SERVER else int(e["l0"][i])) for i in servers_of(model)}
    q, hi = {i: 0 for i in cap}, {i: 0 for i in cap}
    for rc in records[:n_events]:
        i, kind = int(rc["entity"]), int(rc["kind"])
        if i not in cap:
            continue
        if kind == A.HS_EV_REQ_ENQUEUE and not (cap[i] >= 0 and q[i] >= cap[i]):
            q[i] += 1
            hi[i] = max(hi[i], q[i])
        elif kind == A.HS_EV_POLL and q[i] > 0:
            q[i] -= 1
    return hi


@pytest.mark.parametrize("seed", range(20))
def test_queue_high_water_equals_a_recount_from_the_records(seed):
    model, end_s, _ = RM.random_model(seed)[:3]
    p = O.make_params(seed=100 + seed, end_ns=int(end_s * 1e9), n_replicas=4, record_cap=1 << 15)
    out, hw = HW.run(model, p)
    n_ev = out["summaries"]["events_processed"]
    assert n_ev.max() <= p.record_cap
    for r in range(p.n_replicas):
        hi = recount_queues(model, out["records"][r], int(n_ev[r]))
        assert {i: int(hw["queue"][r, i]) for i in hi} == hi, r
    others = [i for i in range(model.n_entities) if i not in servers_of(model)]
    assert not hw["queue"][:, others].any()


# ---- the instrumented build runs the same replicas ----------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 3, 7, 11])
def test_instrumented_build_outputs_equal_the_default_build(seed):
    model, end_s, _ = RM.random_model(seed)[:3]
    p = O.make_params(seed=seed, end_ns=int(end_s * 1e9), n_replicas=9, record_cap=300, sample_cap=40, service_cap=30,
                      flags=A.HS_RUN_ORDER_HASH | A.HS_RUN_HISTOGRAM)
    got, _ = HW.run(model, p, chunk=4)
    want = O.oracle_run(model, p)
    for k, v in want.items():
        assert (v is None) == (got[k] is None) and (v is None or v.tobytes() == got[k].tobytes()), k


def test_instrumented_linked_outputs_equal_the_default_build():
    lm = CM.linked_tandem()
    kw = dict(CM.LINKED_KW, n_replicas=40)
    ps = [O.make_params(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=kw["n_replicas"], rid_base=q, rid_stride=3,
                        record_cap=500, sample_cap=50) for q in range(2)]
    outs, d, l, _ = HW.run_linked(lm, ps, end_ns=kw["end_ns"], cseed=kw["seed"], chunk=16)
    want, wd, wl, _ = O.oracle_run_linked(lm, ps, end_ns=kw["end_ns"], cseed=kw["seed"])
    assert np.array_equal(d, wd) and np.array_equal(l, wl)
    for q in range(2):
        for k, v in want[q].items():
            assert (v is None) == (outs[q][k] is None) and (v is None or v.tobytes() == outs[q][k].tobytes()), (q, k)


# ---- the GPU file's ensembles straddle their bounds ----------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(CM.RING_CASES))
def test_ring_ensembles_straddle_the_ring(name):
    m, kw = CM.ring_case(name)
    _, hw = HW.run(m, O.make_params(**{k: v for k, v in kw.items() if k != "queue_ring"}))
    for i in servers_of(m):
        if name == "mm1_capacity":
            assert hw["queue"][:, i].max() == CM.RING
            straddles(np.concatenate([hw["queue"][:, i], [CM.RING + 1]]), CM.RING, name)
        else:
            straddles(hw["queue"][:, i], CM.RING, f"{name}, server {i}")
    if name in ("mm1", "mmc4_lifo"):                     # lane-eligible: the lane engine's same-timestamp queue holds it
        assert hw["now"].max() <= HW.HS_NOW_CAP


@pytest.mark.parametrize("name", ["mm1", "mmc4_lifo"])
def test_ring_window_cut_holds_exactly_a_full_ring(name):
    """The cut of the windowed ring runs: some replicas hold exactly RING queued requests there and have never held
    more (c busy servers: queued = accepted - completed - c)."""
    m, kw = CM.ring_case(name)
    c = int(m.entities["i0"][1])
    out, hw = HW.run(m, O.make_params(window_end_ns=CM.ring_cut(kw), **{k: v for k, v in kw.items() if k != "queue_ring"}))
    st = out["entity_stats"][:, 1]
    queued = np.maximum(0, st["c0"] - st["c2"] - c)
    assert ((queued == CM.RING) & (hw["queue"][:, 1] == CM.RING)).any()


@pytest.mark.parametrize("row", ["wide", "rpw2"])
def test_now_tier_ensembles_straddle_both_boundaries(row):
    n = CM.now_replicas(row, H100_SMS)
    _, hw = HW.run(CM.now_farm(), O.make_params(**CM.now_kw(n)))
    straddles(hw["now"], HW.HS_W_NCAP, "now tier")
    straddles(hw["now"], HW.HS_T_KS, "the shared-memory part of the thread engine's now tier")    # 4 shared, the 5th in the block
    # the warp engine moves a popped future event into its now tier first: never with 24 others pending here
    assert not ((hw["now_pop"] >= HW.HS_W_NCAP) & (hw["now"] <= HW.HS_W_NCAP)).any()
    assert (hw["future"] <= HW.fel_slots(CM.now_farm())).all() and hw["queue"].max() < CM.NOW_RING // 4


def test_future_slot_ensemble_straddles_the_slots():
    m = CM.cache_load()
    _, hw = HW.run(m, O.make_params(**CM.FEL_KW))
    straddles(hw["future"], HW.fel_slots(m), "future-event slots")
    assert (hw["now"] <= HW.HS_W_NCAP).all()


def test_linked_ensemble_straddles_outbox_and_inbox():
    lm = CM.linked_tandem()
    _, _, _, hw = HW.run_linked(lm, CM.linked_params(lm), end_ns=CM.LINKED_KW["end_ns"], cseed=CM.LINKED_KW["seed"])
    straddles(hw[0]["outbox"], CM.OUTBOX_CAP, "outbox")
    straddles(hw[1]["inbox"], CM.INBOX_CAP, "inbox")
    assert not hw[1]["outbox"].any() and not hw[0]["inbox"].any()
