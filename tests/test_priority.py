"""PriorityQueue servers (components/queue_policy.py:189-287) with PriorityByKey priorities, CPU part: the priority
oracle (tests/layered_oracle.c) against the unmodified reference's fixtures, bit for bit; the lowering's acceptance
and refusals; the C-ABI's validation; sweeps of different priority tables never sharing a launch.  The device engines
run the same models in tests/test_gpu_priority.py."""
import math
import os

import numpy as np
import pytest

import golden_lib as G
import oracle_lib as O
import priority_models as PM
import layered_oracle_lib as LO
import happysim_b200 as hs
from happysim_b200 import _abi as A
from happysim_b200 import api, engine, lowering, results

FIXTURES = sorted(PM.fixture_models())
RANDOM = np.load(os.path.join(G.GOLDEN_DIR, "prio_random_models.npz"))


def fixture_params(z, kw, n_replicas=1, **extra):
    return O.make_params(seed=kw["seed"], rid_base=kw["rid_base"], end_ns=kw["end_ns"], n_replicas=n_replicas,
                         **G.caps(z), **extra)


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_model_is_what_the_generator_built(name):
    model, _, z = G.load(f"prio_{name}")
    want = PM.fixture_models()[name][0]
    assert model.entities.tobytes() == want.entities.tobytes()
    assert model.profile_table.tobytes() == want.profile_table.tobytes()


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_matches_the_reference(name):
    model, kw, z = G.load(f"prio_{name}")
    engine.validate_model(model)
    G.check_against(z, LO.run(model, fixture_params(z, kw)))


def test_fixtures_exercise_what_they_are_named_for():
    _, _, z = G.load("prio_bounded_drops")
    assert int(z["entity_stats"][0][1]["c1"]) > 0                      # the bounded heap dropped
    _, _, z = G.load("prio_probe_depth")
    assert int(z["summaries"][0]["n_sink_samples"]) > 0
    # the tie fixture: two constant sources tick at the same nanosecond, at first also with the constant service's
    # ends (the ticks then drift by the float sum's rounding), and equal priorities queue up behind each other
    model, kw, z = G.load("prio_tie_insertion_order")
    rec = z["records"]
    ticks = rec["time_ns"][rec["kind"] == A.HS_EV_SOURCE_TICK]
    ends = rec["time_ns"][rec["kind"] == A.HS_EV_CONTINUATION]
    assert len(np.intersect1d(ticks, ends)) >= 5 and len(np.unique(ticks)) <= len(ticks) // 2 + 1
    assert int(z["entity_stats"][0][2]["c0"]) - int(z["entity_stats"][0][2]["c2"]) > 50      # still waiting at the end


def test_priority_order_differs_from_fifo():
    """The same model with FIFO queues gives another event order: the fixtures do test the priority order."""
    model, kw, z = G.load("prio_mm1_two_class")
    fifo = hs.FlatModel(entities=model.entities.copy(), names=model.names)
    fifo.entities["i1"][:], fifo.entities["i3"][:] = A.HS_Q_FIFO, 0
    out = O.oracle_run(fifo, fixture_params(z, kw))
    assert int(out["summaries"][0]["order_hash"]) != int(z["summaries"][0]["order_hash"])


def test_windows_resume_with_waiting_requests():
    """The cut instants of the windowed runs in tests/test_gpu_priority.py fall where the priority heaps are not empty."""
    for name in ("c4", "rr8", "bounded_drops", "tie_insertion_order"):
        model, kw, z = G.load(f"prio_{name}")
        end_ns = kw["end_ns"]
        for c in (end_ns // 5 + 7, end_ns // 2 + 3, (4 * end_ns) // 5):
            part = LO.run(model, O.make_params(seed=kw["seed"], end_ns=end_ns, window_end_ns=c, n_replicas=5))
            st = part["entity_stats"]
            srv = model.ids_of(A.HS_ENT_SERVER)
            waiting = sum(int(st[r][i]["c0"]) - int(st[r][i]["c2"]) - min(int(model.entities["i0"][i]), int(st[r][i]["c0"]) - int(st[r][i]["c2"]))
                          for r in range(5) for i in srv)
            assert waiting > 0, (name, c)


@pytest.mark.parametrize("seed", PM.RANDOM_SEEDS)
def test_oracle_matches_the_reference_on_random_models(seed):
    model, end_s, _ = PM.random_priority_model(seed)
    engine.validate_model(model)
    out = LO.run(model, O.make_params(seed=int(RANDOM["base_seed"]) + seed, end_ns=int(end_s * 1e9)))
    ws, s = RANDOM[f"s{seed}_summary"][0], out["summaries"][0]
    for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
        assert int(s[f]) == int(ws[f]), (seed, f)
    assert out["entity_stats"][0].tobytes() == RANDOM[f"s{seed}_stats"][0].tobytes()


def test_random_models_mix_the_policies():
    pols = [int(x) for s in PM.RANDOM_SEEDS for m in [PM.random_priority_model(s)[0]]
            for x in m.entities["i1"][m.entities["kind"] == A.HS_ENT_SERVER]]
    assert {A.HS_Q_FIFO, A.HS_Q_LIFO, A.HS_Q_PRIORITY} <= set(pols)
    drops = [int(RANDOM[f"s{s}_stats"][0]["c1"][i]) for s in PM.RANDOM_SEEDS
             for i in PM.random_priority_model(s)[0].ids_of(A.HS_ENT_SERVER)]
    assert sum(drops) > 0


# ---- the lowering ---------------------------------------------------------------------------------------------
def build(policy, *, K=4, second_source=None, caching=False, faults=False):
    sink = hs.Sink("Sink")
    if caching:
        srv = hs.CachingServer("Srv", cache_capacity=K + 1)
        srv._queue = api._Queue("Srv.queue", policy)
    else:
        srv = hs.Server("Srv", concurrency=1, service_time=hs.ExponentialLatency(0.1), queue_policy=policy, downstream=sink)
    ctx = hs.UniformKeyContext(K) if K else None
    srcs = [hs.Source.poisson(rate=5.0, name="Src", event_provider=hs.SimpleEventProvider(srv, context_fn=ctx))]
    if second_source is not None:
        srcs.append(hs.Source.poisson(rate=5.0, name="Src2", event_provider=hs.SimpleEventProvider(srv, context_fn=second_source)))
    sched = None
    if faults:
        sched = hs.FaultSchedule()
        sched.add(hs.CrashNode("Srv", at=1.0))
    return hs.lower(srcs, [srv, sink], fault_schedule=sched)


def test_lowering_accepts_priority_by_key():
    vals = [3, -0.0, 2.5, True]
    model, objs = build(hs.PriorityQueue(capacity=7, key=hs.PriorityByKey(vals)))
    i = model.ids_of(A.HS_ENT_SERVER)[0]
    row = model.entities[i]
    assert int(row["i1"]) == A.HS_Q_PRIORITY and int(row["l0"]) == 7
    tab = model.profile_table[int(row["i3"]) - 1: int(row["i3"]) - 1 + 4]
    assert tab.tobytes() == np.array([3.0, -0.0, 2.5, 1.0]).tobytes()
    engine.validate_model(model)


def test_priority_by_key_is_the_references_key():
    class Ev:
        context = {"metadata": {"client_id": 2}}
    assert hs.PriorityByKey([5, 6, -1.5])(Ev()) == -1.5


@pytest.mark.parametrize("case, match", [
    (dict(policy=hs.PriorityQueue(key=lambda e: 0.0)), "PriorityByKey"),
    (dict(policy=hs.PriorityQueue()), "TypeError"),
    (dict(policy=hs.PriorityQueue(key=hs.PriorityByKey([0, 1])), K=0), "no source"),
    (dict(policy=hs.PriorityQueue(key=hs.PriorityByKey([0, 1])), K=4), "2 values"),
    (dict(policy=hs.PriorityQueue(key=hs.PriorityByKey([0, math.nan, 1, 2]))), "NaN"),
    (dict(policy=hs.PriorityQueue(key=hs.PriorityByKey([0, 2 ** 53 + 1, 1, 2]))), "exactly"),
    (dict(policy=hs.PriorityQueue(key=hs.PriorityByKey([0, "1", 1, 2]))), "str"),
    (dict(policy=hs.PriorityQueue(key=hs.PriorityByKey([0, np.int64(1), 1, 2]))), "int64"),
    (dict(policy=hs.PriorityQueue(key=hs.PriorityByKey([0, 1, 2, 3])), caching=True), "queue policy PriorityQueue"),
    (dict(policy=hs.PriorityQueue(key=hs.PriorityByKey([0, 1, 2, 3])), second_source=None, faults=True), "fault"),
])
def test_lowering_refusals(case, match):
    with pytest.raises(lowering.UnsupportedModelError, match=match):
        build(**case)


def test_lowering_refuses_a_request_without_a_key():
    class NoKey:                     # a second source whose requests carry no routing key
        key_population = 0
    with pytest.raises(lowering.UnsupportedModelError, match="arbitrary context_fn|draws none"):
        build(hs.PriorityQueue(key=hs.PriorityByKey([0, 1, 2, 3])), second_source=NoKey())
    sink = hs.Sink("Sink")
    srv = hs.Server("Srv", queue_policy=hs.PriorityQueue(key=hs.PriorityByKey([0, 1, 2, 3])), downstream=sink)
    keyed = hs.Source.poisson(rate=5.0, name="A", event_provider=hs.SimpleEventProvider(srv, context_fn=hs.UniformKeyContext(4)))
    plain = hs.Source.poisson(rate=5.0, name="B", target=srv)
    with pytest.raises(lowering.UnsupportedModelError, match="'B' draws none"):
        hs.lower([keyed, plain], [srv, sink])


def test_int_priorities_up_to_two_to_the_53_lower_exactly():
    model, _ = build(hs.PriorityQueue(key=hs.PriorityByKey([2 ** 53, -(2 ** 53), 0, 1])))
    assert list(model.profile_table[:2]) == [float(2 ** 53), -float(2 ** 53)]


# ---- the C-ABI's checks --------------------------------------------------------------------------------------
def _mm1(values, K=4, **kw):
    b = hs.ModelBuilder()
    src = b.source(rate=5.0, key_population=K)
    srv = b.server(priorities=values, **kw)
    b.set_target(src, srv); b.set_target(srv, b.sink())
    return b.build()


def test_validation():
    engine.validate_model(_mm1([0.0, 1.0, 2.0, 3.0]))
    for bad, match in ((_mm1([0.0, 1.0]), "priority table out of range"),
                       (_mm1([0.0, math.nan, 2.0, 3.0]), "NaN"),
                       (_mm1([0.0, 1.0, 2.0, 3.0], K=0), "routing key")):
        with pytest.raises(engine.EngineError, match=match):
            engine.validate_model(bad)
    m = _mm1([0.0, 1.0, 2.0, 3.0])
    m.entities["i3"][1] = 0
    with pytest.raises(engine.EngineError, match="priority table out of range"):
        engine.validate_model(m)
    m = hs.mm1()
    m.entities["i3"][1] = 1
    with pytest.raises(engine.EngineError, match="reserved"):
        engine.validate_model(m)
    m = hs.mm1()
    m.entities["i1"][1] = 3
    with pytest.raises(engine.EngineError, match="bad queue policy"):
        engine.validate_model(m)


def test_caching_server_row_keeps_fifo_or_lifo():
    b = hs.ModelBuilder()
    src = b.source(rate=5.0, key_population=4)
    cs = b.cache_server(key_slots=4)
    b.set_target(src, cs)
    m = b.build()
    m.entities["i1"][cs] = A.HS_Q_PRIORITY
    with pytest.raises(engine.EngineError, match="bad queue policy"):
        engine.validate_model(m)


# ---- sweeps: different priority tables are different topologies ------------------------------------------------
def test_same_topology_splits_on_the_priority_table():
    a, b, c = _mm1([0.0, 1.0, 2.0, 3.0]), _mm1([0.0, 1.0, 2.0, 3.0]), _mm1([3.0, 1.0, 2.0, 0.0])
    assert api._same_topology(a, b)
    assert not api._same_topology(a, c)
    f = hs.mm1()
    f.entities["d0"][0] = 5.0
    assert not api._same_topology(a, f)


# ---- write-back -------------------------------------------------------------------------------------------------
def test_write_back_publishes_the_insert_counter():
    policy = hs.PriorityQueue(capacity=3, key=hs.PriorityByKey([1, 0, 1, 0]))
    model, objs = build(policy)
    out = LO.run(model, O.make_params(seed=5, end_ns=20 * 10 ** 9, record_cap=4000, sample_cap=4000, service_cap=4000))
    results.write_back(model, objs, out, 0, hs.Instant)
    i = model.ids_of(A.HS_ENT_SERVER)[0]
    assert policy._insert_counter == objs[i].stats_accepted == int(out["entity_stats"][0][i]["c0"]) > 0
    assert objs[i].stats_dropped > 0


# ---- linked partitions ------------------------------------------------------------------------------------------
def _linked(values_b, pop_b=6):
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", service_time=hs.ExponentialLatency(0.012), downstream=sink,
                   queue_policy=hs.PriorityQueue(key=hs.PriorityByKey(values_b)))
    sa = hs.Server("A.server", service_time=hs.ExponentialLatency(0.02), downstream=sb)
    src = hs.Source.poisson(rate=45.0, name="Src", event_provider=hs.SimpleEventProvider(sa, context_fn=hs.UniformKeyContext(6)))
    src_b = hs.Source.poisson(rate=30.0, name="SrcB", event_provider=hs.SimpleEventProvider(sb, context_fn=hs.UniformKeyContext(pop_b)))
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src]),
             hs.SimulationPartition("B", entities=[sb, sink], sources=[src_b])]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=hs.ConstantLatency(0.05))
    return hs.ParallelSimulation(parts, duration=6.0, links=[link], seed=11)


def test_linked_priority_table_covers_every_partitions_keys():
    ps = _linked([1, 1, 0, 1, 1, 1])
    for q, m in enumerate(ps._linked.models):
        engine.validate_model(m, partition=True)
    # B's own source draws 3 keys, A's requests arrive with 6: B's table must cover 6
    with pytest.raises(lowering.UnsupportedModelError, match="every partition"):
        _linked([1, 0, 1], pop_b=3)
