"""PriorityQueue servers on the device: the binary heap in each server's queue ring (csrc/hs_warp_engine.cuh, hs_pq_push /
hs_pq_pop), on both general engines, against the priority oracle (tests/layered_oracle.c) for every replica and the
unmodified reference's fixtures for the fixture's replica -- event records, order hashes, Sink samples, service times
and statistics, bit for bit, with recorder rings that wrap.  Also: runs cut into windows that resume with non-empty
heaps, the thread engine's kernels by ensemble size, a queue ring that starts too small and grows, the engine choice,
a sweep, and a linked ParallelSimulation."""
import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import oracle_lib as O
import priority_models as PM
import layered_oracle_lib as LO
from happysim_b200 import _abi as A, engine
from happysim_b200.linked import LinkedRun
from test_gpu_lane_parity import assert_same
from test_gpu_launch_geometry import GEOMETRY, check_thread_geometry
from test_priority import FIXTURES, RANDOM, fixture_params

pytestmark = pytest.mark.gpu

WRAP = dict(record_cap=29, sample_cap=7, service_cap=5)


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("eng_id", [1, 3])
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_on_the_general_engines(eng, name, eng_id):
    model, kw, z = G.load(f"prio_{name}")
    eng.upload(model)
    p = fixture_params(z, kw, n_replicas=6, queue_ring=256, engine=eng_id)
    eng.run(p)
    got = eng.read_outputs()
    G.check_against(z, got, 0)
    assert_same(got, LO.run(model, p))
    p = O.make_params(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=6, queue_ring=256, engine=eng_id, **WRAP)
    eng.run(p)
    got, want = eng.read_outputs(), LO.run(model, p)
    assert np.all(want["summaries"]["events_processed"] > WRAP["record_cap"])          # the rings wrap
    assert_same(got, want)


@pytest.mark.parametrize("eng_id", [1, 3])
@pytest.mark.parametrize("name", ["c4", "rr8", "bounded_drops", "tie_insertion_order", "probe_depth"])
def test_fixture_cut_into_windows(eng, name, eng_id):
    """Three cuts while the heaps hold waiting requests (the oracle's depth probe / queue lengths say they do)."""
    model, kw, z = G.load(f"prio_{name}")
    end_ns = kw["end_ns"]
    cuts = [end_ns // 5 + 7, end_ns // 2 + 3, (4 * end_ns) // 5]
    base = dict(seed=kw["seed"], n_replicas=5, queue_ring=256, **WRAP)
    want = LO.run(model, O.make_params(end_ns=end_ns, **base))
    eng.upload(model)
    eng.run(engine.make_params(end_ns=end_ns, window_end_ns=cuts[0], engine=eng_id, **base))
    for c in cuts[1:]:
        eng.run(engine.make_params(end_ns=end_ns, window_end_ns=c, resume=1, engine=eng_id, **base))
    eng.run(engine.make_params(end_ns=end_ns, resume=1, engine=eng_id, **base))
    assert_same(eng.read_outputs(), want)


@pytest.mark.parametrize("seed", PM.RANDOM_SEEDS)
def test_random_model_on_every_general_engine(eng, seed):
    model, end_s, _ = PM.random_priority_model(seed)
    kw = dict(seed=int(RANDOM["base_seed"]) + seed, end_ns=int(end_s * 1e9), n_replicas=5, record_cap=12000,
              sample_cap=1500, service_cap=1500, queue_ring=1024)
    want = LO.run(model, O.make_params(**kw))
    ws = RANDOM[f"s{seed}_summary"][0]
    for f in ("events_processed", "order_hash", "n_sink_samples", "n_service_samples"):
        assert int(want["summaries"][0][f]) == int(ws[f])
    assert want["entity_stats"][0].tobytes() == RANDOM[f"s{seed}_stats"][0].tobytes()
    eng.upload(model)
    for eng_id in (0, 1, 3):
        eng.run(engine.make_params(engine=eng_id, **kw))
        assert_same(eng.read_outputs(), want)
    # cut into three windows on both general engines
    cuts = [kw["end_ns"] // 4, kw["end_ns"] // 2 + 1, (3 * kw["end_ns"]) // 4]
    for eng_id in (1, 3):
        eng.run(engine.make_params(engine=eng_id, window_end_ns=cuts[0], **kw))
        for c in cuts[1:]:
            eng.run(engine.make_params(engine=eng_id, window_end_ns=c, resume=1, **kw))
        eng.run(engine.make_params(engine=eng_id, resume=1, **kw))
        assert_same(eng.read_outputs(), want)


@pytest.mark.parametrize("row", sorted(GEOMETRY))
def test_thread_engine_kernels(eng, sm, row):
    """rr8 at every ensemble size that selects a thread-engine kernel, every replica against the oracle."""
    model, kw, z = G.load("prio_rr8")
    n = GEOMETRY[row][0](sm)
    p = dict(seed=kw["seed"], end_ns=int(0.6e9), n_replicas=n, queue_ring=32, **WRAP)
    eng.upload(model)
    eng.run(engine.make_params(engine=3, **p))
    check_thread_geometry(eng.last_launch(), row, n)
    got = eng.read_outputs()
    want = LO.run(model, O.make_params(**p), chunk=1024)
    assert not (want["summaries"]["status"] & A.HS_ST_QUEUE_OVERFLOW).any()
    assert_same(got, want)


def _mm1_sim(end_s=30.0):
    sink = hs.Sink("Sink")
    srv = hs.Server("Srv", service_time=hs.ExponentialLatency(0.1),
                    queue_policy=hs.PriorityQueue(key=hs.PriorityByKey([0, 1, 1, 2, 1])), downstream=sink)
    src = hs.Source.poisson(rate=11.0, name="Src", event_provider=hs.SimpleEventProvider(srv, context_fn=hs.UniformKeyContext(5)))
    return hs.Simulation(end_time=hs.Instant.from_seconds(end_s), sources=[src], entities=[srv, sink], seed=9)


def test_a_queue_ring_too_small_grows():
    """Arrivals outpace service: the heap outgrows a 4-entry ring, the launch is repeated with larger rings, and the
    result equals a run that started large enough."""
    small = _mm1_sim().run_ensemble(64, queue_ring=4, record_cap=4000, sample_cap=2000, service_cap=2000)
    big = _mm1_sim().run_ensemble(64, queue_ring=8192, record_cap=4000, sample_cap=2000, service_cap=2000)
    assert small["queue_ring"] > 4 and big["queue_ring"] == 8192
    assert not small["status"].any() and not big["status"].any()
    for k in ("summaries", "entity_stats", "records", "sink_samples", "service_samples"):
        assert small[k].tobytes() == big[k].tobytes(), k


def test_engine_choice():
    sim = _mm1_sim(end_s=5.0)
    e = engine.Engine(0)
    try:
        e.upload(sim.model)
        e.run(engine.make_params(seed=1, end_ns=5 * 10 ** 9, n_replicas=3))
        assert e.last_launch()["engine"] == 3
        with pytest.raises(engine.EngineError, match="PriorityQueue"):
            e.run(engine.make_params(seed=1, end_ns=5 * 10 ** 9, engine=2))
    finally:
        e.close()


def test_sweep_of_two_priority_tables():
    """Two tables are two topologies: run_sweep launches each group once; configurations that differ in rate only
    share a launch as its cells.  Every result equals that configuration's own run."""
    def build(values, rate):
        def fn():
            sink = hs.Sink("Sink")
            srv = hs.Server("Srv", service_time=hs.ExponentialLatency(0.1),
                            queue_policy=hs.PriorityQueue(key=hs.PriorityByKey(values)), downstream=sink)
            src = hs.Source.poisson(rate=rate, name="Src",
                                    event_provider=hs.SimpleEventProvider(srv, context_fn=hs.UniformKeyContext(4)))
            return hs.Simulation(end_time=hs.Instant.from_seconds(20.0), sources=[src], entities=[srv, sink], seed=3)
        return fn
    cfgs = [hs.RunConfig("a", build([0, 1, 1, 1], 8.0)), hs.RunConfig("b", build([0, 1, 1, 1], 9.0)),
            hs.RunConfig("c", build([1, 1, 0, 0], 8.0))]
    assert hs.api._same_topology(cfgs[0].build_fn().model, cfgs[1].build_fn().model)
    assert not hs.api._same_topology(cfgs[0].build_fn().model, cfgs[2].build_fn().model)
    res = hs.ParallelRunner().run_sweep(cfgs)
    for cfg, r in zip(cfgs, res):
        own = cfg.build_fn().run()
        assert r.status == 0
        assert (r.summary.total_events_processed, r.summary.duration_s) == (own.total_events_processed, own.duration_s), cfg.name
    assert sorted(sorted(g) for g in hs.api._group_by_topology([c.build_fn() for c in cfgs])) == [[0, 1], [2]]


def test_linked_partition_with_a_priority_server():
    """A priority server in each partition; B's also takes requests over the link, whose sort indices come from A's
    counter: there the payloads' sort indices are not the insertion order."""
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", service_time=hs.ExponentialLatency(0.012), downstream=sink,
                   queue_policy=hs.PriorityQueue(key=hs.PriorityByKey([1, 1, 0, 1, 1, 1])))
    sa = hs.Server("A.server", service_time=hs.ExponentialLatency(0.02), downstream=sb,
                   queue_policy=hs.PriorityQueue(capacity=12, key=hs.PriorityByKey([2, 0, 1, 1, 0, 2])))
    src = hs.Source.poisson(rate=45.0, name="Src", event_provider=hs.SimpleEventProvider(sa, context_fn=hs.UniformKeyContext(6)))
    src_b = hs.Source.poisson(rate=30.0, name="SrcB", event_provider=hs.SimpleEventProvider(sb, context_fn=hs.UniformKeyContext(6)))
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src]),
             hs.SimulationPartition("B", entities=[sb, sink], sources=[src_b])]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=hs.ConstantLatency(0.05))
    ps = hs.ParallelSimulation(parts, duration=6.0, links=[link], seed=11)
    lm = ps._linked
    for m in lm.models:
        assert int(m.entities["i1"][m.ids_of(A.HS_ENT_SERVER)[0]]) == A.HS_Q_PRIORITY
    nP, n, end_ns = lm.n_partitions, 37, 6 * 10 ** 9
    caps = [dict(record_cap=900, sample_cap=300, service_cap=300) for _ in range(nP)]
    run = LinkedRun(lm)
    try:
        outs, (delivered, lost, over) = run.run(seed=11, end_ns=end_ns, n_replicas=n, caps=caps)
    finally:
        run.close()
    params = [O.make_params(seed=11, end_ns=end_ns, n_replicas=n, rid_base=q, rid_stride=nP + 1, **caps[q]) for q in range(nP)]
    want, wd, wl, _ = LO.run_linked(lm, params, end_ns=end_ns, cseed=11)
    assert np.array_equal(delivered, wd) and np.array_equal(lost, wl) and not over.any()
    for q in range(nP):
        assert_same(outs[q], want[q])
    assert int(want[0]["entity_stats"][:, lm.models[0].ids_of(A.HS_ENT_SERVER)[0]]["c1"].sum()) > 0     # the heap dropped
