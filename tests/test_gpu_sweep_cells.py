"""Sweep cells of every kind of lowered model on the device (tests/sweep_models.py), every replica against the oracle,
which tests/test_sweep_cells.py pins to each cell's own single run.

(a) the random v1 / v2 / fault models with cells on the auto, warp and thread engines, the lane models on the lane
    engine too: load balancers, tandems, LIFO and bounded servers, CachingServers with per-cell TTLs, TDigests with
    per-cell compressions, probes, profiles and node faults, in rings small enough to wrap;
(b) two cell models at the thread engine's geometries and on the warp engine past its resident warps: one with every
    server at c = 1 in every cell (entity-owned heap slots), one whose cells mix c = 1 and c > 1;
(c) cell runs cut in windows on both general engines against the uncut run (the cell is recomputed on resume);
(d) the per-cell reductions (hs_read_cell_totals, hs_read_bucket_totals) of a model that is not an M/M/c;
(e) node faults in cells whose concurrencies differ;
(f) ParallelRunner.run_sweep over CachingServer TTLs and QuantileEstimator compressions, and independent
    ParallelSimulation partitions that differ only in TTL: one launch, each result equal to its configuration's own
    Simulation.run(), and the configurations of tests/golden/sweep_cells.npz equal to the unmodified reference."""
import numpy as np
import pytest

import fault_oracle_lib as FO
import happysim_b200 as hs
import oracle_lib as O
from happysim_b200 import _abi as A, buckets as B, distributed as D, engine
from sweep_models import (CACHE_TTLS, FIXTURE_END_NS, FIXTURE_SEED, TDIGEST_COMPRESSIONS, cell_case, cells_of,
                          fixture_models, has_kind)
from test_gpu_launch_geometry import CAPS, FLAGS, GEOMETRY, assert_same, check_thread_geometry, compare
from test_gpu_random_faults import KEYS, compare_tie_aware
from test_sweep_cells import CASES, check_cells_against_fixture, launch_shape

pytestmark = pytest.mark.gpu

WF_FAULTS = 32                         # HS_WF_FAULTS of csrc/hs_warp_engine.cuh
RING = 2048                            # a cell can run at rho > 1 for its whole horizon: the queue rings hold that
LANE_CASES = [("lane", s) for s in range(1, 9)]


def _id(c):
    return f"{c[0]}-{c[1]}"


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def oracle(model, p):
    return FO.run(model, p) if has_kind(model, A.HS_ENT_FAULT) else O.oracle_run_parallel(model, p)


def check(eng, model, got, want):
    """bit for bit; a faulted model's replicas whose in-run event tied a fault event are compared by their flag only"""
    if has_kind(model, A.HS_ENT_FAULT):
        compare_tie_aware(got, want, KEYS)
        return
    compare(eng, model, got, want)


# ---- (a) every model, every engine ---------------------------------------------------------------------------------------

def lane_eligible(m) -> bool:
    """classify_lane of csrc/hs_engine.cu: Source -> Server (concurrency <= 64 in every cell) -> Sink | Counter | nothing"""
    E, k = m.entities, m.entities["kind"]
    src, srv = np.flatnonzero(k == A.HS_ENT_SOURCE), np.flatnonzero(k == A.HS_ENT_SERVER)
    dst = np.flatnonzero((k == A.HS_ENT_SINK) | (k == A.HS_ENT_COUNTER))
    if len(E) > 3 or len(src) != 1 or len(srv) != 1 or len(src) + len(srv) + len(dst) != len(E):
        return False
    s, v = int(src[0]), int(srv[0])
    return (int(E["i1"][s]) == 0 and int(E["target"][s]) == v and int(E["target"][v]) == (int(dst[0]) if len(dst) else -1)
            and int(m.cell_i0[:, v].max()) <= 64)


@pytest.mark.parametrize("case", CASES + LANE_CASES, ids=_id)
def test_every_engine_matches_the_oracle(eng, case):
    m, end_ns, run_seed, what = cell_case(*case)
    rpc, base, n = launch_shape(case[1], m.n_cells)
    n += m.n_cells * rpc * 2                           # every cell more than once
    kw = dict(seed=run_seed, seed_stride=1, rid_base=3, rid_stride=2, end_ns=end_ns, n_replicas=n, replica_index_base=base,
              replicas_per_cell=rpc, flags=FLAGS, queue_ring=RING, **CAPS)
    want = oracle(m, O.make_params(**kw))
    assert np.median(want["summaries"]["events_processed"]) > CAPS["record_cap"], what       # the rings wrap
    eng.upload(m)
    lane = lane_eligible(m)
    assert lane or case[0] != "lane", what
    for e in ((0, 1, 2, 3) if lane else (0, 1, 3)):
        eng.run(engine.make_params(engine=e, **kw))
        li = eng.last_launch()
        assert li["engine"] == (e if e else (2 if lane else 3)), (e, li)
        assert bool(li["flags"] & WF_FAULTS) == (case[0] == "fault") or li["engine"] == 2, li
        got = eng.read_outputs()
        assert not (got["summaries"]["status"] & A.HS_ST_QUEUE_OVERFLOW).any(), what
        check(eng, m, got, want)


# ---- (b) thread-engine geometries, the warp engine past its resident warps --------------------------------------------

GEO_CASES = {"one": ("v1", 2, "one", 1), "mixed": ("v1", 24, "mixed", 3)}      # name: (generator, seed, concurrency, rpc)
GEO_SCALE = 0.3


def geo_model(name):
    gen, seed, conc, rpc = GEO_CASES[name]
    m, end_ns, run_seed, _ = cell_case(gen, seed, concurrency=conc)
    return m, int(end_ns * GEO_SCALE), run_seed, rpc


def test_geometry_models_pin_the_slot_rule():
    one, mixed = geo_model("one")[0], geo_model("mixed")[0]
    srv = one.entities["kind"] == A.HS_ENT_SERVER
    assert srv.sum() >= 3 and (one.cell_i0[:, srv] == 1).all() and has_kind(one, A.HS_ENT_LB)
    srv = mixed.entities["kind"] == A.HS_ENT_SERVER
    ci = mixed.cell_i0[:, srv]
    assert srv.sum() >= 3 and ((ci == 1).any(axis=0) & (ci > 1).any(axis=0)).all()


@pytest.mark.parametrize("row", ["wide", "rpw1", "rpw2", "rpw32", "warp"])
@pytest.mark.parametrize("name", sorted(GEO_CASES))
def test_every_geometry_matches_the_oracle(eng, sm, name, row):
    m, end_ns, run_seed, rpc = geo_model(name)
    n = 96 * sm + 3 if row == "warp" else GEOMETRY[row][0](sm)      # warp: more replicas than resident warps
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=n, replica_index_base=7, replicas_per_cell=rpc, flags=FLAGS,
              queue_ring=256, **CAPS)
    eng.upload(m)
    eng.run(engine.make_params(engine=1 if row == "warp" else 3, **kw))
    li = eng.last_launch()
    if row == "warp":
        assert (li["engine"], li["kernel"]) == (1, "warp") and n > li["grid"] * li["block"] // 32, li
    else:
        check_thread_geometry(li, row, n)
    got = eng.read_outputs()
    assert not (got["summaries"]["status"] & A.HS_ST_QUEUE_OVERFLOW).any()
    want = O.oracle_run_parallel(m, O.make_params(**kw))
    assert np.median(want["summaries"]["events_processed"]) > CAPS["record_cap"]
    compare(eng, m, got, want)


# ---- (c) windows --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("eng_id", [1, 3])
@pytest.mark.parametrize("case", CASES[::3], ids=_id)
def test_windows_equal_the_uncut_run(eng, case, eng_id):
    m, end_ns, run_seed, _ = cell_case(*case)
    rpc, base, n = launch_shape(case[1], m.n_cells)
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=n + 16, replica_index_base=base, replicas_per_cell=rpc,
              rid_stride=1, engine=eng_id, flags=FLAGS, queue_ring=RING, **CAPS)
    eng.upload(m)
    eng.run(engine.make_params(**kw))
    whole = eng.read_outputs()
    eng.run(engine.make_params(window_end_ns=end_ns // 7 + 3, **kw))
    eng.run(engine.make_params(window_end_ns=end_ns // 2 + 1, resume=1, **kw))
    eng.run(engine.make_params(window_end_ns=end_ns - 1, resume=1, **kw))
    eng.run(engine.make_params(resume=1, **kw))
    assert eng.last_launch()["engine"] == eng_id
    got = eng.read_outputs()
    for k in KEYS:
        if whole[k] is not None:
            assert got[k].tobytes() == whole[k].tobytes(), k


# ---- (d) per-cell reductions ---------------------------------------------------------------------------------------------

def _close(a, b, n):
    return a == b or abs(a - b) <= 4 * n * np.finfo(float).eps * max(abs(a), abs(b))


def test_cell_totals_of_a_load_balanced_model(eng):
    m, end_ns, run_seed, _ = cell_case("v1", 24, concurrency="mixed")
    rpc, base = 3, 5
    n = 400 * m.n_cells + 7
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=n, replica_index_base=base, replicas_per_cell=rpc,
              flags=A.HS_RUN_ORDER_HASH | A.HS_RUN_HISTOGRAM, queue_ring=RING)
    eng.upload(m)
    eng.run(engine.make_params(engine=3, **kw))
    got = eng.read_outputs()
    assert_same(got, O.oracle_run_parallel(m, O.make_params(**kw)), keys=["summaries", "entity_stats", "histograms"])
    want = D.cell_totals_from_outputs(m, got, m.n_cells, rpc, base)
    cell = cells_of(n, m.n_cells, base, rpc)
    for c, ((d, h), (wt, wh)) in enumerate(zip(eng.read_cell_totals(m.n_cells), want)):
        wd = engine.totals_to_dict(wt)
        assert np.array_equal(h, wh), c
        assert wd["sink_events"] > 0, c
        for k, v in wd.items():
            if isinstance(v, float) and k.startswith("sum"):
                assert _close(d[k], v, int((cell == c).sum())), (c, k, d[k], v)
            else:
                assert d[k] == v, (c, k, d[k], v)


def test_bucket_totals_of_a_load_balanced_model_with_a_probe(eng):
    m, end_ns, run_seed, _ = cell_case("v1", 2, concurrency="any")
    assert has_kind(m, A.HS_ENT_PROBE) and has_kind(m, A.HS_ENT_LB)
    rpc, base = 2, 3
    n = 300 * m.n_cells + 5
    w = 0.25
    nb = int(end_ns / 1e9 / w) + 2
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=n, replica_index_base=base, replicas_per_cell=rpc, rid_stride=1,
              queue_ring=RING, flags=0)
    eng.upload(m)
    eng.set_buckets(w, nb)
    try:
        eng.run(engine.make_params(engine=3, **kw))
        got, _ = eng.read_buckets(nb)
        tot = eng.read_bucket_totals(m.n_cells, got.shape[1], nb)
    finally:
        eng.set_buckets(0.0, 0)
    assert got.shape[1] >= 2 and int(got["count"].sum()) > 0
    want = B.cell_totals_reference(got, m.n_cells, replica_index_base=base, replicas_per_cell=rpc)
    assert tot.tobytes() == want.tobytes()
    cell = cells_of(n, m.n_cells, base, rpc)
    for c in range(m.n_cells):
        assert (tot[c]["count"] == got[cell == c]["count"].sum(0)).all()


# ---- (e) node faults in cells of different concurrency ---------------------------------------------------------------------

def crashes_a_varied_server(m):
    E = m.entities
    for i in m.ids_of(A.HS_ENT_FAULT):
        t = int(E["target"][i])
        if E["i1"][i] and not E["i2"][i] and int(E["kind"][t]) == A.HS_ENT_SERVER and len(set(m.cell_i0[:, t])) > 1:
            return True
    return False


FAULT_CELL_SEEDS = [s for s in range(40) if crashes_a_varied_server(cell_case("fault", s, concurrency="mixed")[0])][:4]


@pytest.mark.parametrize("seed", FAULT_CELL_SEEDS)
def test_faults_in_cells_of_different_concurrency(eng, seed):
    m, end_ns, run_seed, what = cell_case("fault", seed, concurrency="mixed")
    kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=3 * m.n_cells * 4 + 1, replica_index_base=2, replicas_per_cell=3,
              rid_stride=1, flags=FLAGS, queue_ring=RING, **CAPS)
    want = FO.run(m, O.make_params(**kw))
    eng.upload(m)
    for e in (1, 3):
        eng.run(engine.make_params(engine=e, **kw))
        li = eng.last_launch()
        assert li["engine"] == e and li["flags"] & WF_FAULTS, li
        compare_tie_aware(eng.read_outputs(), want, KEYS)


def test_fault_cell_seeds_exist():
    assert len(FAULT_CELL_SEEDS) == 4


# ---- (f) the public API ---------------------------------------------------------------------------------------------------

def _cache_sim(ttl, replica):
    caches = [hs.CachingServer(f"Cache{i}", server_id=i, cache_capacity=13, cache_ttl_s=ttl, cache_read_latency_s=0.001,
                               datastore_read_latency_s=0.02, processing_latency_s=0.004) for i in range(3)]
    lb = hs.LoadBalancer("LB", backends=caches, strategy=hs.RoundRobin())
    src = hs.Source.poisson(rate=200.0, name="Src", event_provider=hs.SimpleEventProvider(lb, context_fn=hs.UniformKeyContext(12)))
    return hs.Simulation(end_time=hs.Instant(FIXTURE_END_NS), sources=[src], entities=[*caches, lb], seed=FIXTURE_SEED,
                         replica=replica), caches


def _tdigest_sim(compression, replica):
    qe = hs.QuantileEstimator("Latency", compression=compression)
    servers = [hs.Server(f"Srv{i}", service_time=hs.ExponentialLatency(0.025), downstream=qe) for i in range(4)]
    lb = hs.LoadBalancer("LB", backends=servers, strategy=hs.RoundRobin())
    src = hs.Source.poisson(rate=120.0, target=lb, name="Src")
    return hs.Simulation(end_time=hs.Instant(FIXTURE_END_NS), sources=[src], entities=[qe, *servers, lb], seed=FIXTURE_SEED,
                         replica=replica), [qe]


def _cache_state(caches):
    return [(c.stats.requests_processed, c.stats.cache_hits, c.stats.cache_misses, c.cache_size, c.stats_accepted,
             sorted(c._insert_times.items())) for c in caches]


def _tdigest_state(qes):
    return [(q._tdigest._means, q._tdigest._counts, q._tdigest._total_count, q._tdigest._min_value, q._tdigest._max_value,
             q._tdigest._buffer) for q in qes]


def _fixture_rows(name, sim, c):
    """the fixture's summary and statistics of configuration c, with the lowered model's rows in the fixture model's order"""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sweep_cells.npz"))
    fm = fixture_models()[name][1][c]
    order = [fm.names.index(nm) for nm in sim.model.names]
    return z[f"{name}_c{c}_summary"][0], z[f"{name}_c{c}_stats"][0][order]


@pytest.mark.parametrize("name", ["cache_ttl", "tdigest_compression"])
def test_run_sweep_gives_every_configuration_its_own_value(name):
    mk, state, vals = ((_cache_sim, _cache_state, CACHE_TTLS) if name == "cache_ttl" else
                       (_tdigest_sim, _tdigest_state, TDIGEST_COMPRESSIONS))
    built = {}

    def build(c):
        def f():
            sim, objs = mk(vals[c], c)
            built[c] = (sim, objs)
            return sim
        return f
    cfgs = [hs.RunConfig(name=f"{name}{c}", build_fn=build(c), seed=FIXTURE_SEED) for c in range(len(vals))]
    res = hs.ParallelRunner().run_sweep(cfgs)
    states = []
    for c in range(len(vals)):
        sim, objs = built[c]
        assert sim.last_run_info["batched_with"] == len(vals) and res[c].status == 0       # one launch
        s = state(objs)
        states.append(repr(s))
        alone, objs2 = mk(vals[c], c)
        one = alone.run()
        assert alone.last_run_info["batched_with"] == 1
        assert res[c].summary.total_events_processed == one.total_events_processed, c
        assert s == state(objs2), (name, c)
        ws, wstats = _fixture_rows(name, sim, c)
        assert one.total_events_processed == int(ws["events_processed"]), c
        for i, obj in enumerate(objs):
            k = sim.model.names.index(obj.name)
            if name == "cache_ttl":
                assert (obj.stats.requests_processed, obj.stats.cache_misses, obj.stats.cache_hits, obj.cache_size) == \
                    (int(wstats[k]["c2"]), int(wstats[k]["c3"]), int(wstats[k]["f0"]), int(wstats[k]["f1"])), (c, obj.name)
            else:
                assert obj.sample_count == int(wstats[k]["c1"]), (c, obj.name)
    assert len(set(states)) == len(vals)                   # every configuration behaves differently


def test_parallel_simulation_partitions_that_differ_only_in_ttl():
    def part(c):
        sim, caches = _cache_sim(CACHE_TTLS[c], 0)
        return hs.SimulationPartition(f"p{c}", entities=sim._entities, sources=sim._sources), caches
    parts = [part(c) for c in range(len(CACHE_TTLS))]
    ps = hs.ParallelSimulation([p for p, _ in parts], duration=FIXTURE_END_NS / 1e9, seed=FIXTURE_SEED)
    summ = ps.run()
    assert ps.launch_groups == [[p.name for p, _ in parts]]
    states = []
    for c, (p, caches) in enumerate(parts):
        alone, caches2 = _cache_sim(CACHE_TTLS[c], c)          # partition c: replica word c
        s = alone.run()
        assert summ.partitions[p.name].total_events_processed == s.total_events_processed, c
        assert _cache_state(caches) == _cache_state(caches2), c
        ws, wstats = _fixture_rows("cache_ttl", alone, c)
        assert s.total_events_processed == int(ws["events_processed"])
        assert [cs.stats.cache_misses for cs in caches] == \
            [int(wstats[alone.model.names.index(cs.name)]["c3"]) for cs in caches2], c
        states.append(repr(_cache_state(caches)))
    assert len(set(states)) == len(CACHE_TTLS)


@pytest.mark.parametrize("name", ["cache_ttl", "tdigest_compression"])
def test_fixture_sweeps_on_every_engine(eng, name):
    """the fixture's cell models as one launch, one replica per cell: every engine equals the reference"""
    m, _ = fixture_models()[name]
    kw = dict(seed=FIXTURE_SEED, end_ns=FIXTURE_END_NS, n_replicas=m.n_cells, rid_stride=1, queue_ring=RING)
    eng.upload(m)
    for e in (0, 1, 3):
        eng.run(engine.make_params(engine=e, **kw))
        assert eng.last_launch()["engine"] == (e or 3)
        check_cells_against_fixture(name, m, eng.read_outputs(), range(m.n_cells))
