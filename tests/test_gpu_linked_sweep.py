"""Linked ParallelSimulations as the cells of one ensemble, on the device: every replica of celled linked runs against
the cell oracle (tests/layered_oracle.c) -- random linked models with per-cell model rows and per-cell link latency
and loss, node faults, replicas_per_cell > 1, a nonzero replica_index_base -- the celled ensemble against each cell's own
ensemble, time buckets per cell, run_sweep over linked configurations, shards, and a sweep-sized point."""
import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import layered_oracle_lib as LO
import linked_fault_models as LF
import linked_sweep_lib as LS
import random_models as RM
from happysim_b200 import _abi as A, api, buckets as B, distributed as D, engine
from happysim_b200.linked import LinkedRun
from happysim_b200.parallel import ParallelSimulation

pytestmark = pytest.mark.gpu

CAPS = dict(record_cap=4096, sample_cap=2048, service_cap=2048)
TIES = A.HS_ST_LINK_TIE | A.HS_ST_FAULT_TIE


def _device(lm, *, seed, end_ns, n, caps=CAPS, base=0, rpc=1, seed_stride=0, rid_stride=None, queue_ring=1024):
    run = LinkedRun(lm)
    try:
        outs, (delivered, lost, over) = run.run(seed=seed, end_ns=end_ns, n_replicas=n, replica_index_base=base, caps=caps,
                                                replicas_per_cell=rpc, seed_stride=seed_stride, rid_stride=rid_stride,
                                                queue_ring=queue_ring)
    finally:
        run.close()
    assert not over.any()
    return outs, delivered, lost


def _oracle(lm, *, seed, end_ns, n, caps=CAPS, base=0, rpc=1):
    ps = LS.partition_params(lm, seed=seed, end_ns=end_ns, n=n, caps=caps, replica_index_base=base, replicas_per_cell=rpc)
    return LO.run_linked_parallel(lm, ps, end_ns=end_ns, cseed=seed, replicas_per_cell=rpc)


def _check(lm, *, seed, end_ns, n, base, rpc, grid=False):
    """every replica of the device's run against the cell oracle.  As in test_gpu_linked's random models, a replica in
    which a delivered event tied with another on time AND index is flagged (HS_ST_LINK_TIE; only grid models can) and
    left out: the oracle restates heapq's order of such a pair, the engines' heaps cannot."""
    outs, delivered, lost = _device(lm, seed=seed, end_ns=end_ns, n=n, base=base, rpc=rpc)
    want, wd, wl, _ = _oracle(lm, seed=seed, end_ns=end_ns, n=n, base=base, rpc=rpc)
    tie = np.zeros(n, bool)
    for o in outs:
        tie |= (o["summaries"]["status"] & A.HS_ST_LINK_TIE) != 0
    assert grid or not tie.any()
    assert int(tie.sum()) <= n // 2, int(tie.sum())
    for r in np.nonzero(~tie)[0]:
        LS.assert_replica_equal(outs, want, r, r, f"replica {r}")
        assert (int(delivered[r]), int(lost[r])) == (int(wd[r]), int(wl[r])), r
    for q, o in enumerate(outs):       # every partition's per-cell totals
        assert len(o["cell_totals"]) == lm.n_cells
        assert sum(int(d["replicas"]) for d, _ in o["cell_totals"]) == n
    return outs


@pytest.mark.parametrize("seed", [0, 4, 11, 17, 26, 40])
def test_random_linked_cells_match_the_oracle(seed):
    lm, end_s, what = RM.random_linked_model(seed)
    celled = LS.celled(lm, seed, 5)
    _check(celled, seed=seed + 300, end_ns=int(end_s * 1e9), n=96, base=7, rpc=3, grid="grid" in what)


@pytest.mark.parametrize("seed", [2, 6, 13])
def test_random_linked_cells_with_node_faults_match_the_oracle(seed):
    lm, end_s, what, _ = LF.random_linked_fault_model(seed)
    celled = LS.celled(lm, seed, 4)
    _check(celled, seed=seed + 400, end_ns=int(end_s * 1e9), n=64, base=0, rpc=2, grid="grid" in what)


def test_lossless_and_lossy_cells_side_by_side():
    lm, kw, _ = G.load_linked("linked_lossy_fanout")
    celled = LS.celled(lm, 1, 3)
    assert (celled.cell_links[0][1, :, 1] == 0).all() and (celled.cell_links[0][2, :, 1] > 0).all()
    _check(celled, seed=kw["seed"], end_ns=kw["end_ns"], n=48, base=1, rpc=1)


def test_sweep_fixture_on_the_device():
    """the reference's run of every configuration (tests/golden/lsweep_cells.npz) as replica k of one celled run"""
    import test_linked_sweep as T
    z = np.load(T.GOLDEN)
    for name in ("tandem", "fanout"):
        lm, seed, end_ns, nc = T.load_sweep_case(z, name)
        outs, delivered, lost = _device(lm, seed=seed, end_ns=end_ns, n=nc, caps=T.sweep_caps(z, name, lm, nc), rid_stride=0)
        T.check_against_sweep_fixture(z, name, lm, outs, delivered, range(nc))


# ---- through the API ----------------------------------------------------------------------------------------------------

def tandem(latency=0.05, loss=0.0, rate=40.0, conc=2, duration=4.0, kind="exp", seed=42):
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=conc, service_time=hs.ExponentialLatency(0.015), downstream=sink)
    sa = hs.Server("A.server", service_time=hs.ExponentialLatency(0.01), downstream=sb)
    src = hs.Source.poisson(rate=rate, target=sa)
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src]), hs.SimulationPartition("B", entities=[sb, sink])]
    lat = hs.ConstantLatency(latency) if kind == "const" else hs.ExponentialLatency(latency)
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=lat, packet_loss=loss)
    return ParallelSimulation(parts, duration=duration, links=[link], seed=seed)


def _configs(**kw):
    return [tandem(0.05, **kw), tandem(0.09, loss=0.1, rate=60.0, **kw), tandem(0.07, conc=1, **kw),
            tandem(0.12, loss=0.3, rate=30.0, conc=3, **kw)]


def _same_outputs(a, b, r_a, r_b, what):
    LS.assert_replica_equal([a[k] for k in a], [b[k] for k in a], r_a, r_b, what)


def test_celled_ensemble_equals_each_cells_own_ensemble_and_shards_compose():
    cells = _configs()
    n, rpc = 64, 4
    outs, delivered, lost = cells[0].run_ensemble(n, cells=cells, replicas_per_cell=rpc)
    own = [c.run_ensemble(n) for c in _configs()]
    for r, c in enumerate(LS.cell_of(n, 0, rpc, 4)):
        o, d, l_ = own[int(c)]
        _same_outputs(outs, o, r, r, f"replica {r}, cell {c}")
        assert (int(delivered[r]), int(lost[r])) == (int(d[r]), int(l_[r]))
    for name, o in outs.items():
        m = cells[0]._linked.models[list(outs).index(name)]
        want = D.cell_totals_from_outputs(m, o, 4, rpc)
        for (d, h), (wt, wh) in zip(o["cell_totals"], want):
            wd = engine.totals_to_dict(wt)
            assert np.array_equal(h, wh) and all(d[k] == wd[k] for k in ("events_processed", "sink_events", "replicas"))
    a = _configs()[0].run_ensemble(24, 0, cells=_configs(), replicas_per_cell=rpc)
    b = _configs()[0].run_ensemble(40, 24, cells=_configs(), replicas_per_cell=rpc)
    for name in outs:
        for key in LS.KEYS:
            if outs[name].get(key) is not None:
                assert np.concatenate([a[0][name][key], b[0][name][key]]).tobytes() == outs[name][key].tobytes(), (name, key)
    assert np.concatenate([a[1], b[1]]).tobytes() == delivered.tobytes()
    assert np.concatenate([a[2], b[2]]).tobytes() == lost.tobytes()


def test_bucket_totals_per_cell():
    """time buckets with p50 / p99: each partition's bucket totals are per cell and equal the numpy reduction of the
    per-replica buckets; every replica's buckets equal its cell's own bucketed ensemble"""
    n, rpc, nc, w, nb = 96, 8, 4, 0.5, 9
    outs, _, _ = _configs()[0].run_ensemble(n, 5, cells=_configs(), replicas_per_cell=rpc, buckets=(w, nb),
                                            bucket_percentiles=True)
    own = [c.run_ensemble(n, 5, buckets=(w, nb), bucket_percentiles=True,
                          bucket_sample_cap=outs["B"]["bucket_sample_cap"])[0] for c in _configs()]
    cells = LS.cell_of(n, 5, rpc, nc)
    for name, o in outs.items():
        if "buckets" not in o:
            continue
        assert o["bucket_totals"].shape[0] == nc
        assert o["bucket_totals"].tobytes() == B.cell_totals_reference(o["buckets"], nc, replica_index_base=5,
                                                                       replicas_per_cell=rpc).tobytes()
        assert o["bucket_percentile_totals"].tobytes() == B.cell_percentile_totals_reference(
            o["buckets"], o["bucket_percentiles"], nc, replica_index_base=5, replicas_per_cell=rpc).tobytes()
        for r in range(n):
            c = int(cells[r])
            for k in ("buckets", "bucket_percentiles"):
                assert o[k][r].tobytes() == own[c][name][k][r].tobytes(), (name, r, k)


def test_run_sweep_results_equal_each_configurations_own_run():
    R = api.RunConfig
    built = []

    def mk(k):
        def f():
            s = _configs()[k]
            built.append(s)
            return s
        return f
    res = api.ParallelRunner().run_sweep([R(f"c{k}", mk(k), 10 + 3 * k) for k in range(4)])
    for k, r in enumerate(res):
        own = _configs()[k]
        own._seed = 10 + 3 * k
        want = own.run()
        assert r.status & ~TIES == 0
        assert r.summary.total_cross_partition_events == want.total_cross_partition_events
        assert r.summary.total_windows == want.total_windows
        for name, s in want.partitions.items():
            g = r.summary.partitions[name]
            assert (g.total_events_processed, g.events_cancelled) == (s.total_events_processed, s.events_cancelled), (k, name)
        got_sink = next(e for e in built[k]._partitions[1].entities if e.name == "B.sink")
        want_sink = next(e for e in own._partitions[1].entities if e.name == "B.sink")
        assert got_sink.latencies_s == want_sink.latencies_s and got_sink.completion_times == want_sink.completion_times
        got_srv = next(e for e in built[k]._partitions[0].entities if e.name == "A.server")
        want_srv = next(e for e in own._partitions[0].entities if e.name == "A.server")
        assert got_srv.stats_accepted == want_srv.stats_accepted


def test_sweep_sized_point():
    """256 cells x 64 replicas of the tandem (configs[4]'s size): completes without status bits other than ties, and
    every partition's cell totals equal the numpy reduction of its replicas"""
    lm, kw, _ = G.load_linked("linked_tandem_const")
    rng = np.random.RandomState(4)
    nc, rpc = 256, 64
    celled = LS.with_link_cells(LS.with_model_cells(lm, rng, nc), rng, nc)
    n = nc * rpc
    outs, delivered, lost = _device(celled, seed=kw["seed"], end_ns=kw["end_ns"], n=n, caps={}, rpc=rpc, queue_ring=4096)
    for q, o in enumerate(outs):
        st = np.bitwise_or.reduce(o["summaries"]["status"])
        assert int(st) & ~TIES == 0, (q, int(st))
        want = D.cell_totals_from_outputs(celled.models[q], o, nc, rpc)
        for c, ((d, h), (wt, wh)) in enumerate(zip(o["cell_totals"], want)):
            wd = engine.totals_to_dict(wt)
            assert np.array_equal(h, wh), c
            for k, v in wd.items():
                if isinstance(v, float) and k.startswith("sum"):
                    assert v == d[k] or abs(v - d[k]) <= 4 * rpc * np.finfo(float).eps * max(abs(v), abs(d[k])), (q, c, k)
                else:
                    assert d[k] == v, (q, c, k)
    assert int(delivered.sum()) > 0 and int(lost.sum()) > 0
    # a sample of replicas against the cell oracle
    sample = [0, 1, 63, 64, 8191, n - 1]
    for g in sample:
        want, wd, wl, _ = _oracle(celled, seed=kw["seed"], end_ns=kw["end_ns"], n=1, caps={}, base=g, rpc=rpc)
        LS.assert_replica_equal(outs, want, g, 0, f"replica {g}")
        assert (int(delivered[g]), int(lost[g])) == (int(wd[0]), int(wl[0]))
