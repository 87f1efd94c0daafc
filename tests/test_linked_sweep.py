"""Linked ParallelSimulations as the cells of one ensemble, without a GPU: which configurations share a linked
topology, the cell oracle (tests/linked_sweep_oracle.c) against the unmodified oracle's standalone run of every cell and
against the reference (tests/golden/lsweep_cells.npz), the host path of run_ensemble(cells=) and run_sweep on the
oracle, and the ABI's refusal of malformed per-cell link tables."""
import os

import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import linked_fault_models as LF
import linked_sweep_lib as LS
import oracle_lib as O
import random_models as RM
from happysim_b200 import _abi as A, api, engine, linked
from happysim_b200.linked import LinkedModel, LinkSpec
from happysim_b200.lowering import UnsupportedModelError
from happysim_b200.parallel import ParallelSimulation, _linked_difference, _same_linked_topology

CAPS = dict(record_cap=4096, sample_cap=2048, service_cap=2048)


# ---- which configurations are one linked topology -------------------------------------------------------------------------

def tandem(latency=0.05, kind="const", loss=0.0, rate=40.0, conc=2, window=None, duration=4.0, names=("A", "B"), seed=42):
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=conc, service_time=hs.ExponentialLatency(0.015), downstream=sink)
    sa = hs.Server("A.server", service_time=hs.ExponentialLatency(0.01), downstream=sb)
    src = hs.Source.poisson(rate=rate, target=sa)
    parts = [hs.SimulationPartition(names[0], entities=[sa], sources=[src]), hs.SimulationPartition(names[1], entities=[sb, sink])]
    lat = hs.ConstantLatency(latency) if kind == "const" else hs.ExponentialLatency(latency)
    link = hs.PartitionLink(names[0], names[1], min_latency=0.05, latency=lat, packet_loss=loss)
    return ParallelSimulation(parts, duration=duration, links=[link], window_size=window, seed=seed)


def fanout(shared=True, lat_b=0.04, lat_c=0.04, loss_b=0.1, loss_c=0.2, seed=42):
    """A: Source -> LB over two servers; s1 -> B's server, s2 -> C's sink, over two exponential links that share one
    latency object (``shared``) or have one each."""
    s1 = hs.Server("A.s1", service_time=hs.ExponentialLatency(0.004))
    s2 = hs.Server("A.s2", service_time=hs.ExponentialLatency(0.006))
    lb = hs.LoadBalancer("A.lb", backends=[s1, s2])
    src = hs.Source.poisson(rate=120.0, target=lb)
    b_sink, c_sink = hs.Sink("B.sink"), hs.Sink("C.sink")
    sb = hs.Server("B.server", concurrency=3, service_time=hs.ExponentialLatency(0.01), downstream=b_sink)
    s1.downstream, s2.downstream = sb, c_sink
    parts = [hs.SimulationPartition("A", entities=[lb, s1, s2], sources=[src]), hs.SimulationPartition("B", entities=[sb, b_sink]),
             hs.SimulationPartition("C", entities=[c_sink])]
    lat = hs.ExponentialLatency(lat_b)
    links = [hs.PartitionLink("A", "B", min_latency=0.02, latency=lat, packet_loss=loss_b),
             hs.PartitionLink("A", "C", min_latency=0.02, latency=lat if shared else hs.ExponentialLatency(lat_c), packet_loss=loss_c)]
    return ParallelSimulation(parts, duration=3.0, links=links, seed=seed)


def test_same_linked_topology_truth_table():
    base = tandem()
    same = {
        "link latency": tandem(latency=0.08),
        "packet loss 0 vs > 0": tandem(loss=0.2),
        "source rate": tandem(rate=70.0),
        "server concurrency": tandem(conc=3),
        "seed": tandem(seed=9),
    }
    for what, other in same.items():
        assert _same_linked_topology(base, other), what
        assert _same_linked_topology(other, base), what
    differ = {
        "window": (tandem(window=0.025), "window"),
        "latency kind": (tandem(kind="exp"), "latency kind"),
        "end time": (tandem(duration=5.0), "end time"),
        "partition names": (tandem(names=("X", "Y")), "partitions"),
        "another model": (fanout(), "partitions"),
    }
    for what, (other, word) in differ.items():
        assert not _same_linked_topology(base, other), what
        assert word in _linked_difference(base, other), (what, _linked_difference(base, other))
    lb = tandem()
    lb.link_buffer = 512
    assert not _same_linked_topology(base, lb) and "link_buffer" in _linked_difference(base, lb)
    # shared vs separate latency objects: two links drawing from one object differ from two objects, whatever the means
    assert _same_linked_topology(fanout(shared=True), fanout(shared=True, lat_b=0.07, loss_b=0.0))
    assert _same_linked_topology(fanout(shared=False), fanout(shared=False, lat_c=0.09))
    assert not _same_linked_topology(fanout(shared=True), fanout(shared=False))
    unlinked = ParallelSimulation([hs.SimulationPartition("A", entities=[hs.Sink("s")])], duration=1.0)
    assert not _same_linked_topology(base, unlinked) and not _same_linked_topology(unlinked, unlinked)


# ---- the cell oracle against the unmodified oracle ------------------------------------------------------------------------

def _standalone(lm, params, g, *, end_ns, cseed, faults):
    """replica g of the standalone linked run of a LinkedModel without cells, on the unmodified oracle (the fault oracle
    when a partition has FAULT rows)"""
    ps = []
    for p in params:
        q = A.RunParams.from_buffer_copy(p)
        q.n_replicas, q.replica_index_base = 1, g
        ps.append(q)
    if faults:
        import linked_fault_oracle_lib as FO
        return FO.run_linked(lm, ps, end_ns=end_ns, cseed=cseed)
    return O.oracle_run_linked(lm, ps, end_ns=end_ns, cseed=cseed)


def check_cells_against_standalone(lm, *, seed, end_ns, n, n_cells, rpc, base, faults=False):
    celled = LS.celled(lm, seed, n_cells)
    celled.validate()
    ps = LS.partition_params(celled, seed=seed, end_ns=end_ns, n=n, caps=CAPS, replica_index_base=base, replicas_per_cell=rpc)
    outs, delivered, lost, _ = LS.run_cells(celled, ps, end_ns=end_ns, cseed=seed, replicas_per_cell=rpc)
    cells = LS.cell_of(n, base, rpc, n_cells)
    for r in range(n):
        c = int(cells[r])
        want, wd, wl, _ = _standalone(celled.cell(c), ps, base + r, end_ns=end_ns, cseed=seed, faults=faults)
        LS.assert_replica_equal(outs, want, r, 0, f"replica {r} (cell {c})")
        assert (int(delivered[r]), int(lost[r])) == (int(wd[0]), int(wl[0])), (r, c)
    return celled, outs, delivered, lost


@pytest.mark.parametrize("seed", [0, 3, 7, 12, 21, 30])
def test_cell_oracle_equals_each_cells_standalone_run_random_linked(seed):
    lm, end_s, what = RM.random_linked_model(seed)
    check_cells_against_standalone(lm, seed=seed + 100, end_ns=int(end_s * 1e9), n=10, n_cells=4, rpc=2, base=3)


@pytest.mark.parametrize("seed", [1, 5, 9])
def test_cell_oracle_equals_each_cells_standalone_run_with_faults(seed):
    lm, end_s, what, _ = LF.random_linked_fault_model(seed)
    check_cells_against_standalone(lm, seed=seed + 200, end_ns=int(end_s * 1e9), n=9, n_cells=3, rpc=1, base=5, faults=True)


def test_a_lossless_cell_next_to_lossy_ones_takes_no_loss_draws():
    """lossy fan-out with cell 1 at loss 0 on every link: its replicas lose nothing and their latency draws are those of
    a lossless run (no loss draw in between); the lossy cells lose events"""
    lm, kw, _ = G.load_linked("linked_lossy_fanout")
    celled, outs, delivered, lost = check_cells_against_standalone(lm, seed=kw["seed"], end_ns=kw["end_ns"], n=6, n_cells=3,
                                                                   rpc=1, base=0)
    assert (celled.cell_links[0][1, :, 1] == 0).all() and (celled.cell_links[0][2, :, 1] > 0).all()
    assert int(lost[1]) == 0 and int(lost[4]) == 0 and int(lost[2]) > 0 and int(lost[5]) > 0


def test_link_descs_of_a_celled_model_are_the_per_cell_table():
    lm, kw, _ = G.load_linked("linked_lossy_fanout")
    celled = LS.with_link_cells(lm, np.random.RandomState(0), 3)
    arr, dst = celled.link_descs(0)
    assert len(arr) == 3 * 2 and dst == [1, 2]
    for c in range(3):
        for k in range(2):
            d = arr[c * 2 + k]
            assert (d.latency_mean_s, d.packet_loss) == tuple(celled.cell_links[0][c, k])
            assert (d.latency_kind, d.stream) == (lm.links[0][k].latency_kind, lm.links[0][k].stream)
    plain, _ = lm.link_descs(0)
    assert bytes(plain) == bytes(lm.cell(0).link_descs(0)[0]) and len(plain) == 2


# ---- the cell oracle against the reference ------------------------------------------------------------------------------

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lsweep_cells.npz")


def load_sweep_case(z, name):
    pre = f"{name}_"
    names = [str(s) for s in z[pre + "names"]]
    models, links, tabs = [], [], []
    n_cells = int(z[pre + "meta"][2])
    for q in range(len(names)):
        pq = f"{pre}p{q}_"
        m = hs.FlatModel(entities=z[pq + "entities"], names=[str(s) for s in z[pq + "enames"]],
                         backends=z[pq + "backends"], key_table=z[pq + "key_table"])
        m.outbox_cap, m.inbox_cap = (int(v) for v in z[pq + "caps"])
        m.cell_d0 = np.tile(np.asarray(m.entities["d0"], np.float64), (n_cells, 1))
        m.cell_i0 = np.tile(np.asarray(m.entities["i0"], np.int32), (n_cells, 1))
        models.append(m)
        t = z[pq + "cell_links"]
        links.append([LinkSpec(int(a[0]), int(a[1]), float(t[0, k, 0]), float(t[0, k, 1]), int(a[2])) for k, a in enumerate(z[pq + "links"])])
        tabs.append(np.asarray(t, np.float64))
    lm = LinkedModel(models, names, links, window_s=float(z[pre + "window_s"]), n_streams=int(z[pre + "n_streams"]), cell_links=tabs)
    seed, end_ns, _ = (int(v) for v in z[pre + "meta"])
    return lm, seed, end_ns, n_cells


def sweep_caps(z, name, lm, n_cells):
    return [dict(record_cap=max(len(z[f"{name}_c{c}_p{q}_records"]) for c in range(n_cells)) + 1,
                 sample_cap=max(len(z[f"{name}_c{c}_p{q}_sink_samples"]) for c in range(n_cells)) + 1,
                 service_cap=max(len(z[f"{name}_c{c}_p{q}_service_samples"]) for c in range(n_cells)) + 1)
            for q in range(lm.n_partitions)]


class _Fixture(dict):
    """one configuration's arrays under the keys of a linked fixture (golden_lib.check_linked_partition reads those)"""
    @property
    def files(self):
        return list(self)


def check_against_sweep_fixture(z, name, lm, outs, delivered, cell_of_replica):
    for r, c in enumerate(cell_of_replica):
        assert int(delivered[r]) == int(z[f"{name}_c{c}_cross_events"]), (name, r, c)
        for q in range(lm.n_partitions):
            sub = {k.split(f"{name}_c{c}_")[1]: z[k] for k in z.files if k.startswith(f"{name}_c{c}_p{q}_")}
            G.check_linked_partition(_Fixture(sub), q, outs[q], r)


@pytest.mark.parametrize("name", ["tandem", "fanout"])
def test_cell_oracle_equals_the_reference_per_configuration(name):
    """one celled run, replica k = configuration k with the seed and replica words of a single run (rid_stride 0, as
    run_sweep runs a group of equal seeds), against the reference's ParallelSimulation of every configuration"""
    z = np.load(GOLDEN)
    lm, seed, end_ns, nc = load_sweep_case(z, name)
    caps = sweep_caps(z, name, lm, nc)
    ps = LS.partition_params(lm, seed=seed, end_ns=end_ns, n=nc, caps=caps, rid_stride=0)
    outs, delivered, lost, ends = LS.run_cells(lm, ps, end_ns=end_ns, cseed=seed, crid_stride=0)
    assert len(ends) == int(z[f"{name}_c0_windows"])
    check_against_sweep_fixture(z, name, lm, outs, delivered, range(nc))


# ---- the host path on the oracle ------------------------------------------------------------------------------------------

@pytest.fixture
def on_oracle(monkeypatch):
    LS.OracleCellsLinkedRun.runs = []
    monkeypatch.setattr(linked, "LinkedRun", LS.OracleCellsLinkedRun)
    return LS.OracleCellsLinkedRun


def _configs():
    return [tandem(latency=0.05), tandem(latency=0.09, loss=0.1, rate=60.0), tandem(latency=0.07, conc=1),
            tandem(latency=0.12, loss=0.3, rate=30.0, conc=3)]


def test_run_ensemble_cells_equal_each_cells_own_ensemble(on_oracle, monkeypatch):
    """replica g of cell c of run_ensemble(cells=) equals replica g of cells[c].run_ensemble(n), on the oracle; two
    shards concatenated equal one run"""
    cells = _configs()
    n, rpc = 10, 2
    outs, delivered, lost = cells[0].run_ensemble(n, cells=cells, replicas_per_cell=rpc)
    lm = on_oracle.runs[-1].lm
    assert lm.n_cells == 4 and lm.cell_links[0].shape == (4, 1, 2)
    names = list(outs)
    own = []
    for c in cells:
        monkeypatch.setattr(linked, "LinkedRun", O.OracleLinkedRun)      # a run without cells, as before they existed
        own.append(c.run_ensemble(n))
    for r, c in enumerate(LS.cell_of(n, 0, rpc, 4)):
        o, d, l_ = own[int(c)]
        LS.assert_replica_equal([outs[k] for k in names], [o[k] for k in names], r, r, f"replica {r}")
        assert (int(delivered[r]), int(lost[r])) == (int(d[r]), int(l_[r]))
    monkeypatch.setattr(linked, "LinkedRun", LS.OracleCellsLinkedRun)
    a = cells[0].run_ensemble(4, 0, cells=cells, replicas_per_cell=rpc)
    b = cells[0].run_ensemble(6, 4, cells=cells, replicas_per_cell=rpc)
    for k in names:
        for key in LS.KEYS:
            if outs[k].get(key) is not None:
                assert np.concatenate([a[0][k][key], b[0][k][key]]).tobytes() == outs[k][key].tobytes(), (k, key)
    assert np.concatenate([a[1], b[1]]).tobytes() == delivered.tobytes()


def test_run_ensemble_refuses_cells_of_another_topology(on_oracle):
    base = tandem()
    with pytest.raises(UnsupportedModelError, match=r"cells\[1\].*window"):
        base.run_ensemble(2, cells=[base, tandem(window=0.025)])
    with pytest.raises(UnsupportedModelError, match=r"cells\[1\].*latency kind"):
        base.run_ensemble(2, cells=[base, tandem(kind="exp")])
    with pytest.raises(UnsupportedModelError, match="seed"):
        base.run_ensemble(2, cells=[base, tandem(seed=3)])
    unlinked = ParallelSimulation([hs.SimulationPartition("A", entities=[hs.Sink("s")])], duration=1.0)
    with pytest.raises(UnsupportedModelError, match="PartitionLinks"):
        base.run_ensemble(2, cells=[base, unlinked])


def test_run_sweep_runs_a_linked_group_once_and_writes_each_config_back(on_oracle, monkeypatch):
    """seeds in arithmetic progression: one linked run (key seed_0 + k * step, rid_stride 0); each configuration's
    summary, objects and cross-partition count equal its own run()"""
    R = api.RunConfig
    built = []

    def mk(k):
        def f():
            s = _configs()[k]
            built.append(s)
            return s
        return f
    res = api.ParallelRunner().run_sweep([R(f"c{k}", mk(k), 10 + 3 * k) for k in range(4)])
    runs = on_oracle.runs
    assert len(runs) == 1 and runs[0].lm.n_cells == 4
    assert all(c["n_replicas"] == 4 and (c["seed"], c["seed_stride"], c["rid_stride"]) == (10, 3, 0) for c in runs[0].calls)
    monkeypatch.setattr(linked, "LinkedRun", O.OracleLinkedRun)
    for k, r in enumerate(res):
        own = _configs()[k]
        own._seed = 10 + 3 * k
        want = own.run()
        assert r.name == f"c{k}" and r.status == 0
        assert r.summary.total_events_processed == want.total_events_processed
        assert r.summary.total_cross_partition_events == want.total_cross_partition_events
        assert r.summary.total_windows == want.total_windows
        for name in want.partitions:
            assert r.summary.partitions[name].total_events_processed == want.partitions[name].total_events_processed
        # written back onto configuration k's own objects
        got_sink = next(e for e in built[k]._partitions[1].entities if e.name == "B.sink")
        want_sink = next(e for e in own._partitions[1].entities if e.name == "B.sink")
        assert got_sink.events_received == want_sink.events_received and got_sink.latencies_s == want_sink.latencies_s


def test_run_sweep_linked_seeds_out_of_progression_run_one_by_one(on_oracle, monkeypatch):
    R = api.RunConfig
    res = api.ParallelRunner().run_sweep([R(f"c{k}", (lambda k=k: _configs()[k]), s) for k, s in enumerate([10, 12, 17])])
    assert [r.lm.n_cells for r in on_oracle.runs] == [0, 0, 0] and [r.name for r in res] == ["c0", "c1", "c2"]


def test_run_sweep_mixes_simulations_and_parallel_simulations_in_order(on_oracle, monkeypatch):
    """Simulations still go through _run_many, unlinked ParallelSimulations through their own run(), linked ones as
    one group; results keep the configurations' order"""
    calls = []
    monkeypatch.setattr(api, "_run_many", lambda sims, **kw: calls.append(len(sims)) or ["sim"] * len(sims))
    unlinked_runs = []

    def unlinked():
        p = ParallelSimulation([hs.SimulationPartition("U", entities=[hs.Sink("u")])], duration=1.0)
        p.run = lambda: unlinked_runs.append(1) or "unlinked"
        return p

    def sim(rate):
        return lambda: hs.Simulation(sources=[hs.Source.poisson(rate=rate, target=hs.Sink("s"))], entities=[], duration=1.0)
    R = api.RunConfig
    cfgs = [R("t0", lambda: tandem(latency=0.05), 5), R("s0", sim(10.0), 5), R("u", unlinked), R("t1", lambda: tandem(latency=0.08), 5),
            R("s1", sim(20.0), 5)]
    res = api.ParallelRunner().run_sweep(cfgs)
    assert [r.name for r in res] == ["t0", "s0", "u", "t1", "s1"]
    assert res[1].summary == "sim" and res[4].summary == "sim" and calls == [2]
    assert res[2].summary == "unlinked" and unlinked_runs == [1]
    assert [r.lm.n_cells for r in on_oracle.runs] == [2]
    assert res[0].summary.total_cross_partition_events > 0


# ---- the ABI ----------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    return engine.load_library()


def _table(rows):
    arr = (A.LinkDesc * len(rows))()
    for d, (kind, stream, mean, loss) in zip(arr, rows):
        d.latency_kind, d.stream, d.latency_mean_s, d.packet_loss = kind, stream, mean, loss
    return arr


def test_abi_refuses_malformed_cell_tables(lib):
    C_, E_ = A.HS_SVC_CONSTANT, A.HS_SVC_EXPONENTIAL
    good = [(E_, 0, 0.05, 0.1), (C_, 1, 0.02, 0.0), (E_, 0, 0.08, 0.0), (C_, 1, 0.03, 0.3)]      # 2 cells x 2 links
    engine.validate_link_cells(_table(good), 2, 2)
    bad = {
        "latency kind differs": [good[0], good[1], (C_, 0, 0.08, 0.0), good[3]],
        "latency stream differs": [good[0], good[1], good[2], (C_, 0, 0.03, 0.3)],
        "packet_loss in": [good[0], good[1], good[2], (C_, 1, 0.03, 1.0)],
    }
    for msg, rows in bad.items():
        with pytest.raises(engine.EngineError, match=msg) as ei:
            engine.validate_link_cells(_table(rows), 2, 2)
        assert ei.value.code == A.HS_ERR_INVALID
    with pytest.raises(engine.EngineError, match="packet_loss in"):
        engine.validate_link_cells(_table([good[0], good[1], (E_, 0, 0.08, -0.1), good[3]]), 2, 2)
    with pytest.raises(engine.EngineError, match="bad arguments"):
        engine.validate_link_cells(_table(good), 2, 0)


def test_linked_model_validate_checks_the_cell_table():
    lm, kw, _ = G.load_linked("linked_tandem_const")
    celled = LS.celled(lm, 0, 3)
    celled.validate()
    import dataclasses
    bad = dataclasses.replace(celled, cell_links=[t.copy() for t in celled.cell_links])
    bad.cell_links[0][1, 0, 1] = 1.0
    with pytest.raises(ValueError, match="loss"):
        bad.validate()
    short = dataclasses.replace(celled, cell_links=[t[:2] for t in celled.cell_links])
    with pytest.raises(ValueError, match="cells"):
        short.validate()
