"""Sweep cells on the CPU oracle (tests/sweep_models.py).  Every replica of a launch with cells equals, byte for byte,
the plain run of its cell's model at the same global replica index -- so a device run that equals the oracle
(tests/test_gpu_sweep_cells.py) runs every cell as its own single run.  Then what api._same_topology batches into one
launch, and the unmodified reference's runs of a CachingServer TTL sweep and a TDigest compression sweep
(tests/golden/sweep_cells.npz, gen_sweep_cells_golden.py)."""
import dataclasses
import os

import numpy as np
import pytest

import layered_oracle_lib as LO
import happysim_b200 as hs
import oracle_lib as O
from happysim_b200 import _abi as A, api, engine
from sweep_models import (FIXTURE_END_NS, FIXTURE_SEED, cache_farm, cell_case, cell_model, cells_of, fixture_models,
                          has_kind, has_tdigest, tdigest_farm)

KEYS = ("summaries", "entity_stats", "records", "sink_samples", "service_samples", "sketches")
WHOLE = dict(record_cap=16384, sample_cap=4096, service_cap=4096)

# about 40 models: every v2 shape with caches or a TDigest among them, the v1 generator, and v1 models with faults
CASES = [("v1", s) for s in range(14)] + [("v2", s) for s in range(16)] + [("fault", s) for s in range(10)]


def _id(c):
    return f"{c[0]}-{c[1]}"


def run_oracle(model, p):
    return LO.run(model, p) if has_kind(model, A.HS_ENT_FAULT) else O.oracle_run(model, p)


def launch_shape(seed, n_cells):
    """(replicas_per_cell, replica_index_base, n_replicas): every cell runs, and n_replicas is not a multiple of
    n_cells x replicas_per_cell"""
    rpc = (1, 3)[seed % 2]
    return rpc, 5 + seed % 7, n_cells * rpc + 1 + seed % 2


def test_cases_cover_what_cells_can_vary():
    ms = [cell_case(*c)[0] for c in CASES]
    assert sum(has_kind(m, A.HS_ENT_CACHE_SERVER) for m in ms) >= 5
    assert sum(has_tdigest(m) for m in ms) >= 3
    assert sum(has_kind(m, A.HS_ENT_FAULT) for m in ms) == 10
    assert sum(has_kind(m, A.HS_ENT_PROBE) for m in ms) >= 2 and sum(has_kind(m, A.HS_ENT_LB) for m in ms) >= 10
    srv = [m for m in ms if has_kind(m, A.HS_ENT_SERVER)]
    ci = [m.cell_i0[:, m.entities["kind"] == A.HS_ENT_SERVER] for m in srv]
    assert sum((c == 1).all() for c in ci) >= 3                          # every cell at c = 1
    assert sum(((c == 1).any(axis=0) & (c > 1).any(axis=0)).any() for c in ci) >= 5     # a server at c = 1 and c > 1
    for m in ms:
        engine.validate_model(m)
        assert all(api._same_topology(cell_model(m, 0), cell_model(m, c)) for c in range(1, m.n_cells))


def test_ttls_and_compressions_differ_between_cells():
    ms = [cell_case(*c)[0] for c in CASES]
    moved = lambda m, sel: any(len(np.unique(m.cell_d0[:, i])) > 1 for i in np.flatnonzero(sel))     # noqa: E731
    assert sum(moved(m, m.entities["kind"] == A.HS_ENT_CACHE_SERVER) for m in ms) >= 5
    assert sum(moved(m, (m.entities["kind"] == A.HS_ENT_SKETCH) & (m.entities["i0"] == A.HS_SK_TDIGEST)) for m in ms) >= 3


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_every_cell_equals_its_single_run(case):
    m, end_ns, run_seed, what = cell_case(*case)
    rpc, base, n = launch_shape(case[1], m.n_cells)
    assert n % (m.n_cells * rpc)
    kw = dict(seed=run_seed, seed_stride=1, rid_base=3, rid_stride=2, end_ns=end_ns, **WHOLE)
    got = run_oracle(m, O.make_params(n_replicas=n, replica_index_base=base, replicas_per_cell=rpc, **kw))
    assert int(got["summaries"]["events_processed"].max()) < WHOLE["record_cap"], what
    cells = cells_of(n, m.n_cells, base, rpc)
    assert len(set(cells.tolist())) == m.n_cells
    plain = [cell_model(m, c) for c in range(m.n_cells)]
    for r in range(n):
        want = run_oracle(plain[cells[r]], O.make_params(n_replicas=1, replica_index_base=base + r, **kw))
        for k in KEYS:
            if want[k] is not None:
                assert got[k][r].tobytes() == want[k][0].tobytes(), (what, r, int(cells[r]), k)


def test_cells_differ_from_the_lead_configuration():
    """the cells of the TTL and compression cases are not all the lead's run: a kernel that used the lead's value would
    fail the device comparison"""
    differ = 0
    for case in CASES:
        m, end_ns, run_seed, _ = cell_case(*case)
        if not (has_kind(m, A.HS_ENT_CACHE_SERVER) or has_tdigest(m)):
            continue
        kw = dict(seed=run_seed, end_ns=end_ns, n_replicas=m.n_cells, seed_stride=0, rid_stride=0)
        a = run_oracle(m, O.make_params(**kw))
        lead = run_oracle(cell_model(m, 0), O.make_params(**kw))
        differ += sum(a["entity_stats"][r].tobytes() != lead["entity_stats"][r].tobytes() or
                      a["sketches"][r].tobytes() != lead["sketches"][r].tobytes() for r in range(1, m.n_cells))
    assert differ >= 10


# ---- what _same_topology / _group_by_topology batch ----------------------------------------------------------------------

def _sources_servers():
    b = hs.ModelBuilder()
    src = b.source("Src", rate=50.0, key_population=8)
    srv = b.server("Srv", concurrency=2, mean_service_s=0.02)
    snk = b.sink("Sink")
    b.set_target(src, srv)
    b.set_target(srv, snk)
    return b


def _mm1_variant(**kw):
    args = dict(rate=8.0, mean_service_s=0.1, concurrency=1)
    args.update(kw)
    return hs.mm1(**args)


BATCH_TABLE = [
    # name, model a, model b, batched into one launch
    ("ttl_only", lambda: cache_farm(0.05), lambda: cache_farm(30.0), True),
    ("rate_only", lambda: _mm1_variant(rate=8.0), lambda: _mm1_variant(rate=11.0), True),
    ("mean_and_concurrency", lambda: _mm1_variant(), lambda: _mm1_variant(mean_service_s=0.3, concurrency=4), True),
    ("compression_same_buffer", lambda: tdigest_farm(20.0), lambda: tdigest_farm(20.45), True),
    ("compression_moves_buffer", lambda: tdigest_farm(20.0), lambda: tdigest_farm(20.5), False),
    ("capacity", lambda: _mm1_variant(), lambda: _mm1_variant(capacity=5), False),
    ("lifo", lambda: _mm1_variant(), lambda: _mm1_variant(lifo=True), False),
    ("cache_key_slots", lambda: cache_farm(), lambda: _with_i0(cache_farm(), A.HS_ENT_CACHE_SERVER, 40), False),
    ("source_arrival_kind", lambda: _mm1_variant(), lambda: _mm1_variant(poisson=False), False),
    ("lb_strategy", lambda: cache_farm(), lambda: _with_i0(cache_farm(), A.HS_ENT_LB, A.HS_LB_KEY_TABLE), False),
    ("sink_i0", lambda: _sources_servers().build(), lambda: _with_i0(_sources_servers().build(), A.HS_ENT_SINK, 1), False),
]


def _with_i0(m, kind, v):
    E = m.entities.copy()
    E["i0"][E["kind"] == kind] = v
    m.entities = E
    return m


@pytest.mark.parametrize("row", BATCH_TABLE, ids=lambda r: r[0])
def test_same_topology_table(row):
    _, a, b, batched = row
    assert api._same_topology(a(), b()) is batched
    assert api._same_topology(b(), a()) is batched


def test_models_with_cells_are_never_batched():
    m = cell_case("v2", 0)[0]
    assert not api._same_topology(m, cell_model(m, 0)) and not api._same_topology(cell_model(m, 0), m)


class _Sim:                    # the attributes _group_by_topology and run_sweep's grouping read
    def __init__(self, model, seed, end_ns=10**9, device=0):
        self.model, self._seed, self._replica, self._device = model, seed, 0, device
        self._end_time = type("T", (), {"nanoseconds": end_ns})()


def test_group_by_topology_table():
    sims = [_Sim(cache_farm(0.05), 1), _Sim(tdigest_farm(20.0), 1), _Sim(cache_farm(1.0), 2), _Sim(tdigest_farm(20.5), 3),
            _Sim(tdigest_farm(20.2), 4), _Sim(cache_farm(30.0), 3), _Sim(cache_farm(0.3), 4, end_ns=2 * 10**9),
            _Sim(cache_farm(0.3), 5, device=1)]
    assert api._group_by_topology(sims) == [[0, 2, 5], [1, 4], [3], [6], [7]]


def test_run_sweep_launches_once_per_group(monkeypatch):
    """a group whose seeds are an arithmetic progression is one _run_many launch; any other group one run per config"""
    calls = []
    monkeypatch.setattr(api, "_run_many", lambda sims, **kw: calls.append((len(sims), kw)) or [None] * len(sims))
    runs = []

    def build(ttl):
        def mk():
            s = _Sim(cache_farm(ttl), 0)
            s.run = lambda: runs.append(ttl)
            s.last_run_info = {}
            return s
        return mk
    R = api.RunConfig
    api.ParallelRunner().run_sweep([R("a", build(0.05), 10), R("b", build(0.3), 12), R("c", build(1.0), 14)])
    assert calls == [(3, dict(seed=10, seed_stride=2, rid_base=0, rid_stride=0))] and runs == []
    calls.clear()
    api.ParallelRunner().run_sweep([R("a", build(0.05), 10), R("b", build(0.3), 12), R("c", build(1.0), 17)])
    assert calls == [] and runs == [0.05, 0.3, 1.0]


# ---- the unmodified reference (tests/golden/sweep_cells.npz) -------------------------------------------------------------

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sweep_cells.npz")


def check_cells_against_fixture(name, model, out, cell_of_replica):
    """replica r of ``out`` ran cell cell_of_replica[r] with replica word cell_of_replica[r]: equal to the reference's
    run of that configuration"""
    z = np.load(GOLDEN)
    canon = model.canonical_sketches(out["sketches"])
    for r, c in enumerate(cell_of_replica):
        ws = z[f"{name}_c{c}_summary"][0]
        s = out["summaries"][r]
        for f in ("events_processed", "final_time_ns", "order_hash", "heap_left", "n_sink_samples", "n_service_samples"):
            assert int(s[f]) == int(ws[f]), (name, c, f, int(s[f]), int(ws[f]))
        assert out["entity_stats"][r].tobytes() == z[f"{name}_c{c}_stats"][0].tobytes(), (name, c, "entity statistics")
        assert canon[r].tobytes() == z[f"{name}_c{c}_sketches"].tobytes(), (name, c, "sketch / cache states")


@pytest.mark.parametrize("name", ["cache_ttl", "tdigest_compression"])
def test_oracle_cells_match_the_reference(name):
    m, plains = fixture_models()[name]
    n = m.n_cells
    out = O.oracle_run(m, O.make_params(seed=FIXTURE_SEED, end_ns=FIXTURE_END_NS, n_replicas=n, rid_stride=1))
    check_cells_against_fixture(name, m, out, range(n))
    z = np.load(GOLDEN)
    stats = [z[f"{name}_c{c}_stats"][0].tobytes() + z[f"{name}_c{c}_sketches"].tobytes() for c in range(n)]
    assert len(set(stats)) == n                               # every configuration behaves differently


def test_fixture_cache_misses_fall_with_the_ttl():
    z = np.load(GOLDEN)
    m = fixture_models()["cache_ttl"][0]
    caches = m.ids_of(A.HS_ENT_CACHE_SERVER)
    misses = [int(sum(z[f"cache_ttl_c{c}_stats"][0][i]["c3"] for i in caches)) for c in range(m.n_cells)]
    assert all(a > b for a, b in zip(misses, misses[1:])), misses


def test_validation_rejects_cells_the_rows_cannot_hold():
    """a cell's TTL must be positive, and a cell's TDigest compression must keep the row's buffer size int(2c): the
    state layout and the buffer are the model row's, shared by every cell"""
    m = fixture_models()["cache_ttl"][0]
    engine.validate_model(m)
    bad = m.cell_d0.copy()
    bad[2, m.ids_of(A.HS_ENT_CACHE_SERVER)[1]] = 0.0
    with pytest.raises(engine.EngineError, match="ttl must be > 0"):
        engine.validate_model(dataclasses.replace(m, cell_d0=bad))
    m = fixture_models()["tdigest_compression"][0]
    engine.validate_model(m)
    td = [i for i in m.ids_of(A.HS_ENT_SKETCH) if int(m.entities["i0"][i]) == A.HS_SK_TDIGEST][0]
    for c in (20.5, 19.99, 0.0):
        bad = m.cell_d0.copy()
        bad[1, td] = c
        with pytest.raises(engine.EngineError, match="buffer size"):
            engine.validate_model(dataclasses.replace(m, cell_d0=bad))
