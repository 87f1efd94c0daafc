"""Stock-generator ensembles on the device: every replica with its own row of the reference's MT19937 draws.

In stock mode (Engine.set_trace, Simulation(rng="stock"), install()) replica r reads draw k of a stream at
trace[r * n + k].  A wrong row still gives plausible results, so every case compares every replica bit for bit with
the oracle fed the same rows (oracle_lib.oracle_run_trace), on every engine and kernel that reads a trace:

  A  the model families of tests/stock_ensemble_models.py on the thread, warp and (where the model fits it) lane
     engines, at a partial warp, at the thread engine's launch geometries, past the warp engine's resident warps, and
     with the rows reversed;
  B  ParallelRunner.run_sweep over rng="stock" M/M/c configurations: sweep cells with a trace, in one lane launch;
  C  rows cut at the exact boundary of what replicas need: which replicas HS_ST_TRACE_EXHAUSTED flags;
  D  a trace that is too short for the first launch: Simulation's grow-and-retry path, and the same under install();
  E  run_sweep against the reference's own runs (tests/golden/stockens_*.npz).

Rows come from happysim_b200.api.stock_streams (-math.log(1.0 - u), the host libm the reference calls)."""
import time

import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import oracle_lib as O
import stock_ensemble_models as SM
from happysim_b200 import _abi as A, engine
from happysim_b200.api import stock_streams
from test_gpu_lane_parity import KEYS, assert_same
from test_gpu_launch_geometry import GEOMETRY, check_thread_geometry

pytestmark = pytest.mark.gpu

CAPS = dict(record_cap=29, sample_cap=7, service_cap=5)      # rings that wrap
FLAGS = A.HS_RUN_ORDER_HASH
KERNEL = {3: ("thread", "thread_wide"), 1: ("warp",), 2: ("lane",)}
# The lane engine reads its draws ahead into a buffer of HS_DRAW_BUF slots per stream (csrc/hs_lane_engine.cuh:
# HS_DRAW_BUF_SUMMARY = 16, HS_DRAW_BUF_RECORD = 8 with the recorder).  HS_REFILL_ROUND reads the pair of draws
# starting at k = a_gen & ~1 only while a_gen - consumed + 2 <= HS_DRAW_BUF, and flags the replica when k + 1 >= n.  So a
# flag means n - 1 <= k <= consumed + HS_DRAW_BUF - 2 <= need + HS_DRAW_BUF - 2: a replica that needs fewer than
# n - (HS_DRAW_BUF - 1) draws is never flagged.
READ_AHEAD = {True: 8 - 1, False: 16 - 1}                   # recorder on: HS_DRAW_BUF_RECORD - 1, off: SUMMARY - 1


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def family(name):
    """(model, seed s0, end_ns, lane-capable, max draws of one stream any fixture seed needed)"""
    model, kw, z = G.load("stockens_" + name)
    arr, svc = stock_streams(kw["seed"], len(z["summaries"]), int(z["n_draws"]))
    used = O.oracle_run_trace(model, O.make_params(end_ns=kw["end_ns"], n_replicas=len(arr)), arr, svc)
    need = int(max(used["arr_used"].max(), used["svc_used"].max()))
    return model, kw["seed"], kw["end_ns"], SM.FAMILIES[name][3], need


def device_run(eng, model, arr, svc, *, eng_id, **kw):
    eng.upload(model)
    eng.set_trace(arr, svc)
    try:
        eng.run(engine.make_params(engine=eng_id, **kw))
        got = eng.read_outputs()
    finally:
        eng.set_trace(None, None)
    li = eng.last_launch()
    assert li["engine"] == eng_id and li["kernel"] in KERNEL[eng_id], li
    return got, li


def run_and_compare(eng, model, arr, svc, *, eng_id, **kw):
    """The device and the oracle on the same rows; every replica must stay inside its rows and match bit for bit."""
    got, li = device_run(eng, model, arr, svc, eng_id=eng_id, **kw)
    want = O.oracle_run_trace(model, O.make_params(**kw), arr, svc)
    assert want["arr_used"].max() <= arr.shape[1] and want["svc_used"].max() <= svc.shape[1]
    assert not (got["summaries"]["status"] & A.HS_ST_TRACE_EXHAUSTED).any()
    assert_same(got, want)
    return got, want, li


def engines_of(name):
    return [3, 1] + ([2] if SM.FAMILIES[name][3] else [])


# ---- A: every replica, every engine -----------------------------------------------------------------------------------

@pytest.mark.parametrize("name,eng_id", [(f, e) for f in SM.FAMILIES for e in engines_of(f)])
def test_partial_warp_every_replica_reads_its_own_row(eng, name, eng_id):
    model, s0, end_ns, _, need = family(name)
    n = 37
    arr, svc = stock_streams(s0, n, 2 * need + 64)
    got, want, _ = run_and_compare(eng, model, arr, svc, eng_id=eng_id, seed=s0, end_ns=end_ns, n_replicas=n,
                                   flags=FLAGS, **CAPS)
    assert np.median(want["summaries"]["events_processed"]) > CAPS["record_cap"]
    assert len(set(want["summaries"]["order_hash"].tolist())) == n          # 37 different rows, 37 different runs


@pytest.mark.parametrize("eng_id", [3, 1, 2])
def test_reversed_rows_reverse_the_results(eng, eng_id):
    name = "counter" if eng_id == 2 else "two_sources"
    model, s0, end_ns, _, need = family(name)
    n = 37
    arr, svc = stock_streams(s0, n, 2 * need + 64)
    kw = dict(seed=s0, end_ns=end_ns, n_replicas=n, flags=FLAGS, **CAPS)
    fwd, _ = device_run(eng, model, arr, svc, eng_id=eng_id, **kw)
    rev, _ = device_run(eng, model, arr[::-1].copy(), svc[::-1].copy(), eng_id=eng_id, **kw)
    for k in ("summaries", "entity_stats", "records", "sink_samples", "service_samples"):
        if fwd[k] is not None:
            assert rev[k][::-1].tobytes() == fwd[k].tobytes(), k


GEOMETRY_ROWS = ["wide", "rpw1", "rpw2", "rpw8", "rpw32"]


@pytest.mark.parametrize("row", GEOMETRY_ROWS)
@pytest.mark.parametrize("name", ["two_sources", "rr4_c2"])
def test_thread_engine_geometry_with_a_trace(eng, sm, name, row):
    """HEAPTOP kernels (2 to 32 replicas per warp) and the wide kernels, each lane of a warp on its own row."""
    model, s0, end_ns, _, need = family(name)
    n = GEOMETRY[row][0](sm)
    t0 = time.perf_counter()
    arr, svc = stock_streams(s0, n, int(1.3 * need) + 32)
    print(f"stock_streams({n} replicas, {arr.shape[1]} draws per stream): {time.perf_counter() - t0:.2f} s")
    _, _, li = run_and_compare(eng, model, arr, svc, eng_id=3, seed=s0, end_ns=end_ns, n_replicas=n, flags=FLAGS,
                               queue_ring=64, **CAPS)
    check_thread_geometry(li, row, n)


@pytest.mark.parametrize("name", ["two_sources", "tandem3"])
def test_warp_engine_second_replicas_with_a_trace(eng, sm, name):
    """More replicas than resident warps: a persistent warp stages a second replica, which must read its own row."""
    model, s0, end_ns, _, need = family(name)
    n = 96 * sm + 3
    arr, svc = stock_streams(s0, n, int(1.3 * need) + 32)
    _, _, li = run_and_compare(eng, model, arr, svc, eng_id=1, seed=s0, end_ns=end_ns, n_replicas=n, flags=FLAGS,
                               queue_ring=64, **CAPS)
    assert n > li["grid"] * li["block"] // 32, li


# ---- B: sweep cells with a trace ---------------------------------------------------------------------------------------

def mmc(rate, mean, c, end_s, made):
    def build():
        sink = hs.Sink()
        srv = hs.Server("Server", concurrency=c, service_time=hs.ExponentialLatency(mean), downstream=sink)
        sim = hs.Simulation(end_time=hs.Instant.from_seconds(end_s), sources=[hs.Source.poisson(rate=rate, target=srv)],
                            entities=[srv, sink], rng="stock")
        made.append((sim, srv, sink))
        return sim
    return build


def oracle_of(sim, seed, n_draws):
    """The oracle run of one Simulation's own model on its own stock row (seed); rows long enough for the whole run."""
    arr, svc = stock_streams(seed, 1, n_draws)
    c = sim._caps()
    want = O.oracle_run_trace(sim.model, O.make_params(end_ns=sim._end_time.nanoseconds, sample_cap=4 * c["sample_cap"],
                                                       service_cap=4 * c["service_cap"]), arr, svc)
    assert int(want["arr_used"][0]) < n_draws and int(want["svc_used"][0]) < n_draws
    return want


def assert_single_server_run(summary, srv, sink, want):
    s, st = want["summaries"][0], want["entity_stats"][0]
    assert summary.total_events_processed == int(s["events_processed"])
    assert summary.duration_s == float(int(s["final_time_ns"])) / 1e9
    n = int(s["n_sink_samples"])
    assert sink.latencies_s == [float(x) for x in want["sink_samples"][0][:n]["latency_s"]]
    assert srv.stats.total_service_time == float(st[1]["f0"]) and srv.stats.requests_completed == int(st[1]["c2"])
    assert summary.entities[sink.name].events_handled == int(st[2]["c0"])


def test_sweep_cells_with_a_trace_are_one_lane_launch(eng):
    grid = [(6.0, 0.1, 1), (8.0, 0.1, 1), (20.0, 0.1, 3), (9.0, 0.05, 2), (30.0, 0.2, 8), (12.0, 0.15, 2), (40.0, 0.05, 3)]
    made = []
    cfgs = [hs.RunConfig(name=f"c{i}", build_fn=mmc(*g, 30.0, made), seed=900 + 3 * i) for i, g in enumerate(grid)]
    res = hs.ParallelRunner().run_sweep(cfgs)
    assert hs.api._engine(0).last_launch()["kernel"] == "lane"
    for cfg, r, (sim, srv, sink) in zip(cfgs, res, made):
        assert sim.last_run_info["batched_with"] == len(grid) and sim.last_run_info["launches"] == 1 and r.status == 0
        assert_single_server_run(r.summary, srv, sink, oracle_of(sim, cfg.seed, 8192))


# ---- C: exhaustion at the exact boundary -------------------------------------------------------------------------------

def boundary(need):
    """A row length L that one replica needs exactly and another needs L + 1 draws of, nearest the median need."""
    have = set(need.tolist())
    cands = sorted((v for v in have if v + 1 in have), key=lambda v: abs(v - float(np.median(need))))
    assert cands, "no two replicas need consecutive numbers of draws"
    return int(cands[0])


BOUNDARY_CASES = [("two_sources", 3), ("two_sources", 1), ("tandem3", 3), ("tandem3", 1),
                  ("mmc3_lifo_cap", 2), ("counter", 2), ("ramp", 2), ("ramp", 3)]


@pytest.mark.parametrize("streams", ["both", "arrivals", "service"])
@pytest.mark.parametrize("name,eng_id", BOUNDARY_CASES)
def test_trace_exhaustion_flags_exactly_the_replicas_that_run_out(eng, name, eng_id, streams):
    model, s0, end_ns, _, need_max = family(name)
    n = 256
    arr, svc = stock_streams(s0, n, 2 * need_max + 256)
    if streams == "arrivals":
        svc = svc[:, :0]
    elif streams == "service":
        arr = arr[:, :0]
    rec_modes = (True, False) if eng_id == 2 else (True,)
    for rec in rec_modes:
        caps = CAPS if rec else dict(record_cap=0, sample_cap=0, service_cap=0)
        kw = dict(seed=s0, end_ns=end_ns, n_replicas=n, flags=FLAGS, **caps)
        full = O.oracle_run_trace(model, O.make_params(**kw), arr, svc)
        assert full["arr_used"].max() < arr.shape[1] or not arr.shape[1]
        assert full["svc_used"].max() < svc.shape[1] or not svc.shape[1]
        need = np.maximum(full["arr_used"] if arr.shape[1] else 0, full["svc_used"] if svc.shape[1] else 0).astype(np.int64)
        assert need.min() > 0, "the supplied stream is not drawn from"
        L = boundary(need)
        cut_arr, cut_svc = np.ascontiguousarray(arr[:, :L]), np.ascontiguousarray(svc[:, :L])
        got, _ = device_run(eng, model, cut_arr, cut_svc, eng_id=eng_id, **kw)
        flagged = (got["summaries"]["status"] & A.HS_ST_TRACE_EXHAUSTED) != 0
        assert flagged[need > L].all(), f"a replica that needed more than {L} draws was not flagged"
        if eng_id == 2:
            assert not flagged[need < L - READ_AHEAD[rec]].any(), "the lane engine flagged a replica far from the end"
        else:
            assert not flagged[need <= L].any(), f"a replica that needed at most {L} draws was flagged"
        assert (need == L).any() and (need == L + 1).any() and flagged.any() and not flagged.all()
        ok = np.flatnonzero(~flagged)
        sub = lambda out: {k: (None if out[k] is None else np.ascontiguousarray(out[k][ok])) for k in KEYS}  # noqa: E731
        assert_same(sub(got), sub(full))


# ---- D: a first trace that is too short --------------------------------------------------------------------------------

def tandem4(S):
    """Four exponential servers in a row: four service draws per arrival, more than the first trace
    (2 * sample_cap + 64, sample_cap ~ 1.3 x arrivals) holds."""
    sink = S.Sink()
    servers = []
    nxt = sink
    for i in reversed(range(4)):
        nxt = S.Server(f"T{i}", service_time=S.ExponentialLatency(0.01), downstream=nxt)
        servers.insert(0, nxt)
    return [S.Source.poisson(rate=20.0, target=servers[0])], servers, sink


def test_too_short_trace_is_grown_and_the_run_repeated():
    sources, servers, sink = tandem4(hs)
    sim = hs.Simulation(end_time=hs.Instant.from_seconds(60), sources=sources, entities=[*servers, sink], seed=77,
                        rng="stock")
    first = 2 * sim._caps()["sample_cap"] + 64
    summary = sim.run()
    assert sim.last_run_info["launches"] > 1 and sim.last_run_info["status"] == 0
    want = oracle_of(sim, 77, 16384)
    assert int(want["svc_used"][0]) > first                     # the first trace did run out
    s, st = want["summaries"][0], want["entity_stats"][0]
    assert summary.total_events_processed == int(s["events_processed"])
    n = int(s["n_sink_samples"])
    assert sink.latencies_s == [float(x) for x in want["sink_samples"][0][:n]["latency_s"]]
    for i, srv in enumerate(servers):
        assert srv.stats.total_service_time == float(st[1 + i]["f0"]), srv.name


def test_too_short_trace_under_install_matches_the_reference_loop():
    if not G.HAVE_REF:
        pytest.skip(G.NO_REF)
    import random

    ref = G.import_reference()
    from happysimulator.components.server.server import Server
    from happysimulator.distributions.exponential import ExponentialLatency

    class S:                                   # the reference's own classes, for tandem4
        Sink, Source = ref.Sink, ref.Source
    S.Server, S.ExponentialLatency = Server, ExponentialLatency

    def script():
        random.seed(77); np.random.seed(77)
        sources, servers, sink = tandem4(S)
        summary = ref.Simulation(sources=sources, entities=[*servers, sink], end_time=ref.Instant.from_seconds(60)).run()
        return summary, servers, sink, (random.random(), float(np.random.random()))
    want_s, want_srv, want_sink, want_tail = script()
    hs.install()
    try:
        got_s, got_srv, got_sink, got_tail = script()
        st = hs.install_stats()
    finally:
        hs.uninstall()
    assert st["device_runs"] >= 1
    assert got_s.total_events_processed == want_s.total_events_processed and got_s.duration_s == want_s.duration_s
    assert got_sink.latencies_s == want_sink.latencies_s
    for a, b in zip(got_srv, want_srv):
        assert a.stats.total_service_time == b.stats.total_service_time
    assert got_tail == want_tail


# ---- E: against the reference ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(SM.FAMILIES))
def test_run_sweep_reproduces_the_stock_seeded_reference(eng, name):
    _, kw, z = G.load("stockens_" + name)
    s0, n = kw["seed"], len(z["summaries"])
    made = []

    def build():
        made.append(SM.simulation(name))
        return made[-1]
    res = hs.ParallelRunner().run_sweep([hs.RunConfig(name=f"seed{s0 + k}", build_fn=build, seed=s0 + k) for k in range(n)])
    assert hs.api._engine(0).last_launch()["kernel"] == ("lane" if SM.FAMILIES[name][3] else "thread_wide")
    for k, (r, sim) in enumerate(zip(res, made)):
        assert sim.last_run_info["batched_with"] == n and r.status == 0
        ws, st = z["summaries"][k], z["entity_stats"][k]
        assert r.summary.total_events_processed == int(ws["events_processed"])
        assert r.summary.duration_s == float(int(ws["final_time_ns"])) / 1e9
        kinds, names = sim.model.entities["kind"], list(sim.model.names)
        for obj in sim._entities:
            i = names.index(obj.name)
            if kinds[i] == A.HS_ENT_SINK:
                m = int(z["n_samples"][k])
                assert obj.latencies_s == [float(x) for x in z["sink_samples"][k][:m]["latency_s"]]
                assert r.summary.entities[obj.name].events_handled == int(st[i]["c0"])
            elif kinds[i] == A.HS_ENT_SERVER:
                assert obj.stats.total_service_time == float(st[i]["f0"]), obj.name
                assert obj.stats.requests_completed == int(st[i]["c2"]), obj.name
                q = r.summary.entities[obj.name].queue_stats
                assert (q.total_accepted, q.total_dropped) == (int(st[i]["c0"]), int(st[i]["c1"])), obj.name
            elif kinds[i] == A.HS_ENT_COUNTER:
                assert obj.total == int(st[i]["c0"])
