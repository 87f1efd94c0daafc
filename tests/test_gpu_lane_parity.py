"""GPU parity of the lane engine (single-server topology) against the CPU oracle.

Bit-exact: event counts, the (time_ns, sort_index, kind, entity) sequence of every
processed event, the order hash, per-entity statistics (the floating-point sums are
accumulated in the reference's order, so they are compared bitwise too), Sink samples
and service-time samples.  All calls go through the C-ABI (happysim_b200.engine)."""
import numpy as np
import pytest

import happysim_b200 as hs
from happysim_b200 import engine
import oracle_lib as O

pytestmark = pytest.mark.gpu

KEYS = ("summaries", "entity_stats", "records", "sink_samples", "service_samples")


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


def run_both(eng, model, **kw):
    eng.upload(model)
    eng.run(engine.make_params(**kw))
    got = eng.read_outputs()
    want = O.oracle_run(model, O.make_params(**kw))
    return got, want


def assert_same(got, want, keys=KEYS, chunk=2048):
    """Bit-exact equality of the outputs in ``keys`` that ``want`` holds, compared in slices of ``chunk`` replicas (no
    copy of a whole ring array; the arrays need C-contiguous rows, as read_outputs and the oracle allocate them).  A mismatch names the first differing replica r, with its warp and lane in the lane
    kernel (r // 32, r % 32), and its first differing slot."""
    for k in keys:
        if want[k] is None:
            continue
        g, w = got[k], want[k]
        assert g is not None and g.shape == w.shape and g.dtype == w.dtype, f"{k}: got {g if g is None else g.shape}, want {w.shape}"
        n, bad, first = w.shape[0], 0, None
        for r0 in range(0, n, chunk):
            m = min(chunk, n - r0)
            gb, wb = g[r0:r0 + m].view(np.uint8).reshape(m, -1), w[r0:r0 + m].view(np.uint8).reshape(m, -1)
            rows = np.flatnonzero((gb != wb).any(axis=1))
            bad += rows.size
            if first is None and rows.size:
                first = r0 + int(rows[0])
                byte = int(np.flatnonzero(gb[rows[0]] != wb[rows[0]])[0])
        if first is None:
            continue
        r = first
        where = f"replica {r} (warp {r // 32}, lane {r % 32})"
        if g.ndim == 2:
            c = byte // g.dtype.itemsize
            detail = f"{where} slot {c}: got {g[r][max(0, c - 2):c + 3]} want {w[r][max(0, c - 2):c + 3]}"
        else:
            detail = f"{where}: got {g[r]} want {w[r]}"
        raise AssertionError(f"{k}: {bad} replicas differ; first {detail}")


CASES = {
    "mm1_config1": (dict(), 60),
    "mm1_heavy": (dict(rate=9.5), 200),
    "md1_constant": (dict(poisson=False, exponential=False, rate=10, mean_service_s=0.05), 20),
    "dm1": (dict(poisson=False, rate=7.0), 60),
    "mm1_capacity5": (dict(rate=50, mean_service_s=0.1, capacity=5), 20),
    "mm1_capacity0": (dict(rate=5, mean_service_s=0.1, capacity=0), 20),
    "mm1_lifo": (dict(rate=9, mean_service_s=0.1, lifo=True), 60),
    "overload": (dict(rate=20, mean_service_s=0.1), 10),
    "mmc4": (dict(rate=32, concurrency=4), 30),
    "mmc32_lifo_bounded": (dict(rate=300, concurrency=32, lifo=True, capacity=6), 8),
    "mmc3_constant_service": (dict(rate=25, concurrency=3, exponential=False, mean_service_s=0.1), 20),
    "mmc64": (dict(rate=500, concurrency=64), 4),
    # inter-arrivals of a few ns: many SourceEvents tie with their own chain (generic path)
    "zero_gap_poisson": (dict(rate=3e8, mean_service_s=2e-9), 2e-5),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_lane_matches_oracle(eng, name):
    kw, end_s = CASES[name]
    model = hs.mm1(**kw)
    got, want = run_both(eng, model, seed=7, end_ns=int(end_s * 1e9), n_replicas=96, record_cap=6000,
                         sample_cap=800, service_cap=800)
    assert int(want["summaries"]["events_processed"].min()) > 50
    assert_same(got, want)


def test_seed_stride_mirrors_parallel_runner(eng):
    model = hs.mm1()
    got, want = run_both(eng, model, seed=42, seed_stride=1, rid_stride=0, end_ns=30 * 10**9, n_replicas=40,
                         record_cap=2500)
    assert_same(got, want)
    # replica i of base seed 42 == replica 0 of base seed 42 + i
    g2, _ = run_both(eng, model, seed=45, seed_stride=1, rid_stride=0, end_ns=30 * 10**9, n_replicas=1, record_cap=2500)
    assert g2["records"][0].tobytes() == got["records"][3].tobytes()


def test_no_hash_mode_same_counts(eng):
    model = hs.mm1()
    kw = dict(seed=3, end_ns=120 * 10**9, n_replicas=256)
    eng.upload(model)
    eng.run(engine.make_params(**kw))
    a = eng.read_outputs()
    eng.run(engine.make_params(flags=0, **kw))
    b = eng.read_outputs()
    assert np.array_equal(a["summaries"]["events_processed"], b["summaries"]["events_processed"])
    assert np.array_equal(a["summaries"]["final_time_ns"], b["summaries"]["final_time_ns"])
    assert (b["summaries"]["order_hash"] == 0).all()
    assert a["entity_stats"].tobytes() == b["entity_stats"].tobytes()
    want = O.oracle_run(model, O.make_params(**kw))
    assert a["summaries"].tobytes() == want["summaries"].tobytes()


def test_windowed_run_equals_uncut_run(eng):
    """Simulation._run_window semantics: cutting a run into windows must not change the
    processed-event sequence (order hash, counts, statistics)."""
    model = hs.mm1(rate=9.0)
    end = 100 * 10**9
    kw = dict(seed=11, n_replicas=128, record_cap=3000, sample_cap=500)
    want = O.oracle_run(model, O.make_params(end_ns=end, **kw))
    eng.upload(model)
    cuts = [13 * 10**9, 13 * 10**9 + 1, 50 * 10**9, 99_999_999_999]
    eng.run(engine.make_params(end_ns=end, window_end_ns=cuts[0], **kw))
    paused = eng.read_outputs()
    pw = O.oracle_run(model, O.make_params(end_ns=end, window_end_ns=cuts[0], **kw))
    assert paused["summaries"].tobytes() == pw["summaries"].tobytes()
    assert paused["entity_stats"].tobytes() == pw["entity_stats"].tobytes()
    for c in cuts[1:]:
        eng.run(engine.make_params(end_ns=end, window_end_ns=c, resume=1, **kw))
    eng.run(engine.make_params(end_ns=end, window_end_ns=-1, resume=1, **kw))
    got = eng.read_outputs()
    assert_same(got, want)


def test_queue_overflow_is_flagged_not_silent(eng):
    model = hs.mm1(rate=200.0, mean_service_s=0.1)      # rho = 20: queue grows without bound
    eng.upload(model)
    eng.run(engine.make_params(seed=1, end_ns=10 * 10**9, n_replicas=32, queue_ring=64))
    got = eng.read_outputs()
    assert (got["summaries"]["status"] & hs._abi.HS_ST_QUEUE_OVERFLOW).all()


def test_totals_match_per_replica_sums(eng):
    model = hs.mm1()
    eng.upload(model)
    eng.run(engine.make_params(seed=5, end_ns=60 * 10**9, n_replicas=1000))
    got = eng.read_outputs()
    t = engine.totals_to_dict(eng.read_totals())
    assert t["events_processed"] == int(got["summaries"]["events_processed"].sum())
    assert t["replicas"] == 1000 and t["replicas_flagged"] == 0
    sink = got["entity_stats"][:, 2]
    assert t["sink_events"] == int(sink["c0"].sum())
    assert t["min_latency"] == float(sink["f2"].min()) and t["max_latency"] == float(sink["f3"].max())
    assert abs(t["sum_latency"] - float(sink["f0"].sum())) <= 1e-9 * abs(t["sum_latency"])
    assert t["server_completions"] == int(got["entity_stats"][:, 1]["c2"].sum())


@pytest.mark.parametrize("engine_id", [1, 2])
def test_event_limit_stops_a_model_whose_clock_cannot_advance(eng, engine_id):
    """A constant source faster than one event per ns computes every next tick at the same
    nanosecond (int((t/1e9 + 5e-10) * 1e9) == t): the reference would spin forever.  max_events is
    the safety valve; until it trips, every SourceEvent ties with its own chain, so this also
    drives the generic (tie) path hard -- on both engines, against the oracle."""
    model = hs.mm1(poisson=False, rate=2e9, mean_service_s=1e-7, exponential=False, capacity=5)   # bounded queue
    kw = dict(seed=1, end_ns=10**9, n_replicas=40, record_cap=6000, max_events=5003, engine=engine_id)
    got, want = run_both(eng, model, **kw)
    assert (want["summaries"]["events_processed"] == 5003).all()
    assert (want["summaries"]["status"] & hs._abi.HS_ST_EVENT_LIMIT).all()
    assert_same(got, want)


# ---------------------------------------------------------------------------------------------------
# The configuration bench.py times: hash OFF (flags=0), small recorder rings that wrap many times,
# one continuing run cut into resumed windows.  hs_lane_kernel<10> (REC|SIMPLE) and <2> (REC), and
# with the hash on <11>/<3>; rings are compared raw (slot = item number mod cap on both sides).

BENCH_CAPS = dict(record_cap=1024, sample_cap=128, service_cap=128)


@pytest.mark.parametrize("flags", [0, hs._abi.HS_RUN_ORDER_HASH])
@pytest.mark.parametrize("name,model_kw,end_s,n_rep", [
    ("mm1_simple", dict(), 400.0, 160),                      # configs[1] shape -> HS_LF_SIMPLE kernels
    ("mm1_heavy_simple", dict(rate=9.7), 300.0, 96),         # long queues: ring push/pop + prefetch path
    ("mm1_lifo", dict(rate=9.0, lifo=True), 200.0, 64),      # not SIMPLE -> the general fused chains
    ("mmc4", dict(rate=32.0, concurrency=4), 60.0, 64),
])
def test_bench_configuration_windows_and_wrapping_rings(eng, name, model_kw, end_s, n_rep, flags):
    model = hs.mm1(**model_kw)
    end = int(end_s * 1e9)
    kw = dict(seed=1234, n_replicas=n_rep, flags=flags, **BENCH_CAPS)
    want = O.oracle_run(model, O.make_params(end_ns=end, **kw))
    assert int(want["summaries"]["events_processed"].min()) > 4 * 1024      # every ring wrapped
    eng.upload(model)
    cuts = [end // 7, end // 7 + 1, end // 3, end // 2 + 12345, (4 * end) // 5]
    eng.run(engine.make_params(end_ns=end, window_end_ns=cuts[0], **kw))
    for c in cuts[1:]:
        eng.run(engine.make_params(end_ns=end, window_end_ns=c, resume=1, **kw))
        # a paused state is itself comparable: the oracle paused at the same cut
    mid = eng.read_outputs()
    pw = O.oracle_run(model, O.make_params(end_ns=end, window_end_ns=cuts[-1], **kw))
    assert_same(mid, pw)
    eng.run(engine.make_params(end_ns=end, window_end_ns=-1, resume=1, **kw))
    got = eng.read_outputs()
    assert_same(got, want)
    if flags == 0:
        assert (got["summaries"]["order_hash"] == 0).all()


@pytest.mark.parametrize("caps", [dict(record_cap=1000, sample_cap=125, service_cap=126),    # not sector multiples
                                  dict(record_cap=24, sample_cap=2, service_cap=4),          # smallest staged rings
                                  dict(record_cap=0, sample_cap=64, service_cap=0),
                                  dict(record_cap=0, sample_cap=0, service_cap=64)])
def test_recorder_ring_shapes(eng, caps):
    """Ring capacities that are not multiples of the 32-byte store sector, minimal rings, and single streams."""
    model = hs.mm1()
    end = 120 * 10**9
    kw = dict(seed=99, n_replicas=70, flags=0, **caps)
    want = O.oracle_run(model, O.make_params(end_ns=end, **kw))
    eng.upload(model)
    eng.run(engine.make_params(end_ns=end, window_end_ns=37 * 10**9 + 5, **kw))
    eng.run(engine.make_params(end_ns=end, window_end_ns=-1, resume=1, **kw))
    assert_same(eng.read_outputs(), want)
