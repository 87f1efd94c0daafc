"""The lane engine's twelve kernels against the oracle, every replica bit for bit.

launch_lane (csrc/hs_engine.cu) instantiates hs_lane_kernel<fl> with fl = HASH | REC | PROFILE | SIMPLE (1, 2, 4, 8;
SIMPLE excludes PROFILE, so fl <= 11): the order hash, the recorder rings, a non-constant rate profile, and the
compile-time M/M/1 shape whose chain is one predicated straight line.  Every run here asserts through
Engine.last_launch() which of them it reached, so a change of the selection fails here instead of silently moving the
coverage, and compares summaries, entity statistics, the three recorder rings raw and the latency histograms.

- A kernel matrix: every model family under {hash, no hash} x {summary, two recorder ring shapes}, at 64 k + 37
  replicas (the last block's second warp has 5 live lanes; its idle lanes alias replica n - 1 and must store nothing),
  uncut and cut into windows at awkward instants.  The rings are small enough to wrap, and the cut leaves replicas at
  every residue of the record group (8), the Sink-sample pair (2) and the service-time quad (4).  Sources whose rate
  profile falls to a negligible rate for good run dry in the four profile kernels.
- Lanes of one warp that stop apart: max_events in the middle of the chains, at every position of a chain, and
  exactly at a window cut.
- Full size, as bench.py runs configs[1] (65 536 replicas, two waves of blocks) and as one GPU of eight runs
  configs[4] (32 768 replicas, per-cell and whole-run reductions against a correctly rounded reduction of the
  oracle's outputs)."""
import math

import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import oracle_lib as O
from happysim_b200 import _abi as A, engine
from test_gpu_lane_parity import KEYS, assert_same

pytestmark = pytest.mark.gpu

LF_HASH, LF_REC, LF_PROFILE, LF_SIMPLE = 1, 2, 4, 8      # HS_LF_* of csrc/hs_lane_engine.cuh
N = 64 * 20 + 37                                         # 1 317 replicas: a partial last block and warp
OUT = KEYS + ("histograms",)
HASH, HIST = A.HS_RUN_ORDER_HASH, A.HS_RUN_HISTOGRAM
# recorder rings: group-aligned records (staged, flushed warp-wide), even Sink samples (pairs), service times in quads;
# the smallest such rings; and capacities that take the per-entry stores
CAPS = {"summary": {},
        "rec": dict(record_cap=48, sample_cap=14, service_cap=12),
        "rec_min": dict(record_cap=16, sample_cap=2, service_cap=4),
        "rec_odd": dict(record_cap=60, sample_cap=15, service_cap=13)}


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


def run(eng, kw, fl):
    """One launch; asserts it ran hs_lane_kernel<fl> over ceil(n / 64) blocks of 64 threads."""
    eng.run(engine.make_params(engine=2, **kw))
    li = eng.last_launch()
    n = kw["n_replicas"]
    assert (li["engine"], li["kernel"], li["flags"], li["block"], li["grid"]) == (2, "lane", fl, 64, math.ceil(n / 64)), li


def kernel_flags(family, kw):
    rec = any(kw.get(k, 0) for k in ("record_cap", "sample_cap", "service_cap"))
    return ((LF_HASH if kw["flags"] & HASH else 0) | (LF_REC if rec else 0) |
            {"simple": LF_SIMPLE, "general": 0, "profile": LF_PROFILE}[family])


def run_in_windows(eng, model, kw, fl, want, cuts):
    """Windows cut at ``cuts``: the first paused state equals the oracle paused there, the end ``want`` (the uncut
    oracle run).  Returns the oracle's paused outputs."""
    eng.upload(model)
    run(eng, dict(kw, window_end_ns=cuts[0]), fl)
    paused = O.oracle_run_parallel(model, O.make_params(**dict(kw, window_end_ns=cuts[0])))
    assert_same(eng.read_outputs(), paused, OUT)
    for c in cuts[1:]:
        run(eng, dict(kw, window_end_ns=c, resume=1), fl)
    run(eng, dict(kw, resume=1), fl)
    assert_same(eng.read_outputs(), want, OUT)
    return paused


def awkward_cuts(end):
    return [end // 7 + 3, end // 7 + 4, end // 2 + 12345]


# ---- A. the kernel matrix ---------------------------------------------------------------------------------------------

def source_server(*, sink="sink", profile=None, rate=8.0, stop_after_ns=-1, **server):
    b = hs.ModelBuilder()
    src = b.source(rate=rate, profile=profile, stop_after_ns=stop_after_ns)
    srv = b.server(**server)
    b.set_target(src, srv)
    if sink:
        b.set_target(srv, b.sink() if sink == "sink" else b.counter())
    return b.build()


def fixture(name):
    return lambda: G.load(name)[0]


# name: (model, horizon in s, kernel family, run keywords, random: the replicas differ from each other)
MATRIX = {
    "mm1": (hs.mm1, 40.0, "simple", {}, True),
    # all cells c = 1: per-cell rates in the SIMPLE kernel; neighbouring lanes run different rates
    "sweep_c1": (lambda: hs.mmc_sweep(cs=(1,), rhos=(0.5, 0.8, 0.95)), 20.0, "simple", dict(replicas_per_cell=3), True),
    # lanes of one warp run c = 1 ... 64: continuation heaps in HBM at stride c_max = 64
    "sweep_c1_to_64": (lambda: hs.mmc_sweep(cs=(1, 2, 7, 64), rhos=(0.6, 0.95)), 3.0, "general",
                       dict(replicas_per_cell=3, replica_index_base=5), True),
    "lifo_bounded": (lambda: hs.mm1(rate=9.0, lifo=True, capacity=6), 30.0, "general", {}, True),
    "counter": (lambda: source_server(sink="counter", mean_service_s=0.1), 30.0, "general", {}, True),
    "no_downstream": (lambda: source_server(sink=None, mean_service_s=0.1), 30.0, "general", {}, True),
    "stop_after": (lambda: source_server(stop_after_ns=12 * 10**9, mean_service_s=0.1), 20.0, "general", {}, True),
    # arrivals every 100 ms into 100 ms of constant service: completions tie with ticks (the generic step)
    "constant_ties": (lambda: hs.mm1(rate=10.0, mean_service_s=0.1, poisson=False, exponential=False), 20.0,
                      "general", {}, False),
    "ramp": (lambda: source_server(profile=("linear_ramp", 10.0, 2.0, 14.0), mean_service_s=0.05), 15.0, "profile",
             {}, True),
    "spike": (lambda: source_server(profile=("spike", 4.0, 12.0, 3.0, 4.0), mean_service_s=0.05), 12.0, "profile",
              {}, True),
    "step": (lambda: source_server(profile=("step", (4.0, 9.0), (3.0, 11.0, 6.0)), mean_service_s=0.06), 14.0,
             "profile", {}, True),
    "philox_ramp_poisson_mm1": (fixture("philox_ramp_poisson_mm1"), 30.0, "profile", {}, True),
    "philox_step_metastable_mm1": (fixture("philox_step_metastable_mm1"), 130.0, "profile", {}, True),
    "philox_ramp_down_constant": (fixture("philox_ramp_down_constant"), 20.0, "profile", {}, True),
}


@pytest.mark.parametrize("caps", ["summary", "rec", "rec_min"])
@pytest.mark.parametrize("hash_on", [0, 1], ids=["nohash", "hash"])
@pytest.mark.parametrize("name", sorted(MATRIX))
def test_lane_kernel_matrix(eng, name, hash_on, caps):
    mk, end_s, family, extra, varied = MATRIX[name]
    model = mk()
    kw = dict(seed=71, end_ns=int(end_s * 1e9), n_replicas=N, flags=(HASH if hash_on else 0) | HIST, **extra,
              **CAPS[caps])
    fl = kernel_flags(family, kw)
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    s = want["summaries"]
    assert (s["status"] == 0).all()
    if caps != "summary":
        assert np.median(s["events_processed"]) > 2 * kw["record_cap"]          # the rings wrap
    if name == "sweep_c1_to_64":
        ev = s["events_processed"][:32 * (N // 32)].reshape(-1, 32)
        assert (ev.max(axis=1) > 20 * ev.min(axis=1)).all()                       # warp-mates with very different loads
    eng.upload(model)
    run(eng, kw, fl)
    assert_same(eng.read_outputs(), want, OUT)
    paused = run_in_windows(eng, model, kw, fl, want, awkward_cuts(kw["end_ns"]))["summaries"]
    if varied and caps != "summary":
        # the cut leaves partly filled record groups, Sink-sample pairs and service-time quads to resume from
        assert set(paused["events_processed"] % 8) == set(range(8))
        assert set(paused["n_service_samples"] % 4) == set(range(4))
        if (model.entities["kind"] == A.HS_ENT_SINK).any():
            assert set(paused["n_sink_samples"] % 2) == {0, 1}


@pytest.mark.parametrize("name", ["mm1", "lifo_bounded", "ramp"])
def test_per_entry_ring_stores(eng, name):
    """Ring capacities that are not multiples of the record group, the sample pair or the service quad: every entry
    is stored on its own, in each kernel family."""
    mk, end_s, family, extra, _ = MATRIX[name]
    model = mk()
    kw = dict(seed=72, end_ns=int(end_s * 1e9), n_replicas=N, flags=HIST, **extra, **CAPS["rec_odd"])
    fl = kernel_flags(family, kw)
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    eng.upload(model)
    run(eng, kw, fl)
    assert_same(eng.read_outputs(), want, OUT)
    run_in_windows(eng, model, kw, fl, want, awkward_cuts(kw["end_ns"]))


# Rate profiles that fall to a negligible rate for good.  The engine refuses a profile rate of 0 (hs_model_validate),
# but 1e-300 / s does the same: the 50 widening brackets of the arrival search (out to ~1e22 s) cannot hold the next
# target, the search fails (HS_T_EXHAUSTED) and the Source never ticks again.  The lane kernel turns that into a dead
# source when it takes the tick (HS_NEXT_TICK), a chain whose next tick is exhausted takes the generic step, and a
# Source whose very first search fails never ticks at all.  (A linear ramp from a positive rate down to the floor fails
# the search too, but costs the oracle about 13 CPU-seconds per replica: Simpson's rule refines the ramp's kink in every
# bracket.  A step fails it cheaply.)
RUNS_DRY = {
    "step_down": ("step", (2.0,), (10.0, 1e-300)),              # 10 / s for 2 s, then dry
    # from 0 s the search's first bracket is 3 600 s wide, and Simpson's samples of it all miss the 2-s spike: the
    # integral is ~0, the bracket never holds the target, and the Source never ticks (as in the reference)
    "spike_missed": ("spike", 1e-300, 10.0, 0.5, 2.0),
    "ramp_flat": ("linear_ramp", 2.0, 1e-300, 1e-300),           # no first tick
}


@pytest.mark.parametrize("caps", ["summary", "rec"])
@pytest.mark.parametrize("hash_on", [0, 1], ids=["nohash", "hash"])
@pytest.mark.parametrize("name", sorted(RUNS_DRY))
def test_source_whose_rate_profile_runs_dry(eng, name, hash_on, caps):
    model = source_server(profile=RUNS_DRY[name], mean_service_s=0.05)
    end = 8 * 10**9
    kw = dict(seed=73, end_ns=end, n_replicas=N, flags=(HASH if hash_on else 0) | HIST, **CAPS[caps])
    fl = kernel_flags("profile", kw)
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    s, ticks = want["summaries"], want["entity_stats"][:, 0]["c0"]
    assert (s["status"] == 0).all() and (s["heap_left"] == 0).all()           # the model ran dry before the end
    if name == "step_down":
        assert (s["final_time_ns"] < end // 2).all() and (ticks > 0).all()
    else:
        assert (s["events_processed"] == 0).all() and (ticks == 0).all()
    eng.upload(model)
    run(eng, kw, fl)
    assert_same(eng.read_outputs(), want, OUT)
    run_in_windows(eng, model, kw, fl, want, awkward_cuts(end))


def test_a_rate_profile_that_reaches_zero_is_refused(eng):
    with pytest.raises(engine.EngineError, match="profile rates must stay > 0"):
        eng.upload(source_server(profile=("linear_ramp", 6.0, 12.0, 0.0), mean_service_s=0.05))


# ---- B. lanes of one warp that stop apart -----------------------------------------------------------------------------

STOP_MODELS = {"mm1": (hs.mm1, 40.0, "simple"),                                   # the SIMPLE chain
               "mmc4": (lambda: hs.mm1(rate=32.0, concurrency=4), 10.0, "general")}   # the general fused chains
STOP_MODES = {"summary": (HASH | HIST, {}), "rec": (HIST, CAPS["rec"])}


def stop_kw(name, mode, seed):
    mk, end_s, family = STOP_MODELS[name]
    flags, caps = STOP_MODES[mode]
    kw = dict(seed=seed, end_ns=int(end_s * 1e9), n_replicas=N, flags=flags, **caps)
    return mk(), kw, kernel_flags(family, kw)


@pytest.mark.parametrize("mode", sorted(STOP_MODES))
@pytest.mark.parametrize("name", sorted(STOP_MODELS))
def test_event_limit_stops_lanes_of_a_warp_apart(eng, name, mode):
    """max_events = m, m + 1, ..., m + 7 around the median count: the limit falls at every position of the chains
    (up to 6 events) for many replicas, and stops some lanes of a warp while their warp-mates run on and keep
    flushing records.  At m, also cut into windows."""
    model, kw, fl = stop_kw(name, mode, 81)
    probe = O.oracle_run_parallel(model, O.make_params(**dict(kw, n_replicas=256)))
    m = int(np.median(probe["summaries"]["events_processed"]))
    eng.upload(model)
    for k in range(8):
        kw["max_events"] = m + k
        want = O.oracle_run_parallel(model, O.make_params(**kw))
        run(eng, kw, fl)
        assert_same(eng.read_outputs(), want, OUT)
        if k == 0:
            stopped = (want["summaries"]["status"] & A.HS_ST_EVENT_LIMIT) != 0
            assert (want["summaries"]["events_processed"][stopped] == m).all()
            per_warp = stopped[:32 * (N // 32)].reshape(-1, 32).sum(axis=1)
            assert ((per_warp > 0) & (per_warp < 32)).mean() > 0.8, per_warp
            run_in_windows(eng, model, kw, fl, want, awkward_cuts(kw["end_ns"]))


@pytest.mark.parametrize("mode", sorted(STOP_MODES))
@pytest.mark.parametrize("name", sorted(STOP_MODELS))
def test_event_limit_exactly_at_a_cut(eng, name, mode):
    """A replica that has processed exactly max_events when the window ends, and whose next event lies beyond the
    window end, is flagged and stops there; it does not resume in the next window."""
    model, kw, fl = stop_kw(name, mode, 82)
    cut = kw["end_ns"] // 7 + 3
    free = O.oracle_run_parallel(model, O.make_params(**dict(kw, window_end_ns=cut)))["summaries"]
    kw["max_events"] = int(np.bincount(free["events_processed"]).argmax())        # the most frequent count at the cut
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    paused = run_in_windows(eng, model, kw, fl, want, [cut])["summaries"]
    at = (free["events_processed"] == kw["max_events"]) & ((paused["status"] & A.HS_ST_EVENT_LIMIT) != 0)
    assert at.sum() >= 2 and (paused["events_processed"][at] == kw["max_events"]).all()
    assert (want["summaries"]["events_processed"][at] == kw["max_events"]).all()


# ---- C. full size, every replica --------------------------------------------------------------------------------------

@pytest.mark.parametrize("caps", ["summary", "rec"])
@pytest.mark.parametrize("flags", [0, HASH], ids=["nohash", "hash"])
def test_config1_full_size_as_bench_runs_it(eng, flags, caps):
    """BASELINE configs[1] as bench.py runs it: 65 536 M/M/1 replicas (1 024 blocks, more than one wave), recorder
    rings of 1 024 / 128 / 128 that wrap about four times, 80 sim-s in four 20-s windows."""
    model = hs.mm1()
    end = 80 * 10**9
    kw = dict(seed=1234, end_ns=end, n_replicas=65536, flags=flags,
              **({} if caps == "summary" else dict(record_cap=1024, sample_cap=128, service_cap=128)))
    fl = kernel_flags("simple", kw)
    eng.upload(model)
    for w in range(4):
        run(eng, dict(kw, window_end_ns=(w + 1) * end // 4, resume=int(w > 0)), fl)
        if w == 1:
            got = eng.read_outputs()
            assert_same(got, O.oracle_run_parallel(model, O.make_params(**dict(kw, window_end_ns=end // 2))), OUT)
    got = eng.read_outputs(got)
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    assert (want["summaries"]["status"] == 0).all()
    if caps == "rec":
        assert want["summaries"]["events_processed"].min() > 4 * 1024
    assert_same(got, want, OUT)


U = 2.0 ** -53


def gamma(h):
    """Higham's gamma_h: a sum whose every term passes through at most h roundings is within gamma_h * sum |x|."""
    return h * U / (1 - h * U)


def assert_reduction(d, hist, out, idx, depth, what):
    """Device totals ``d`` (and histogram ``hist``) of the replicas ``idx`` against the oracle's outputs: integers,
    min / max and histograms exactly, the float sums within ``depth`` roundings of math.fsum."""
    s, st = out["summaries"][idx], out["entity_stats"][idx]
    src, srv, snk = st[:, 0], st[:, 1], st[:, 2]
    ints = {"events_processed": s["events_processed"], "sink_events": snk["c0"], "server_completions": srv["c2"],
            "source_ticks": src["c0"], "dropped": srv["c1"], "replicas": np.ones(len(idx), np.int64),
            "replicas_flagged": (s["status"] != 0).astype(np.int64), "sum_final_time_us": s["final_time_ns"] // 1000}
    for k, v in ints.items():
        assert d[k] == int(v.sum(dtype=np.int64)), (what, k)
    assert d["min_latency"] == snk["f2"].min() and d["max_latency"] == snk["f3"].max(), what
    for k, v in (("sum_latency", snk["f0"]), ("sum_latency_sq", snk["f1"]), ("sum_service", srv["f0"])):
        exact = math.fsum(v.tolist())
        assert abs(d[k] - exact) <= gamma(depth) * math.fsum(np.abs(v).tolist()), (what, k, d[k], exact)
    if hist is not None:
        assert np.array_equal(hist, out["histograms"][idx].sum(axis=0, dtype=np.uint64)), what


def test_config4_full_size_one_gpus_share(eng):
    """BASELINE configs[4] as one GPU of eight runs it: 32 768 replicas = 256 (c, rho) cells x 128 seeds (global
    replica ids of rank 5), histograms on, 10 sim-s in two windows.  Every replica against the oracle, then the 256
    per-cell reductions and the whole-run reduction against the oracle's outputs."""
    model = hs.mmc_sweep()
    n, per_cell, base, n_cells = 32768, 128, 5 * 32768, 256
    kw = dict(seed=1234, end_ns=10 * 10**9, n_replicas=n, replica_index_base=base, replicas_per_cell=per_cell,
              flags=HIST, queue_ring=4096)
    eng.upload(model)
    run(eng, dict(kw, window_end_ns=kw["end_ns"] // 2), 0)
    run(eng, dict(kw, resume=1), 0)
    got = eng.read_outputs()
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    assert (want["summaries"]["status"] == 0).all()
    assert_same(got, want, OUT)
    # hs_cell_totals_kernel: 128 threads stride over the replicas, each folds its replicas of the cell in index
    # order, then 5 shuffle levels and 4 warps in series
    cell_of = ((base + np.arange(n)) // per_cell) % n_cells
    for c, (d, h) in enumerate(eng.read_cell_totals(n_cells)):
        idx = np.flatnonzero(cell_of == c)
        assert_reduction(d, h, want, idx, int(np.bincount(idx % 128).max()) + 5 + 3, f"cell {c}")
    # hs_totals_partial_kernel over 256 blocks of 256 threads, 5 shuffle levels, 8 warps in series, then the 256
    # block partials in series
    per_thread = math.ceil(math.ceil(n / 256) / 256)
    assert_reduction(engine.totals_to_dict(eng.read_totals()), None, want, np.arange(n), per_thread + 5 + 7 + 256,
                     "whole run")
