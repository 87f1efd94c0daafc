"""The lane engine's recorder rings in 64-byte chunks, every replica bit for bit against the oracle.

With a sample_cap that is a multiple of 4 the Sink samples are staged in shared memory and written by the warp, four
per group; with a service_cap that is a multiple of 8 the refill round writes the service times as it generates them,
eight per chunk, ahead of their service start.  At the end of every launch the slots written ahead get back what they
held: the service time one ring pass earlier, or 0 on the first pass; and service times consumed from a chunk not
generated whole yet are written from the draw buffer.  The oracle writes each entry when it happens, so any slot the
end of a launch gets wrong differs from it, in paused windows as much as at the end.

- Windows cut so that the service count stops at every residue mod 8 and the Sink-sample count at every residue mod
  4, in the SIMPLE chain, the general fused chains and the profile kernels, with and without the order hash: every
  resumed launch begins inside a service chunk and a sample group.
- A first ring pass that the windows do not finish: the slots written ahead are restored to 0.
- Service times from a trace (stock mode): the restore regenerates them from the trace rather than from Philox.
- max_events right after a refill wrote a chunk ahead, at every position of the chains.
- Capacities that are multiples of the old 32-byte sectors but not of the chunks take the per-entry stores."""
import numpy as np
import pytest

import happysim_b200 as hs
import oracle_lib as O
from happysim_b200 import _abi as A, engine
from test_gpu_lane_kernels import (HASH, HIST, LF_HASH, LF_REC, MATRIX, N, OUT, STOP_MODELS, kernel_flags, run,
                                   run_in_windows)
from test_gpu_lane_parity import assert_same

pytestmark = pytest.mark.gpu

CHUNK_CAPS = {"chunk": dict(record_cap=48, sample_cap=16, service_cap=24),      # rings that wrap many times
              "chunk_min": dict(record_cap=16, sample_cap=4, service_cap=8),    # one group / one chunk per ring
              "sectors": dict(record_cap=48, sample_cap=18, service_cap=20)}    # per-entry stores


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


def many_cuts(end):
    """Thirteen windows at irregular instants: enough pauses for every residue of both counts in a 1 317-replica run,
    the first one within the first pass of an 8-entry service ring (with constant service times, the only pause at which
    a slot written ahead differs from what it held: 0.0)."""
    return [end // 40 + 7] + [end * k // 13 + 7919 * k for k in range(1, 13)]


def paused_counts(model, kw, cuts):
    """The oracle's (service count, Sink-sample count) of every replica at every cut."""
    svc, smp = [], []
    for c in cuts:
        s = O.oracle_run_parallel(model, O.make_params(**dict(kw, window_end_ns=c)))["summaries"]
        svc.append(s["n_service_samples"]); smp.append(s["n_sink_samples"])
    return np.concatenate(svc), np.concatenate(smp)


def windows_against_oracle(eng, model, kw, fl, cuts):
    """Every paused state and the end equal the oracle's (run_in_windows checks the first pause and the end; the pauses
    between are checked here)."""
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    eng.upload(model)
    run(eng, dict(kw, window_end_ns=cuts[0]), fl)
    for i, c in enumerate(cuts):
        if i:
            run(eng, dict(kw, window_end_ns=c, resume=1), fl)
        assert_same(eng.read_outputs(), O.oracle_run_parallel(model, O.make_params(**dict(kw, window_end_ns=c))), OUT)
    run(eng, dict(kw, resume=1), fl)
    assert_same(eng.read_outputs(), want, OUT)


@pytest.mark.parametrize("caps", sorted(CHUNK_CAPS))
@pytest.mark.parametrize("hash_on", [0, 1], ids=["nohash", "hash"])
@pytest.mark.parametrize("name", ["mm1", "lifo_bounded", "constant_ties", "ramp"])
def test_chunked_rings_in_windows(eng, name, hash_on, caps):
    mk, end_s, family, extra, varied = MATRIX[name]
    model = mk()
    kw = dict(seed=91, end_ns=int(end_s * 1e9), n_replicas=N, flags=(HASH if hash_on else 0) | HIST, **extra,
              **CHUNK_CAPS[caps])
    fl = kernel_flags(family, kw)
    assert fl & LF_REC and bool(fl & LF_HASH) == bool(hash_on)
    cuts = many_cuts(kw["end_ns"])
    if varied:
        n_svc, n_smp = paused_counts(model, kw, cuts)
        assert set(n_svc % 8) == set(range(8)) and set(n_smp % 4) == set(range(4))
    windows_against_oracle(eng, model, kw, fl, cuts)


@pytest.mark.parametrize("name", ["mm1", "lifo_bounded"])
def test_first_ring_pass_restored_to_zero(eng, name):
    """service_cap 64, windows of about 1.5 services per replica: the first pass is not finished at most cuts, so the
    slots written ahead lie beyond every service time so far and go back to 0."""
    mk, _, family, extra, _ = MATRIX[name]
    model = mk()
    kw = dict(seed=92, end_ns=6 * 10**9, n_replicas=N, flags=HIST, record_cap=64, sample_cap=64, service_cap=64, **extra)
    fl = kernel_flags(family, kw)
    cuts = [k * 200_000_000 + 31 * k for k in range(1, 20)]
    n_svc, _ = paused_counts(model, kw, cuts[:3])
    assert (n_svc < 64).all() and set(n_svc % 8) == set(range(8))
    windows_against_oracle(eng, model, kw, fl, cuts)


def test_service_times_from_a_trace(eng):
    """Stock mode: the service draws come from the trace rows, and so do the values the restore puts back."""
    model = hs.mm1()
    rng = np.random.default_rng(93)
    n_draws = 1200
    arr = rng.exponential(size=(N, n_draws))
    svc = rng.exponential(size=(N, n_draws))
    kw = dict(seed=93, end_ns=40 * 10**9, n_replicas=N, flags=HIST, **CHUNK_CAPS["chunk"])
    cuts = many_cuts(kw["end_ns"])
    p = lambda **o: O.make_params(**dict(kw, **o))                             # noqa: E731
    want = O.oracle_run_trace(model, p(), arr, svc)
    assert int(want["svc_used"].max()) < n_draws and int(want["arr_used"].max()) < n_draws
    eng.upload(model)
    eng.set_trace(arr, svc)
    try:
        for i, c in enumerate(cuts):
            eng.run(engine.make_params(engine=2, **dict(kw, window_end_ns=c, resume=int(i > 0))))
            assert eng.last_launch()["flags"] == LF_REC                        # the general kernel: a trace is not SIMPLE
            assert_same(eng.read_outputs(), O.oracle_run_trace(model, p(window_end_ns=c), arr, svc), OUT[:-1])
        eng.run(engine.make_params(engine=2, **dict(kw, resume=1)))
        assert_same(eng.read_outputs(), want, OUT[:-1])
    finally:
        eng.set_trace(None, None)


@pytest.mark.parametrize("name", sorted(STOP_MODELS))
def test_event_limit_after_a_chunk_was_written_ahead(eng, name):
    """max_events = m ... m + 7 around the median count: lanes stop at every position of the chains, most of them with
    service draws generated, and written, beyond the last service start."""
    mk, end_s, family = STOP_MODELS[name]
    model = mk()
    kw = dict(seed=94, end_ns=int(end_s * 1e9), n_replicas=N, flags=HIST, **CHUNK_CAPS["chunk"])
    fl = kernel_flags(family, kw)
    probe = O.oracle_run_parallel(model, O.make_params(**dict(kw, n_replicas=256)))
    m = int(np.median(probe["summaries"]["events_processed"]))
    eng.upload(model)
    for k in range(8):
        kw["max_events"] = m + k
        want = O.oracle_run_parallel(model, O.make_params(**kw))
        stopped = (want["summaries"]["status"] & A.HS_ST_EVENT_LIMIT) != 0
        assert stopped.mean() > 0.3 and set(want["summaries"]["n_service_samples"][stopped] % 8) == set(range(8))
        run(eng, kw, fl)
        assert_same(eng.read_outputs(), want, OUT)
        if k == 0:
            run_in_windows(eng, model, kw, fl, want, many_cuts(kw["end_ns"])[::4])
