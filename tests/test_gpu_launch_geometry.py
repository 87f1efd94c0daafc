"""The general engines at the ensemble sizes that select each of their compiled kernels, every replica against the oracle.

The thread engine picks its kernel from the ensemble size and the device's SM count (launch_thread, csrc/hs_engine.cu):
up to 8 x SMs replicas run the spill-free wide kernel with one replica per warp, up to 16 x SMs the 128-register kernel;
beyond that 2 to 32 replicas share a warp, the warp walks the handler kinds in a fixed cycle of passes (phase-locked
dispatch) and the top levels of every heap live in shared memory (21 keys at 2 to 16 replicas per warp, 5 at 32).  The
warp engine's persistent warps stage a second replica once the ensemble outgrows the grid, and a linked run's barrier
spans several blocks once it has more than 128 replicas.  Smaller ensembles run none of this.

Every case asserts through Engine.last_launch() that it reached the geometry it is about -- so a change of the sizing
rule fails here instead of silently moving the coverage -- and compares every replica with the oracle bit for bit:
summaries, entity statistics, event records, Sink and service-time samples in rings small enough to wrap, latency
histograms, sketch states and the device's merged sketch image.  Horizons are short: the point is the geometry."""
import math

import numpy as np
import pytest

import golden_lib as G
import happysim_b200 as hs
import oracle_lib as O
from happysim_b200 import _abi as A, distributed as D, engine
from happysim_b200.linked import LinkedRun
from random_models import random_model, random_model_v2
from test_gpu_lane_parity import assert_same
from test_gpu_warp_parity import chash, tandem, two_sources

pytestmark = pytest.mark.gpu

WF_HEAPTOP, WF_LINKED = 8, 16          # HS_WF_* template flags of csrc/hs_warp_engine.cuh
CAPS = dict(record_cap=29, sample_cap=7, service_cap=5)
FLAGS = A.HS_RUN_ORDER_HASH | A.HS_RUN_HISTOGRAM
# Queue rings are allocated for every replica and server (n x servers x ring x 24 B, kept by the module's engine): at
# these horizons queues stay a few entries deep, and a deeper one sets HS_ST_QUEUE_OVERFLOW, which the oracle never
# does, so it fails the comparison instead of passing unnoticed.  64 servers x 33 797 replicas x 32 entries = 1.7 GB.
RING = 32

# row: (replicas for an SM count, kernel, lane_stride, heap_top).  Each size is the smallest that selects its row plus an
# odd remainder, so the last block and the last warp are partial ("wide" is the largest size of its row instead).
GEOMETRY = {
    "wide": (lambda sm: 8 * sm - 5, "thread_wide", 32, 0),
    "rpw1": (lambda sm: 8 * sm + 3, "thread", 32, 0),
    "rpw2": (lambda sm: 16 * sm + 5, "thread", 16, 21),
    "rpw4": (lambda sm: 32 * sm + 7, "thread", 8, 21),
    "rpw8": (lambda sm: 64 * sm + 3, "thread", 4, 21),
    "rpw16": (lambda sm: 128 * sm + 9, "thread", 2, 21),
    "rpw32": (lambda sm: 256 * sm + 5, "thread", 1, 5),
}


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine(0)
    yield e
    e.close()


def check_thread_geometry(li, row, n, linked=False):
    _, kernel, stride, top = GEOMETRY[row]
    assert (li["engine"], li["kernel"], li["lane_stride"], li["heap_top"]) == (3, kernel, stride, top), li
    assert bool(li["flags"] & WF_HEAPTOP) == (top > 0) and bool(li["flags"] & WF_LINKED) == linked, li
    assert li["grid"] == math.ceil(n * stride / li["block"]), li


def sketch_farm(K=400, n_servers=8):
    """Keyed requests through a round-robin farm into a HyperLogLog and a Count-Min sketch."""
    b = hs.ModelBuilder()
    src = b.source(rate=60.0 * n_servers, key_population=K)
    servers = [b.server(f"S{i}", mean_service_s=0.02) for i in range(n_servers)]
    hll = b.sketch_hll("uniques", precision=8, table=hs.hll_table(8, 1, K))
    cms = b.sketch_cms("freq", width=67, depth=3, table=hs.cms_table(67, 3, 2, K))
    lb = b.load_balancer(backends=servers)
    b.set_target(src, lb)
    for k, sv in enumerate(servers):
        b.set_target(sv, hll if k % 2 else cms)
    return b.build()


def random_case(gen, seed, scale):
    def mk():
        model, end_s, _ = gen(seed)
        return model, end_s * scale
    return mk


def fixed(mk, end_s):
    return lambda: (mk(), end_s)


# name: () -> (model, horizon in seconds)
MODELS = {
    # 64 servers at rho 0.94: from ~40 ms on more than 21 continuations are pending, so pops sift below TOP = 21 and TOP = 5
    "farm64": fixed(lambda: hs.lb_round_robin(64, 600.0), 0.08),
    "mmc32": fixed(lambda: hs.mm1(rate=300.0, concurrency=32), 0.15),
    "tandem": fixed(tandem, 2.0),                   # generic-path events in every pass of the cycle
    "two_sources": fixed(two_sources, 2.5),
    "key_table": fixed(chash, 0.3),
    "sketch_farm": fixed(sketch_farm, 0.08),
    "probe": fixed(lambda: G.load("philox_probe_mm1")[0], 1.5),
    "ramp": fixed(lambda: G.load("philox_ramp_poisson_mm1")[0], 3.0),     # PROFILE
    "random_3": random_case(random_model, 3, 0.1),
    "random_11": random_case(random_model, 11, 0.1),
    "random_v2_5": random_case(random_model_v2, 5, 0.1),
}


def compare(eng, model, got, want):
    assert_same(got, want)
    assert got["histograms"].tobytes() == want["histograms"].tobytes(), "latency histograms differ"
    if want["sketches"] is not None:
        assert got["sketches"].tobytes() == want["sketches"].tobytes(), "sketch states differ"
        merged, host = eng.read_sketches(), D.merge_sketch_states(model, want["sketches"])
        for i, m in merged.items():
            assert m.dtype == host[i].dtype and np.array_equal(m, host[i]), f"merged sketch of entity {i} differs"


@pytest.mark.parametrize("row", sorted(GEOMETRY))
@pytest.mark.parametrize("name", sorted(MODELS))
def test_thread_engine_geometry_matches_the_oracle(eng, sm, name, row):
    model, end_s = MODELS[name]()
    n = GEOMETRY[row][0](sm)
    kw = dict(seed=61, end_ns=int(end_s * 1e9), n_replicas=n, flags=FLAGS, queue_ring=RING, **CAPS)
    eng.upload(model)
    eng.run(engine.make_params(engine=3, **kw))
    check_thread_geometry(eng.last_launch(), row, n)
    got = eng.read_outputs()
    want = O.oracle_run_parallel(model, O.make_params(**kw))
    assert np.median(want["summaries"]["events_processed"]) > CAPS["record_cap"]       # the rings wrap
    if name == "farm64":
        assert np.median(want["summaries"]["heap_left"]) > 21
    compare(eng, model, got, want)


def run_in_windows(eng, model, kw, eng_id):
    """Three windows cut at awkward instants: the paused prefix equals the oracle paused there, the end the uncut run."""
    end = kw["end_ns"]
    cuts = [end // 7 + 3, end // 2 + 1]
    eng.upload(model)
    eng.run(engine.make_params(engine=eng_id, window_end_ns=cuts[0], **kw))
    paused = eng.read_outputs()
    assert_same(paused, O.oracle_run_parallel(model, O.make_params(window_end_ns=cuts[0], **kw)))
    eng.run(engine.make_params(engine=eng_id, window_end_ns=cuts[1], resume=1, **kw))
    eng.run(engine.make_params(engine=eng_id, resume=1, **kw))
    li = eng.last_launch()
    compare(eng, model, eng.read_outputs(), O.oracle_run_parallel(model, O.make_params(**kw)))
    return li, paused


@pytest.mark.parametrize("row", ["rpw8", "rpw32"])
@pytest.mark.parametrize("name", ["farm64", "tandem", "sketch_farm", "random_11"])
def test_heap_top_survives_windows(eng, sm, name, row):
    """The shared-memory heap top is loaded from the replica block on resume and written back at the end of a launch,
    and the shared part of the now tier is parked and unparked across the block's replica columns."""
    model, end_s = MODELS[name]()
    n = GEOMETRY[row][0](sm)
    kw = dict(seed=62, end_ns=int(end_s * 1e9), n_replicas=n, flags=FLAGS, queue_ring=RING, **CAPS)
    check_thread_geometry(run_in_windows(eng, model, kw, 3)[0], row, n)


def test_neighbouring_lanes_run_different_sweep_cells(eng, sm):
    """An M/M/c sweep at 8 replicas per warp with 3 replicas per cell: the lanes of one warp run different (c, rho)."""
    model = hs.mmc_sweep(cs=(1, 2, 5, 32), rhos=(0.5, 0.9))
    n = GEOMETRY["rpw8"][0](sm)
    kw = dict(seed=63, end_ns=int(1.5e9), n_replicas=n, replicas_per_cell=3, flags=FLAGS, **CAPS)
    eng.upload(model)
    eng.run(engine.make_params(engine=3, **kw))
    check_thread_geometry(eng.last_launch(), "rpw8", n)
    got, want = eng.read_outputs(), O.oracle_run_parallel(model, O.make_params(**kw))
    compare(eng, model, got, want)
    ev = want["summaries"]["events_processed"][:8 * (n // 8)].reshape(-1, 8)
    assert (ev.max(axis=1) > 4 * ev.min(axis=1)).mean() > 0.5           # warp-mates with very different loads


def test_event_limit_stops_some_lanes_of_a_warp(eng, sm):
    """max_events stops some replicas of a warp while their warp-mates run on to the end."""
    model, end_s = MODELS["farm64"]()
    n = GEOMETRY["rpw8"][0](sm)
    kw = dict(seed=64, end_ns=int(end_s * 1e9), n_replicas=n, flags=FLAGS, queue_ring=RING, **CAPS)
    probe = O.oracle_run_parallel(model, O.make_params(**dict(kw, n_replicas=256)))
    kw["max_events"] = int(np.median(probe["summaries"]["events_processed"]))
    eng.upload(model)
    eng.run(engine.make_params(engine=3, **kw))
    check_thread_geometry(eng.last_launch(), "rpw8", n)
    got, want = eng.read_outputs(), O.oracle_run_parallel(model, O.make_params(**kw))
    stopped = (want["summaries"]["status"] & A.HS_ST_EVENT_LIMIT) != 0
    per_warp = stopped[:8 * (n // 8)].reshape(-1, 8).sum(axis=1)
    assert ((per_warp > 0) & (per_warp < 8)).sum() > 100
    compare(eng, model, got, want)


# ---- warp engine: more replicas than resident warps ------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["fresh", "windows", "windows_event_limit"])
@pytest.mark.parametrize("name", ["farm64", "tandem"])
def test_warp_engine_stages_second_replicas(eng, sm, name, mode):
    """Once the ensemble outgrows the grid a persistent warp pulls further replicas: it re-zeroes its block, carries the
    mbarrier phase over, and stores one replica and loads the next through the same shared memory; on resume it skips
    the replicas that are done -- with an event limit about half of them stop in the first window.  (64 warps per SM is
    the most any launch can keep resident.)"""
    model, end_s = MODELS[name]()
    n = 96 * sm + 3
    kw = dict(seed=65, end_ns=int(end_s * 1e9), n_replicas=n, flags=FLAGS, queue_ring=RING, **CAPS)
    if mode == "windows_event_limit":
        first = O.oracle_run_parallel(model, O.make_params(**dict(kw, n_replicas=256, window_end_ns=kw["end_ns"] // 7 + 3)))
        kw["max_events"] = int(np.median(first["summaries"]["events_processed"]))
    if mode != "fresh":
        li, paused = run_in_windows(eng, model, kw, 1)
        if mode == "windows_event_limit":
            done = (paused["summaries"]["status"] & A.HS_ST_EVENT_LIMIT) != 0
            assert 0.2 < done.mean() < 0.8, done.mean()
    else:
        eng.upload(model)
        eng.run(engine.make_params(engine=1, **kw))
        li = eng.last_launch()
        compare(eng, model, eng.read_outputs(), O.oracle_run_parallel(model, O.make_params(**kw)))
    assert (li["engine"], li["kernel"]) == (1, "warp") and n > li["grid"] * li["block"] // 32, li


# ---- linked runs: several replicas per warp, a barrier of several blocks -----------------------------------------------

@pytest.mark.parametrize("name", ["linked_lossy_fanout", "linked_aligned_ring_spread"])
def test_linked_ensemble_at_two_replicas_per_warp(sm, name):
    lm, kw, z = G.load_linked(name)
    nP, n = lm.n_partitions, GEOMETRY["rpw2"][0](sm)
    assert n > 128                                              # hs_exchange_kernel: 128 replicas per block
    run = LinkedRun(lm)
    try:
        outs, (delivered, lost, over) = run.run(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=n, caps=[CAPS] * nP,
                                                flags=FLAGS)
        for e in run.engines:
            check_thread_geometry(e.last_launch(), "rpw2", n, linked=True)
    finally:
        run.close()
    ps = [O.make_params(seed=kw["seed"], end_ns=kw["end_ns"], n_replicas=n, rid_base=q, rid_stride=nP + 1, flags=FLAGS,
                        **CAPS) for q in range(nP)]
    want, wd, wl, _ = O.oracle_run_linked_parallel(lm, ps, end_ns=kw["end_ns"], cseed=kw["seed"])
    assert np.array_equal(delivered, wd) and np.array_equal(lost, wl) and not over.any()
    assert wd.min() > 0 and (name != "linked_lossy_fanout" or wl.min() > 0)
    for q in range(nP):
        assert_same(outs[q], want[q])
        assert outs[q]["histograms"].tobytes() == want[q]["histograms"].tobytes(), "latency histograms differ"
        if want[q]["sketches"] is not None:
            assert outs[q]["sketches"].tobytes() == want[q]["sketches"].tobytes(), "sketch states differ"
