"""Ensembles whose replicas straddle the bounds of the device's fixed-size structures (tests/high_water_lib.py): the
queue rings, the general engines' same-timestamp ("now") tier and future-event slots, and the linked partitions'
outboxes and inboxes.  tests/test_high_water.py checks on the CPU that every ensemble has replicas on both sides of
its bound; tests/test_gpu_capacity.py runs them on the device.  Test infrastructure."""
import numpy as np

import happysim_b200 as hs
from happysim_b200 import _abi as A, engine
from happysim_b200.linked import LinkedModel, LinkSpec

RING = 64                    # queue_ring of every ring case: a power of two, so the device uses it as given
N_RING = 64 * 64 + 37        # replicas of a ring case: 64 whole lane blocks and a partial one


def tandem3(rate=10.0, mean_s=0.1):
    """Source.poisson -> three exponential servers in a row -> Sink, every server at rho = 1."""
    b = hs.ModelBuilder()
    src = b.source(rate=rate)
    sink = b.sink()
    s3 = b.server("S3", mean_service_s=mean_s, downstream=sink)
    s2 = b.server("S2", mean_service_s=mean_s, downstream=s3)
    s1 = b.server("S1", mean_service_s=mean_s, downstream=s2)
    b.set_target(src, s1)
    return b.build()


# name: (model, run keywords); each queue's high-water straddles RING in some replicas
RING_CASES = {
    "mm1": (lambda: hs.mm1(rate=10.0, mean_service_s=0.1), dict(seed=3, end_ns=260 * 10**9)),
    "mmc4_lifo": (lambda: hs.mm1(rate=40.0, mean_service_s=0.1, concurrency=4, lifo=True), dict(seed=5, end_ns=70 * 10**9)),
    "tandem3": (tandem3, dict(seed=7, end_ns=200 * 10**9)),
    "mm1_capacity": (lambda: hs.mm1(rate=10.0, mean_service_s=0.1, capacity=RING), dict(seed=9, end_ns=260 * 10**9)),
}


def ring_case(name, n=N_RING):
    mk, kw = RING_CASES[name]
    return mk(), dict(kw, n_replicas=n, queue_ring=RING)


def ring_cut(kw):
    """Where the windowed ring runs pause: mid-run, off any event's nanosecond."""
    return kw["end_ns"] // 2 + 12345


# ---- the now tier ------------------------------------------------------------------------------------------------------

N_NOW_SOURCES = 26
NOW_TIES = (1, 2, 3, 19, 20, 21)     # sources that share a rate, per sweep cell


def now_farm(ties=NOW_TIES, n_servers=5, rate=2.0, mean_s=0.1):
    """N_NOW_SOURCES constant-rate sources into a round-robin farm of exponential servers.  In sweep cell k the first
    ties[k] sources tick at ``rate`` together; the others at rates that never meet it or each other within the run.
    Every shared tick puts one request per tied source into the now tier, and each request's chain (LB, ENQUEUE,
    NOTIFY, LB_RESPONSE, POLL, ...) briefly adds more: the tier's high-water varies by replica around a depth set by
    the cell."""
    b = hs.ModelBuilder()
    srcs = [b.source(f"Src{i}", rate=rate, poisson=False) for i in range(N_NOW_SOURCES)]
    sink = b.sink()
    servers = [b.server(f"S{i}", mean_service_s=mean_s, downstream=sink) for i in range(n_servers)]
    lb = b.load_balancer(backends=servers)
    for s in srcs:
        b.set_target(s, lb)
    m = b.build()
    ne = m.n_entities
    cd = np.tile(m.entities["d0"].astype(np.float64), (len(ties), 1))
    for k, t in enumerate(ties):
        for i in range(t, N_NOW_SOURCES):
            cd[k, srcs[i]] = rate * (1.0 + 0.0137 * np.sqrt(i + 2))
    m.cell_d0 = cd
    m.cell_i0 = np.tile(m.entities["i0"].astype(np.int32), (len(ties), 1))
    assert m.cell_d0.shape == (len(ties), ne)
    return m


def now_replicas(row, sm):
    """Replicas of a now-tier run at a thread-engine launch geometry of test_gpu_launch_geometry.GEOMETRY"""
    from test_gpu_launch_geometry import GEOMETRY
    return GEOMETRY[row][0](sm)


NOW_RING = 1024             # the farm runs a little above capacity: its queues stay far below this ring


def now_kw(n):
    return dict(seed=11, end_ns=30 * 10**9, n_replicas=n, replicas_per_cell=-(-n // len(NOW_TIES)), queue_ring=NOW_RING)


# ---- the future-event slots ---------------------------------------------------------------------------------------------

def cache_load(rate=1000.0, key_population=4000):
    """Keyed Poisson requests into one CachingServer whose TTL is far shorter than a key's return time: nearly every
    request misses and stays in flight for the cache read, the datastore read and the processing (61.1 ms), each a
    pending continuation in a future-event slot."""
    b = hs.ModelBuilder()
    src = b.source(rate=rate, key_population=key_population)
    cs = b.cache_server(key_slots=key_population, cache_ttl_s=0.001, cache_read_latency_s=0.0001,
                        datastore_read_latency_s=0.05, processing_latency_s=0.011)
    b.set_target(src, cs)
    return b.build()


FEL_KW = dict(seed=13, end_ns=4 * 10**9, n_replicas=512)


# ---- linked partitions --------------------------------------------------------------------------------------------------

OUTBOX_CAP, INBOX_CAP = 7, 5


def linked_tandem(outbox_cap=OUTBOX_CAP, inbox_cap=INBOX_CAP, rate=40.0):
    """Partition A: Source.poisson -> server -> (link, 50 ms) -> partition B: server -> Sink.  A window is 50 ms, so A
    sends about rate / 20 events per window; the outbox and the inbox are a little larger than that."""
    a = hs.ModelBuilder()
    src = a.source(rate=rate)
    rem = a.remote(link=0, dest_entity=0)
    sa = a.server("A.server", mean_service_s=0.012, downstream=rem)
    a.set_target(src, sa)
    ma = a.build()
    ma.outbox_cap = outbox_cap
    b = hs.ModelBuilder()
    sb = b.server("B.server", concurrency=2, mean_service_s=0.02)
    b.set_target(sb, b.sink("B.sink"))
    mb = b.build()
    mb.inbox_cap = inbox_cap
    return LinkedModel(models=[ma, mb], names=["A", "B"],
                       links=[[LinkSpec(dest=1, latency_kind=A.HS_SVC_CONSTANT, latency_mean_s=0.05)], []], window_s=0.05)


LINKED_KW = dict(seed=17, end_ns=6 * 10**9, n_replicas=256)


def linked_params(lm, **caps):
    """Run parameters of every partition, with LinkedRun's replica words (partition q: q + g * (P + 1))"""
    nP = lm.n_partitions
    return [engine.make_params(seed=LINKED_KW["seed"], end_ns=LINKED_KW["end_ns"], n_replicas=LINKED_KW["n_replicas"],
                               rid_base=q, rid_stride=nP + 1, **caps) for q in range(nP)]
