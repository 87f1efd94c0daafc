"""Fixtures for partitions joined by PartitionLinks (SURVEY.md 8(f) row 4): the unmodified reference's
ParallelSimulation + WindowedCoordinator (parallel/simulation.py, parallel/coordinator.py) run on linked models, with
the Philox streams injected as in gen_golden.py (ref_harness.run_reference_linked).

    python tests/golden/gen_linked_golden.py        # needs /root/reference; writes tests/golden/linked_*.npz
    python tests/golden/gen_linked_golden.py tandem_heavy     # only the cases whose name contains the argument

Per case: the partition models, the link table, and per partition the reference's summaries, entity statistics, event
records, Sink samples and service times; plus the coordinator's window and cross-partition event counts."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import conftest  # noqa: F401,E402
import happysim_b200 as hs  # noqa: E402
from happysim_b200 import _abi as A  # noqa: E402
from happysim_b200.linked import LinkedModel, LinkSpec  # noqa: E402
import ref_harness as RH  # noqa: E402

CONST, EXPO = A.HS_SVC_CONSTANT, A.HS_SVC_EXPONENTIAL


def tandem_over_a_link(loss=0.0, kind=CONST, latency=0.05):
    """A: Source -> Server -> [link] -> B: Server -> Sink.  The window equals the link latency, so an event sent late
    in a window lands just behind the receiver's overshoot event every now and then ("time travel", skipped)."""
    a = hs.ModelBuilder()
    src = a.source(rate=40.0)
    sa = a.server("A.server", mean_service_s=0.01)
    rem = a.remote("B.server@A", link=0, dest_entity=0)
    a.set_target(src, sa); a.set_target(sa, rem)
    ma = a.build(); ma.outbox_cap = 64
    b = hs.ModelBuilder()
    sb = b.server("B.server", concurrency=2, mean_service_s=0.015)
    snk = b.sink("B.sink")
    b.set_target(sb, snk)
    mb = b.build(); mb.inbox_cap = 64
    return LinkedModel([ma, mb], ["A", "B"], [[LinkSpec(1, kind, latency, loss, 0)], []], window_s=0.05)


def tandem_heavy():
    """A: Source(500/s) -> Server(c=4, exp 1 ms) -> [50 ms link] -> B: Server(c=4, exp 2 ms) -> Sink over 10 s: about
    5 000 Sink samples in B, far more than the recorder rings of the light tandem hold.  The boxes are
    ParallelSimulation.link_buffer wide, as the API lowers this declaration (tests/test_linked_volume.py)."""
    a = hs.ModelBuilder()
    src = a.source(rate=500.0)
    sa = a.server("A.server", concurrency=4, mean_service_s=0.001)
    rem = a.remote("B.server@A", link=0, dest_entity=0)
    a.set_target(src, sa); a.set_target(sa, rem)
    ma = a.build(); ma.outbox_cap = 256
    b = hs.ModelBuilder()
    sb = b.server("B.server", concurrency=4, mean_service_s=0.002)
    snk = b.sink("B.sink")
    b.set_target(sb, snk)
    mb = b.build(); mb.inbox_cap = 256
    return LinkedModel([ma, mb], ["A", "B"], [[LinkSpec(1, CONST, 0.05, 0.0, 0)], []], window_s=0.05)


def aligned_ring(pumps=False):
    """Three partitions in a ring, everything on a 5 ms grid (constant sources, constant service times, constant link
    latencies): cross-partition requests and local ones land on the same nanosecond all the time and are ordered by
    sort indices that come from DIFFERENT partitions' counters (event_heap.py:46-48).
    A: Source(100/s) -> S_A -> B.S_B;  B: Source(50/s) -> S_B -> C.S_C;  C: S_C -> A.counter;  A also counts.
    Without ``pumps`` the three counters grow at about the same pace and a few delivered events tie with a local one
    on time AND index -- the reference then orders the pair by the accident of heapq's array layout.  With ``pumps``
    (a fast local Source -> Counter in B and in C) the counters spread apart: same-nanosecond ties only."""
    a = hs.ModelBuilder()
    sa_src = a.source("A.src", rate=100.0, poisson=False)
    s_a = a.server("A.server", concurrency=2, mean_service_s=0.01, exponential=False)
    cnt = a.counter("A.counter")
    to_b = a.remote("B.server@A", link=0, dest_entity=1)
    a.set_target(sa_src, s_a); a.set_target(s_a, to_b)
    ma = a.build(); ma.outbox_cap, ma.inbox_cap = 64, 64
    b = hs.ModelBuilder()
    sb_src = b.source("B.src", rate=50.0, poisson=False)
    s_b = b.server("B.server", concurrency=4, mean_service_s=0.01, exponential=False)
    to_c = b.remote("C.server@B", link=0, dest_entity=0)
    b.set_target(sb_src, s_b); b.set_target(s_b, to_c)
    if pumps:
        b.set_target(b.source("B.pump", rate=400.0, poisson=False), b.counter("B.pumped"))
    mb = b.build(); mb.outbox_cap, mb.inbox_cap = 64, 64
    c = hs.ModelBuilder()
    s_c = c.server("C.server", concurrency=1, mean_service_s=0.005, exponential=False, capacity=3)
    to_a = c.remote("A.counter@C", link=0, dest_entity=2)
    c.set_target(s_c, to_a)
    if pumps:
        c.set_target(c.source("C.pump", rate=3000.0, poisson=False), c.counter("C.pumped"))
    mc = c.build(); mc.outbox_cap, mc.inbox_cap = 64, 64
    links = [[LinkSpec(1, CONST, 0.02, 0.0, 0)], [LinkSpec(2, CONST, 0.03, 0.0, 1)], [LinkSpec(0, CONST, 0.02, 0.0, 0)]]
    return LinkedModel([ma, mb, mc], ["A", "B", "C"], links, window_s=0.02, n_streams=2)


def lossy_fanout():
    """A sends to B and to C from two servers behind a load balancer (one outbox, interleaved destinations: the
    coordinator's loss draws follow the outbox order); both links lose packets and share ONE exponential latency object
    (PartitionLink.bidirectional style); B answers back into A's sink over a third, lossless link."""
    a = hs.ModelBuilder()
    src = a.source(rate=120.0, key_population=50)
    s1 = a.server("A.s1", mean_service_s=0.004)
    s2 = a.server("A.s2", mean_service_s=0.006)
    lb = a.load_balancer("A.lb", backends=[s1, s2])
    snk = a.sink("A.sink")
    to_b = a.remote("B.server@A", link=0, dest_entity=0)
    to_c = a.remote("C.sketch@A", link=1, dest_entity=0)
    a.set_target(src, lb); a.set_target(s1, to_b); a.set_target(s2, to_c)
    ma = a.build(); ma.outbox_cap, ma.inbox_cap = 128, 128
    b = hs.ModelBuilder()
    s_b = b.server("B.server", concurrency=3, mean_service_s=0.01)
    back = b.remote("A.sink@B", link=0, dest_entity=4)
    b.set_target(s_b, back)
    mb = b.build(); mb.outbox_cap, mb.inbox_cap = 128, 128
    c = hs.ModelBuilder()
    c.sketch_topk("C.heavy", k=6, key_population=50)
    mc = c.build(); mc.inbox_cap = 128
    links = [[LinkSpec(1, EXPO, 0.04, 0.15, 0), LinkSpec(2, EXPO, 0.04, 0.3, 0)], [LinkSpec(0, CONST, 0.025, 0.0, 1)], []]
    return LinkedModel([ma, mb, mc], ["A", "B", "C"], links, window_s=0.025, n_streams=2)


def cases():
    return {
        "tandem_const": (tandem_over_a_link(), dict(seed=5, end_s=4.0)),
        "tandem_lossy_exp": (tandem_over_a_link(loss=0.2, kind=EXPO), dict(seed=7, end_s=4.0)),
        "aligned_ring": (aligned_ring(), dict(seed=1, end_s=1.5)),
        "aligned_ring_spread": (aligned_ring(pumps=True), dict(seed=1, end_s=1.5)),
        "lossy_fanout": (lossy_fanout(), dict(seed=11, end_s=3.0)),
        "tandem_heavy": (tandem_heavy(), dict(seed=5, end_s=10.0)),
    }


def save(path, lm, outs, summ, meta):
    z = dict(names=np.array(lm.names), window_s=np.float64(lm.window_s), n_streams=np.int64(lm.n_streams),
             meta=np.array([meta["seed"], int(meta["end_s"] * 1e9)], dtype=np.int64),
             total_windows=np.int64(summ.total_windows), cross_events=np.int64(summ.total_cross_partition_events),
             total_events=np.int64(summ.total_events_processed))
    for q, (m, o) in enumerate(zip(lm.models, outs)):
        pre = f"p{q}_"
        z[pre + "entities"], z[pre + "backends"], z[pre + "key_table"] = m.entities, m.backends, m.key_table
        z[pre + "enames"] = np.array(m.names)
        z[pre + "caps"] = np.array([m.outbox_cap, m.inbox_cap], dtype=np.int64)
        z[pre + "links"] = np.array([[l.dest, l.latency_kind, l.stream] for l in lm.links[q]], dtype=np.int64).reshape(-1, 3)
        z[pre + "link_params"] = np.array([[l.latency_mean_s, l.packet_loss] for l in lm.links[q]], dtype=np.float64).reshape(-1, 2)
        z[pre + "summaries"], z[pre + "entity_stats"] = o["summaries"], o["entity_stats"]
        z[pre + "records"], z[pre + "sink_samples"], z[pre + "service_samples"] = o["records"], o["sink_samples"], o["service_samples"]
        if "sketches" in o:
            z[pre + "sketch_state"] = o["sketches"]
    np.savez_compressed(path, **z)


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    for name, (lm, kw) in cases().items():
        if only not in name:
            continue
        lm.validate()
        outs, summ = RH.run_reference_linked(lm, seed=kw["seed"], end_ns=int(kw["end_s"] * 1e9))
        save(os.path.join(HERE, f"linked_{name}.npz"), lm, outs, summ, kw)
        skipped = [int(o["summaries"]["heap_left"][0]) for o in outs]
        print(f"linked_{name}: {summ.total_windows} windows, {summ.total_cross_partition_events} cross-partition events, "
              f"{[int(o['summaries']['events_processed'][0]) for o in outs]} events, heap_left {skipped}")


if __name__ == "__main__":
    main()
