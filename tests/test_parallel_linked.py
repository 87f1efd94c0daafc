"""ParallelSimulation with PartitionLinks through the API mirror (CPU part): the declarations are checked like
parallel/validation.py does, a Server whose downstream lives in another partition becomes a REMOTE row, and the
partitions lower to exactly the models of the reference-generated fixtures."""
import pytest

import golden_lib as G
import happysim_b200 as hs
from happysim_b200 import _abi as A


def tandem(latency=None, **kw):
    sink = hs.Sink("B.sink")
    sb = hs.Server("B.server", concurrency=2, service_time=hs.ExponentialLatency(0.015), downstream=sink)
    sa = hs.Server("A.server", service_time=hs.ExponentialLatency(0.01), downstream=sb)
    src = hs.Source.poisson(rate=40.0, target=sa)
    parts = [hs.SimulationPartition("A", entities=[sa], sources=[src]), hs.SimulationPartition("B", entities=[sb, sink])]
    link = hs.PartitionLink("A", "B", min_latency=0.05, latency=latency if latency is not None else hs.ConstantLatency(0.05), **kw)
    return parts, link, (src, sa, sb, sink)


def test_partitions_lower_to_the_fixture_models():
    parts, link, _ = tandem()
    ps = hs.ParallelSimulation(parts, duration=4.0, links=[link], seed=5)
    lm, kw, z = G.load_linked("linked_tandem_const")
    got = ps._linked
    assert got.window_s == lm.window_s == 0.05 and got.n_streams == 1 and ps._end_ns == kw["end_ns"]
    for q in range(2):
        assert got.models[q].entities.tobytes() == lm.models[q].entities.tobytes()
    assert got.links[0] == lm.links[0] and got.links[1] == []
    assert got.models[0].outbox_cap > 0 and got.models[1].inbox_cap > 0 and got.models[0].inbox_cap == 0
    row = got.models[0].entities[2]
    assert (int(row["kind"]), int(row["i0"]), int(row["i1"])) == (A.HS_ENT_REMOTE, 0, 0)
    hs.engine.validate_model(got.models[0]); hs.engine.validate_model(got.models[1])
    # the exponential, lossy variant: the link's own distribution object is the latency stream
    parts, link, _ = tandem(latency=hs.ExponentialLatency(0.05), packet_loss=0.2)
    ps = hs.ParallelSimulation(parts, duration=4.0, links=[link], seed=7)
    lm, kw, z = G.load_linked("linked_tandem_lossy_exp")
    assert ps._linked.links[0] == lm.links[0]


def test_a_servers_hidden_parts_may_be_listed_like_a_reference_script_must():
    """The reference's router only knows the entities a partition lists (parallel/routing.py:40-61), so a script has
    to list server.queue / .driver / .worker next to the server; they are not entities of the model."""
    parts, link, (src, sa, sb, sink) = tandem()

    class Part:            # stand-ins for the reference's hidden entities
        def __init__(self, name):
            self.name = name
    sa.queue, sa.driver, sa.worker = Part("A.server.queue"), Part("A.server.driver"), Part("A.server.worker")
    parts[0].entities = [sa, sa.queue, sa.driver, sa.worker]
    ps = hs.ParallelSimulation(parts, duration=1.0, links=[link])
    assert ps._linked.models[0].n_entities == 3


def test_declaration_errors_follow_the_reference():
    parts, link, (src, sa, sb, sink) = tandem()
    with pytest.raises(ValueError, match="unknown dest partition"):
        hs.ParallelSimulation(parts, duration=1.0, links=[hs.PartitionLink("A", "C", min_latency=0.1, latency=hs.ConstantLatency(0.1))])
    with pytest.raises(ValueError, match="window_size"):
        hs.ParallelSimulation(parts, duration=1.0, links=[link], window_size=0.2)
    with pytest.raises(ValueError, match="without a PartitionLink"):
        hs.ParallelSimulation(parts, duration=1.0, links=[hs.PartitionLink("B", "A", min_latency=0.05, latency=hs.ConstantLatency(0.05))])
    with pytest.raises(hs.UnsupportedModelError, match="no latency override"):
        hs.ParallelSimulation(parts, duration=1.0, links=[hs.PartitionLink("A", "B", min_latency=0.05)])
    with pytest.raises(hs.UnsupportedModelError, match="end time"):
        hs.ParallelSimulation(parts, links=[link])
    src2 = hs.Source.poisson(rate=5.0, target=sb)            # a source may not feed another partition
    parts[0].sources.append(src2)
    with pytest.raises(ValueError, match="another partition"):
        hs.ParallelSimulation(parts, duration=1.0, links=[link])
    parts[0].sources.pop()
    parts[1].entities.append(sa)
    with pytest.raises(ValueError, match="is in partitions"):
        hs.ParallelSimulation(parts, duration=1.0, links=[link])


@pytest.mark.skipif(not G.HAVE_REF, reason=G.NO_REF)
def test_the_references_own_objects_lower_the_same_way():
    G.import_reference()
    from happysimulator.components.common import Sink
    from happysimulator.components.server.server import Server
    from happysimulator.distributions.constant import ConstantLatency
    from happysimulator.distributions.exponential import ExponentialLatency
    from happysimulator.load.source import Source
    from happysimulator.parallel.link import PartitionLink
    from happysimulator.parallel.partition import SimulationPartition
    sink = Sink("B.sink")
    sb = Server("B.server", concurrency=2, service_time=ExponentialLatency(0.015), downstream=sink)
    sa = Server("A.server", service_time=ExponentialLatency(0.01), downstream=sb)
    src = Source.poisson(rate=40.0, target=sa)
    parts = [SimulationPartition(name="A", entities=[sa, sa.queue, sa.driver, sa.worker], sources=[src]),
             SimulationPartition(name="B", entities=[sb, sb.queue, sb.driver, sb.worker, sink])]
    link = PartitionLink(source_partition="A", dest_partition="B", min_latency=0.05, latency=ConstantLatency(0.05))
    ps = hs.ParallelSimulation(parts, duration=4.0, links=[link], seed=5)
    lm, kw, z = G.load_linked("linked_tandem_const")
    for q in range(2):
        assert ps._linked.models[q].entities.tobytes() == lm.models[q].entities.tobytes()


def test_a_full_queue_ring_is_grown_the_run_repeated_and_the_last_ring_reported(monkeypatch):
    """The reference's queues are unbounded; a device queue ring that filled up (HS_ST_QUEUE_OVERFLOW) is not the
    caller's problem: the whole linked run is repeated with a larger ring (host logic, no device: LinkedRun is stubbed).
    The stub returns whole summary records, as the engine does: a clean run's recorder-ring counts are checked too."""
    import numpy as np
    from happysim_b200 import linked as L, parallel as P
    rings = []

    class StubRun:
        def __init__(self, lm, *, device=0):
            self.lm, self.windows = lm, 0
        def run(self, *, seed, end_ns, n_replicas=1, replica_index_base=0, caps=None, flags=0, queue_ring=0):
            rings.append(queue_ring)
            st = np.zeros(n_replicas, dtype=A.SUMMARY_DTYPE)
            if queue_ring < 2048:
                st["status"][0] = A.HS_ST_QUEUE_OVERFLOW
            self.windows = 80
            z = np.zeros(n_replicas, np.uint64)
            return [{"summaries": st.copy()} for _ in self.lm.models], (z, z.copy(), z.copy())
        def close(self):
            pass

    monkeypatch.setattr(L, "LinkedRun", StubRun)
    parts, link, _ = tandem()
    ps = hs.ParallelSimulation(parts, duration=4.0, links=[link], seed=5)
    outs, delivered, lost, wall, windows = ps._run_linked(3)
    assert rings == [0, 512, 2048] and ps.last_queue_ring == 2048 and windows == 80
    # a caller's own starting size is respected, and a ring that never suffices ends in an error that names the cause
    rings.clear()
    ps.queue_ring = 4096
    ps._run_linked(1)
    assert rings == [4096]
    def always_full(self, *, queue_ring, **kw):
        rings.append(queue_ring)
        st = np.zeros(1, dtype=A.SUMMARY_DTYPE)
        st["status"] = A.HS_ST_QUEUE_OVERFLOW
        return [{"summaries": st.copy()} for _ in self.lm.models], (np.zeros(1, np.uint64),) * 3
    StubRun.run = always_full
    rings.clear()
    # six attempts from 4096 slots, x4 each: the message and last_queue_ring name the ring the last attempt ran with
    with pytest.raises(RuntimeError, match=r"outgrew 4194304 device slots \(ParallelSimulation.queue_ring\)"):
        ps._run_linked(1)
    assert rings == [4096 * 4 ** k for k in range(6)] and ps.last_queue_ring == 4194304
