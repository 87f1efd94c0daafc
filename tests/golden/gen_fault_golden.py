"""Record the fixtures of node faults (tests/golden/fault_*.npz) from the UNMODIFIED reference.

Each case is a model of happysim_b200.ModelBuilder rows, built as reference objects by ref_harness (Philox plug-ins),
plus a reference ``happysimulator.faults.FaultSchedule`` of CrashNode / PauseNode faults handed to the reference's own
``Simulation(fault_schedule=)``.  The pop tap records the fault events itself (ref_harness's classifier knows no
CallbackEntity): kind HS_EV_FAULT, entity = the FAULT row the lowering gives the event.  A cancelled fault event is
popped without being processed, so it is counted (FAULT row c1) and not recorded.  The fixture's model is the
case's rows plus the FAULT rows lowering.fault_events gives the schedule, so the engines replay it through the C-ABI.

    python tests/golden/gen_fault_golden.py
"""
import dataclasses
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import __graft_entry__  # noqa: E402,F401  (puts the repository root on sys.path)
import happysim_b200 as hs  # noqa: E402
from happysim_b200 import _abi as A, lowering  # noqa: E402

import gen_golden as GG  # noqa: E402
import ref_harness as RH  # noqa: E402


def mm1():
    return hs.mm1(rate=8.0, mean_service_s=0.1)


def lb_rr8():
    return hs.lb_round_robin(n_servers=8, rate=64.0, mean_service_s=0.1)


def tandem_probe():
    """Source -> A -> B -> C -> Sink with a depth probe on the middle stage"""
    b = hs.ModelBuilder()
    src = b.source(rate=6.0)
    s1 = b.server("A", mean_service_s=0.08)
    s2 = b.server("B", concurrency=2, mean_service_s=0.2)
    s3 = b.server("C", mean_service_s=0.05)
    snk = b.sink()
    b.set_target(src, s1); b.set_target(s1, s2); b.set_target(s2, s3); b.set_target(s3, snk)
    b.probe("Probe_B_depth", target=s2, metric="depth", interval_s=0.25)
    return GG.reorder_sources_first(b.build())


def cases():
    """name -> (model, schedule builder(ref objects by name, faults module) -> FaultSchedule, run kwargs)"""
    c = {}

    def crash_server(by, F):
        s = F.FaultSchedule()
        s.add(F.CrashNode("Server", at=3.0, restart_at=6.5))
        return s
    c["mm1_crash_restart"] = (mm1(), crash_server, dict(seed=42, rid=0, end_s=12))

    def pause_sink(by, F):
        s = F.FaultSchedule()
        s.add(F.PauseNode("Sink", start=2.0, end=5.0))
        return s
    c["mm1_pause_sink"] = (mm1(), pause_sink, dict(seed=7, rid=1, end_s=10))

    def crash_source(by, F):
        s = F.FaultSchedule()
        s.add(F.CrashNode("Source", at=2.5, restart_at=4.0))     # silent from 2.5 s on, restart or not
        return s
    c["mm1_crash_source"] = (mm1(), crash_source, dict(seed=3, rid=2, end_s=8))

    def crash_backends(by, F):
        s = F.FaultSchedule()
        s.add(F.CrashNode("S2", at=1.0, restart_at=3.0))
        s.add(F.CrashNode("S5", at=1.5))                          # for good: its LB entries stay in flight
        return s
    c["lb_rr8_crash_backends"] = (lb_rr8(), crash_backends, dict(seed=11, rid=0, end_s=5))

    def crash_lb(by, F):
        s = F.FaultSchedule()
        s.add(F.CrashNode("LB", at=1.0, restart_at=2.0))
        return s
    c["lb_rr8_crash_lb"] = (lb_rr8(), crash_lb, dict(seed=13, rid=3, end_s=4))

    def mixed(by, F):
        """overlapping faults on one entity, a cancelled handle, a fault at t = 0 and one after end_time"""
        s = F.FaultSchedule()
        s.add(F.CrashNode("Server", at=0.0, restart_at=1.0))
        s.add(F.PauseNode("Server", start=2.0, end=4.0))
        s.add(F.CrashNode("Server", at=3.0, restart_at=3.5))     # clears the flag inside the pause
        s.add(F.CrashNode("Sink", at=5.0, restart_at=20.0))       # its restart lies beyond end_time: heap_left
        s.add(F.CrashNode("Sink", at=6.0, restart_at=6.5))        # cancelled below: both events popped, not processed
        return s
    c["mm1_mixed"] = (mm1(), mixed, dict(seed=5, rid=0, end_s=9, cancel=[4]))

    def crash_cache(by, F):
        s = F.FaultSchedule()
        s.add(F.CrashNode("Server_2", at=1.0, restart_at=3.0))
        return s
    c["cache_chash5_crash"] = (GG.cache_farm(5, 40, 200.0, 0.8, vnodes=30), crash_cache,
                               dict(seed=41, rid=2, end_s=5, chash_vnodes=30))

    def crash_middle(by, F):
        s = F.FaultSchedule()
        s.add(F.CrashNode("B", at=2.0, restart_at=4.0))
        s.add(F.PauseNode("Probe_B_depth", start=5.0, end=6.0))   # the probe's ticks are dropped, and it stays silent
        return s
    c["tandem_probe_crash_middle"] = (tandem_probe(), crash_middle, dict(seed=17, rid=1, end_s=8))

    def tie(by, F):
        """the source's in-run tick at 2 s takes sort index 1 from the run's counter; the crash at 2.0 s has bootstrap
        index 1 too: heapq orders the pair by its array layout (the generator asserts that the tie occurred)"""
        s = F.FaultSchedule()
        s.add(F.CrashNode("Server", at=2.0, restart_at=3.5))
        return s
    c["tie_constant"] = (hs.mm1(rate=1.0, mean_service_s=0.25, poisson=False, exponential=False), tie,
                         dict(seed=1, rid=0, end_s=6, expect_tie=True))
    return c


def build_case(model, build_schedule, kw):
    """The reference's Simulation of a case, built and not run: (harness context, Simulation, FaultSchedule, the
    lowering.fault_events of the schedule, the model plus its FAULT rows)"""
    RH._import_reference()
    from happysimulator import faults as F
    from happysimulator.core.simulation import Simulation
    from happysimulator.core.temporal import Instant
    end_ns = int(kw["end_s"] * 1e9)
    ctx = RH.run_reference(model, seed=kw["seed"], rid=kw["rid"], end_ns=end_ns, chash_vnodes=kw.get("chash_vnodes"),
                           sketch_seeds=kw.get("sketch_seeds"), zipf_s=kw.get("zipf_s"),
                           profile_objects=kw.get("profile_objects"), _build_only=True)
    objs = ctx["objs"]
    schedule = build_schedule({getattr(o, "name", None): o for o in objs}, F)
    handles = list(schedule._handles)
    sim = Simulation(end_time=Instant(end_ns), sources=ctx["sources"], entities=ctx["entities"],
                     probes=ctx["probes"] or None, fault_schedule=schedule)
    for k in kw.get("cancel", []):
        handles[k].cancel()
    # the model's rows plus one FAULT row per fault event, as lowering.lower appends them
    oid = {id(o): i for i, o in enumerate(objs)}
    fev = lowering.fault_events(schedule, ctx["sources"], ctx["entities"], ctx["probes"])
    rows = [(A.HS_ENT_FAULT, oid[id(tgt)], 0, int(crash), int(ev._cancelled), idx, t_ns, 0.0, 0.0)
            for tgt, t_ns, crash, idx, ev in fev]
    fm = dataclasses.replace(model, entities=np.concatenate([model.entities, np.array(rows, dtype=A.ENTITY_DTYPE)]),
                             names=list(model.names) + [f"fault:{tgt.name}" for tgt, *_ in fev])
    return ctx, sim, schedule, fev, fm


def run_case(model, build_schedule, kw):
    ctx, sim, schedule, fev, fm = build_case(model, build_schedule, kw)
    objs = ctx["objs"]
    row_of = {id(ev): model.n_entities + k for k, (*_, ev) in enumerate(fev)}
    fired = {i: 0 for i in row_of.values()}
    cancelled = {i: 0 for i in row_of.values()}
    recs = ctx["attach"](sim)
    heap = sim._event_heap
    inner = heap.pop
    import heapq

    def tap():
        top = heap._heap[0]
        if id(top) not in row_of:
            n0 = len(recs)
            crashed = bool(getattr(top.target, "_crashed", False))
            ev = inner()
            if crashed and len(recs) > n0:
                dropped.add(n0)                      # Event.invoke returns [] (core/event.py:261-262)
            return ev
        ev = heapq.heappop(heap._heap)              # EventHeap.pop for a fault event (it is never a daemon-counted one
        if ev._cancelled:                            # in these runs: auto-termination is off with an end_time)
            cancelled[row_of[id(ev)]] += 1
        elif not ev.time < sim._clock.now:
            recs.append((ev.time.nanoseconds, ev._sort_index, A.HS_EV_FAULT, row_of[id(ev)]))
            fired[row_of[id(ev)]] += 1
        return ev

    dropped = set()
    heap.pop = tap
    summary = sim.run()
    # a dropped event leaves no sample and no handled response: hide it from the harness's bookkeeping, then put the
    # true record stream (and its hash) back
    masked = [(t, i, 255 if k in dropped else kd, e) for k, (t, i, kd, e) in enumerate(recs)]
    ref = ctx["extract"](sim, masked, summary)
    if recs:
        arr = np.array(recs, dtype=np.int64)
        rec = np.zeros(len(recs), A.RECORD_DTYPE)
        rec["time_ns"], rec["sort_index"], rec["kind"], rec["entity"] = arr[:, 0], arr[:, 1], arr[:, 2], arr[:, 3]
        ref["records"] = rec
    import oracle_lib as O
    h = 0xcbf29ce484222325
    for t, i, kd, e in recs:
        h = O.lib().hs_cpu_hash_step(h, t, i, kd, e)
    ref["summaries"]["order_hash"] = h
    stats = np.zeros((1, fm.n_entities), A.STATS_DTYPE)
    stats[0, :model.n_entities] = ref["entity_stats"][0]
    for i in fired:
        stats[0, i]["c0"], stats[0, i]["c1"] = fired[i], cancelled[i]
    ref["entity_stats"] = stats
    assert summary.events_cancelled == sum(cancelled.values())
    keys = {}
    for t, i, kd, e in recs:
        keys.setdefault((t, i), set()).add(kd == A.HS_EV_FAULT)
    tied = any(len(v) == 2 for v in keys.values())
    assert kw.get("expect_tie") == "any" or tied == bool(kw.get("expect_tie")), "a tie of an in-run event with a fault event " + ("did not occur" if not tied else "occurred")
    crashed = np.array([int(bool(getattr(o, "_crashed", False))) for o in objs], dtype=np.int8)
    fstats = schedule.stats
    meta = dict(kw, crashed=crashed, events_cancelled=np.array(summary.events_cancelled, dtype=np.int64),
                fault_stats=np.array([fstats.faults_scheduled, fstats.faults_activated, fstats.faults_deactivated,
                                      fstats.faults_cancelled], dtype=np.int64))
    meta.pop("cancel", None); meta.pop("expect_tie", None); meta.pop("chash_vnodes", None); meta.pop("profile_objects", None)
    return fm, ref, meta


def main():
    for name, (model, build, kw) in cases().items():
        fm, ref, meta = run_case(model, build, kw)
        GG.save_case(os.path.join(HERE, f"fault_{name}.npz"), fm, ref, meta)
        print(f"fault_{name}: {len(ref['records'])} events, cancelled {int(meta['events_cancelled'])}, "
              f"heap_left {int(ref['summaries']['heap_left'][0])}")


if __name__ == "__main__":
    main()
