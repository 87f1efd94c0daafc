"""Record the fixtures of linked partitions with node faults (tests/golden/lfault_*.npz, random_linked_faults.npz) from
the UNMODIFIED reference: its ParallelSimulation + WindowedCoordinator (ref_harness.run_reference_linked, Philox
plug-ins as in gen_linked_golden.py), every partition handed its own ``happysimulator.faults.FaultSchedule`` through
``SimulationPartition(fault_schedule=)``.  As in gen_fault_golden.py, a pop tap records the fault events itself (kind
HS_EV_FAULT, entity = the FAULT row of the partition's model), counts the cancelled ones and masks the events a crashed
entity drops from the harness's sample bookkeeping.  Each partition's model is its rows plus the FAULT rows
lowering.fault_events gives that partition's schedule; the generator asserts that these are the rows
tests/linked_fault_models.fault_rows derives (sort indices from the partition's own counter).

    python tests/golden/gen_linked_fault_golden.py          # needs the reference checkout
    python tests/golden/gen_linked_fault_golden.py random   # only random_linked_faults.npz

Per fixture, on top of gen_linked_golden.save's arrays: per partition the reference's events_cancelled, the _crashed
flag of every row's object after the run, and whether a delivered or in-run event tied with a fault event
(p{q}_tie: a pushed event met a fault event with its time and sort index in the heap -- in the grid tie case only,
which the generator asserts)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import __graft_entry__  # noqa: E402,F401  (puts the repository root on sys.path)
import happysim_b200 as hs  # noqa: E402
from happysim_b200 import _abi as A, lowering  # noqa: E402
from happysim_b200.linked import LinkedModel, LinkSpec  # noqa: E402

import gen_linked_golden as GL  # noqa: E402
import linked_fault_models as LF  # noqa: E402
import random_models as RM  # noqa: E402
import ref_harness as RH  # noqa: E402

CONST, EXPO = A.HS_SVC_CONSTANT, A.HS_SVC_EXPONENTIAL


def busy_sender():
    """A: Source(60/s) -> Server(c=1, exp 15 ms: a queue builds up) -> [50 ms link] -> B: Server(c=2) -> Sink"""
    a = hs.ModelBuilder()
    src = a.source("A.src", rate=60.0)
    sa = a.server("A.server", mean_service_s=0.015)
    rem = a.remote("B.server@A", link=0, dest_entity=0)
    a.set_target(src, sa); a.set_target(sa, rem)
    ma = a.build(); ma.outbox_cap = 64
    b = hs.ModelBuilder()
    sb = b.server("B.server", concurrency=2, mean_service_s=0.01)
    b.set_target(sb, b.sink("B.sink"))
    mb = b.build(); mb.inbox_cap = 64
    return LinkedModel([ma, mb], ["A", "B"], [[LinkSpec(1, CONST, 0.05, 0.0, 0)], []], window_s=0.05)


def fan_in():
    """A and B: Source -> Server -> [links of 50 and 75 ms, one latency object each] -> C: Server(c=2) -> Sink"""
    ms = []
    for p, rate in (("A", 30.0), ("B", 45.0)):
        b = hs.ModelBuilder()
        src = b.source(f"{p}.src", rate=rate)
        s = b.server(f"{p}.server", mean_service_s=0.008)
        rem = b.remote(f"C.server@{p}", link=0, dest_entity=0)
        b.set_target(src, s); b.set_target(s, rem)
        m = b.build(); m.outbox_cap = 64
        ms.append(m)
    c = hs.ModelBuilder()
    sc = c.server("C.server", concurrency=2, mean_service_s=0.02)
    c.set_target(sc, c.sink("C.sink"))
    mc = c.build(); mc.inbox_cap = 128
    links = [[LinkSpec(2, CONST, 0.05, 0.0, 0)], [LinkSpec(2, EXPO, 0.075, 0.0, 1)], []]
    return LinkedModel(ms + [mc], ["A", "B", "C"], links, window_s=0.05, n_streams=2)


def grid_pair():
    """A: constant Source(100/s) -> Server(constant 5 ms) -> [constant 20 ms link] -> B: Server(c=1, constant 5 ms) ->
    Counter: every event on a 5 ms grid, B's deliveries carry A's small early sort indices.  B's own constant source
    (-> a second Counter) stops B's windows on time, so a fault event just past a window end is still pending when the
    barrier delivers"""
    a = hs.ModelBuilder()
    src = a.source("A.src", rate=100.0, poisson=False)
    sa = a.server("A.server", mean_service_s=0.005, exponential=False)
    rem = a.remote("B.server@A", link=0, dest_entity=0)
    a.set_target(src, sa); a.set_target(sa, rem)
    ma = a.build(); ma.outbox_cap = 64
    b = hs.ModelBuilder()
    sb = b.server("B.server", mean_service_s=0.005, exponential=False)
    b.set_target(sb, b.counter("B.counter"))
    b.set_target(b.source("B.tick", rate=200.0, poisson=False), b.counter("B.ticks"))   # ends B's windows on time
    mb = b.build(); mb.inbox_cap = 64
    return LinkedModel([ma, mb], ["A", "B"], [[LinkSpec(1, CONST, 0.02, 0.0, 0)], []], window_s=0.02)


def _at_window_end(lm, end_ns, k):
    """a time in seconds that Instant.from_seconds turns into exactly the k-th window end"""
    w = lm.window_ends(end_ns)[k]
    for t in (w / 1e9, round(w / 1e9, 9), np.nextafter(w / 1e9, 1.0), np.nextafter(w / 1e9, 0.0)):
        if LF.from_seconds(float(t)) == w:
            return float(t)
    raise AssertionError(f"no float second lands on window end {w}")


def _grid_tie_schedule(lm, end_s):
    """B's first delivered request, found on the fault-free run of the fault oracle: a crash of B.server at its time,
    with its sort index (the fault events before it, one index each, lie beyond end_time)"""
    import linked_fault_oracle_lib as FO
    import oracle_lib as O
    end_ns = int(end_s * 1e9)
    ps = [O.make_params(seed=3, end_ns=end_ns, rid_base=q, rid_stride=3, record_cap=4096, sample_cap=16, service_cap=16)
          for q in range(2)]
    outs, *_ = FO.run_linked(lm, ps, end_ns=end_ns, cseed=3)
    rec = outs[1]["records"][0]
    first = rec[rec["kind"] == A.HS_EV_REQ_ENQUEUE][0]
    t_ns, idx = int(first["time_ns"]), int(first["sort_index"])
    t_s = t_ns / 1e9
    n = idx - 1                                         # B's one source takes bootstrap index 0
    assert LF.from_seconds(t_s) == t_ns and n >= 0, (t_ns, idx)
    pads = [("pause", "B.counter", end_s + 1.0 + k, end_s + 1.5 + k, False) for k in range(n // 2)]
    pads += [("crash", "B.counter", end_s + 0.5, None, False)] * (n % 2)
    return [[], pads + [("crash", "B.server", t_s, t_s + 0.1, False)]]


def cases():
    """name -> (LinkedModel, per-partition schedules (linked_fault_models), run kwargs)"""
    c = {}
    c["tandem_crash_downstream"] = (GL.tandem_over_a_link(), [[], [("crash", "B.server", 1.0, 2.2, False)]],
                                    dict(seed=5, end_s=4.0))
    c["tandem_pause_sink"] = (GL.tandem_over_a_link(kind=EXPO), [[], [("pause", "B.sink", 1.3, 2.6, False)]],
                              dict(seed=7, end_s=4.0))
    c["sender_crash_drains"] = (busy_sender(), [[("crash", "A.server", 1.0, 2.0, False)], []], dict(seed=11, end_s=3.0))
    fi = fan_in()
    end_s = 3.0
    t_w = _at_window_end(fi, int(end_s * 1e9), 23)
    c["fanin_mixed"] = (fi, [[("crash", "A.server", 1.0, 1.5, True)],                  # a cancelled handle
                             [("crash", "B.server", 0.7, 0.9, False)],
                             [("crash", "C.server", 0.0, 0.4, False),                   # at t = 0
                              ("pause", "C.server", 0.8, 1.6, False),
                              ("crash", "C.server", 1.2, 1.4, False),                   # clears the flag inside the pause
                              ("crash", "C.sink", t_w, 2.2, False),                     # exactly at a window end
                              ("crash", "C.sink", 2.5, 9.0, False)]],                   # its restart after end_time
                        dict(seed=13, end_s=end_s))
    gp = grid_pair()
    c["grid_tie"] = (gp, _grid_tie_schedule(gp, 1.0), dict(seed=3, end_s=1.0, expect_tie=True))
    return c


def run_case(lm, schedules, *, seed, end_s, expect_tie=False):
    """The reference on ``lm`` with partition q's schedule ``schedules[q]``: (LinkedModel with the FAULT rows,
    per-partition outputs, the ParallelSimulationSummary, per-partition extras)."""
    RH._import_reference()
    import heapq
    import happysimulator.parallel.coordinator as CO
    import happysimulator.parallel.partition as PP
    from happysimulator import faults as F
    flm = LF.linked_with_faults(lm, schedules)
    ref_sched = {}
    for q, faults in enumerate(schedules):
        s = F.FaultSchedule()
        for cls, name, t0, t1, _ in faults:
            s.add(F.CrashNode(name, at=t0, restart_at=t1) if cls == "crash" else F.PauseNode(name, start=t0, end=t1))
        ref_sched[lm.names[q]] = s
    ctxs = []
    extra = [dict() for _ in range(lm.n_partitions)]
    orig_run_reference, orig_part = RH.run_reference, PP.SimulationPartition

    def run_reference(model, **kw):
        q = len(ctxs)
        ctx = orig_run_reference(model, **kw)
        ctxs.append(ctx)
        attach0, extract0 = ctx["attach"], ctx["extract"]
        n0 = model.n_entities

        def attach(sim):
            recs = attach0(sim)
            schedule = ref_sched[lm.names[q]]
            for h, f in zip(schedule._handles, schedules[q]):       # FaultHandle.cancel() between building and run()
                if f[4]:
                    h.cancel()
            fev = lowering.fault_events(schedule, ctx["sources"], ctx["entities"], ctx["probes"])
            oid = {id(o): i for i, o in enumerate(ctx["objs"])}
            rows = [(A.HS_ENT_FAULT, oid[id(tgt)], 0, int(crash), int(ev._cancelled), idx, t_ns, 0.0, 0.0)
                    for tgt, t_ns, crash, idx, ev in fev]
            want = LF.fault_rows(model, schedules[q])[0]
            assert rows == want, (lm.names[q], rows, want)          # the partition's own counter, its own names
            row_of = {id(ev): n0 + k for k, (*_, ev) in enumerate(fev)}
            st = extra[q]
            st.update(recs=recs, dropped=set(), tie=False, fired={i: 0 for i in row_of.values()}, cancelled={i: 0 for i in row_of.values()})
            heap = sim._event_heap
            inner = heap.pop

            def tap():
                top = heap._heap[0]
                if id(top) not in row_of:
                    n_before = len(recs)
                    crashed = bool(getattr(top.target, "_crashed", False))
                    ev = inner()
                    if crashed and len(recs) > n_before:
                        st["dropped"].add(n_before)          # Event.invoke returns [] (core/event.py:261-262)
                    return ev
                ev = heapq.heappop(heap._heap)
                if ev._cancelled:
                    st["cancelled"][row_of[id(ev)]] += 1
                elif not ev.time < sim._clock.now:
                    recs.append((ev.time.nanoseconds, ev._sort_index, A.HS_EV_FAULT, row_of[id(ev)]))
                    st["fired"][row_of[id(ev)]] += 1
                return ev
            heap.pop = tap
            push = heap.push

            def push_tap(events):
                # a tie heapq orders by its array layout: a pushed event with the (time, sort index) of a fault event
                # still in the heap (or a pushed fault event with another's).  The engines schedule a barrier's
                # deliveries when the next window starts, so those of the last barrier are left out.
                if not barrier["last"]:
                    for ev in (events if isinstance(events, list) else [events]):
                        key = (ev.time, ev._sort_index)
                        if any((e.time, e._sort_index) == key and (id(e) in row_of or id(ev) in row_of) for e in heap._heap):
                            st["tie"] = True
                return push(events)
            heap.push = push_tap
            return recs

        def extract(sim, recs, summary):
            st = extra[q]
            masked = [(t, i, 255 if k in st["dropped"] else kd, e) for k, (t, i, kd, e) in enumerate(recs)]
            ref = extract0(sim, masked, summary)
            rec = np.zeros(len(recs), A.RECORD_DTYPE)
            if recs:
                arr = np.array(recs, dtype=np.int64)
                rec["time_ns"], rec["sort_index"], rec["kind"], rec["entity"] = arr[:, 0], arr[:, 1], arr[:, 2], arr[:, 3]
            ref["records"] = rec
            import oracle_lib as O
            h = 0xcbf29ce484222325
            for t, i, kd, e in recs:
                h = O.lib().hs_cpu_hash_step(h, t, i, kd, e)
            ref["summaries"]["order_hash"] = h
            stats = np.zeros((1, flm.models[q].n_entities), A.STATS_DTYPE)
            stats[0, :n0] = ref["entity_stats"][0]
            for i in st["fired"]:
                stats[0, i]["c0"], stats[0, i]["c1"] = st["fired"][i], st["cancelled"][i]
            ref["entity_stats"] = stats
            assert summary.events_cancelled == sum(st["cancelled"].values())
            st["events_cancelled"] = int(summary.events_cancelled)
            st["crashed"] = np.array([int(bool(getattr(o, "_crashed", False))) for o in ctx["objs"]], dtype=np.int8)
            return ref
        ctx["attach"], ctx["extract"] = attach, extract
        return ctx

    def partition(**kw):
        return orig_part(**kw, fault_schedule=ref_sched[kw["name"]])
    n_windows = len(lm.window_ends(int(end_s * 1e9)))
    barrier = dict(n=0, last=False)
    orig_exchange = CO.WindowedCoordinator._exchange_events

    def exchange(self, window_end):
        barrier["n"] += 1
        barrier["last"] = barrier["n"] == n_windows
        try:
            return orig_exchange(self, window_end)
        finally:
            barrier["last"] = False
    RH.run_reference, PP.SimulationPartition, CO.WindowedCoordinator._exchange_events = run_reference, partition, exchange
    try:
        outs, summ = RH.run_reference_linked(lm, seed=seed, end_ns=int(end_s * 1e9))
    finally:
        RH.run_reference, PP.SimulationPartition, CO.WindowedCoordinator._exchange_events = \
            orig_run_reference, orig_part, orig_exchange
    assert barrier["n"] <= n_windows          # the coordinator stops early once every heap is empty
    tied = [bool(e["tie"]) for e in extra]
    assert expect_tie is None or any(tied) == expect_tie, "a tie of a delivered or in-run event with a fault event " + \
        ("did not occur" if not any(tied) else "occurred")
    return flm, outs, summ, extra


def save(name, flm, outs, summ, extra, kw):
    path = os.path.join(HERE, f"lfault_{name}.npz")
    GL.save(path, flm, outs, summ, dict(seed=kw["seed"], end_s=kw["end_s"]))
    z = dict(np.load(path))
    for q, e in enumerate(extra):
        z[f"p{q}_events_cancelled"] = np.int64(e["events_cancelled"])
        z[f"p{q}_crashed"] = e["crashed"]
        z[f"p{q}_tie"] = np.int64(e["tie"])
    np.savez_compressed(path, **z)


def random_cases():
    rows, tops = [], []
    for seed in range(LF.RANDOM_SEEDS):
        lm, end_s, what = RM.random_linked_model(seed)
        sch = LF.random_schedules(lm, end_s, seed)
        _, outs, summ, extra = run_case(lm, sch, seed=1000 + seed, end_s=end_s, expect_tie=None)
        for q, o in enumerate(outs):
            s = o["summaries"][0]
            rows.append((seed, q, int(s["events_processed"]), int(s["final_time_ns"]), int(s["order_hash"]), int(s["heap_left"]),
                         int(s["n_sink_samples"]), int(s["n_service_samples"]), LF.digest(o["entity_stats"][0]),
                         extra[q]["events_cancelled"], int(extra[q]["tie"])))
        tops.append((seed, summ.total_windows, summ.total_cross_partition_events, summ.total_events_processed))
        print(what, "->", summ.total_events_processed, "events,", summ.total_cross_partition_events, "delivered,",
              sum(e["events_cancelled"] for e in extra), "cancelled")
    np.savez_compressed(os.path.join(HERE, "random_linked_faults.npz"), rows=np.array(rows, dtype=LF.ROW),
                        tops=np.array(tops, dtype=LF.TOP))


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    if only != "random":
        for name, (lm, schedules, kw) in cases().items():
            if only not in name:
                continue
            flm, outs, summ, extra = run_case(lm, schedules, **kw)
            save(name, flm, outs, summ, extra, kw)
            print(f"lfault_{name}: {summ.total_windows} windows, {summ.total_cross_partition_events} delivered, "
                  f"{[int(o['summaries']['events_processed'][0]) for o in outs]} events, "
                  f"cancelled {[e['events_cancelled'] for e in extra]}, tie {[e['tie'] for e in extra]}")
    if only in ("", "random"):
        random_cases()


if __name__ == "__main__":
    main()
