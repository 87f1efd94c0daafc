"""Record the fixtures of time buckets in linked partitions (tests/golden/lbucket_*.npz)
from the UNMODIFIED reference: its ParallelSimulation + WindowedCoordinator with the Philox plug-ins
(ref_harness.run_reference_linked; with a fault schedule, gen_linked_fault_golden.run_case).  The partitions are the
models this package lowers the mirror scripts of tests/linked_bucket_models.py to; the reference runs its own
LatencyTracker, ThroughputTracker and Probe classes for their rows.  The harness builds a Sink for every SINK row; here
the rows of a tracker get the reference's tracker class instead, which also keeps the Sink's bookkeeping the harness
reads (events_received, latencies_s, completion_times), so the records, samples and statistics are those of
gen_linked_golden.save.  The Probe rows are the harness's own reference Probe objects (instrumentation/probe.py).

    python tests/golden/gen_linked_bucket_golden.py          # needs the reference checkout

On top of gen_linked_golden.save's arrays (and gen_linked_fault_golden.save's for the fault case): every partition's
rate profiles p{q}_profiles / p{q}_profile_table (its Probes tick through them), bucket_w, bucket_n,
and for every bucketed row b (SINK and PROBE rows in entity order) of partition q the reference's own
Data.bucket(bucket_w) lists p{q}_bucket{b}_{times, counts, means, sums, maxes, p50s, p99s}."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import __graft_entry__  # noqa: E402,F401  (puts the repository root on sys.path)
from happysim_b200 import _abi as A, buckets as B  # noqa: E402
from happysim_b200.linked import LinkedModel  # noqa: E402

import gen_linked_fault_golden as GF  # noqa: E402
import gen_linked_golden as GL  # noqa: E402
import linked_bucket_models as LB  # noqa: E402
import ref_harness as RH  # noqa: E402


def _tracker_sinks(kinds):
    """Install a Sink class whose construction by name gives the reference's LatencyTracker / ThroughputTracker for the
    names in ``kinds`` (name -> "lat" | "tp"); returns the function that restores the module."""
    RH._import_reference()
    import happysimulator.components.common as CM
    from happysimulator.instrumentation.collectors import LatencyTracker, ThroughputTracker
    orig = CM.Sink

    class SinkOrTracker(orig):
        def __new__(cls, name="Sink"):
            if cls is SinkOrTracker and name in kinds:
                return object.__new__(Lat if kinds[name] == "lat" else Tp)
            return object.__new__(cls)

    class _Both:
        def handle_event(self, event):
            orig.handle_event(self, event)                  # the harness's bookkeeping (latency, completion time)
            return self._tracker.handle_event(self, event)  # the reference tracker's own Data

    class Lat(_Both, LatencyTracker, SinkOrTracker):
        _tracker = LatencyTracker

    class Tp(_Both, ThroughputTracker, SinkOrTracker):
        _tracker = ThroughputTracker

    CM.Sink = SinkOrTracker

    def restore():
        CM.Sink = orig
    return restore


def _bucket_lists(model, objs):
    """per bucketed row: the reference's Data.bucket(W) of its tracker, Probe Data or (a plain Sink) its samples"""
    from happysimulator.core.temporal import Instant
    from happysimulator.instrumentation.data import Data
    out = []
    for i in B.rows(model):
        o = objs[i]
        if isinstance(o, Data):
            d = o
        elif hasattr(o, "data"):
            d = o.data
        else:
            d = Data()
            for t, v in zip(o.completion_times, o.latencies_s):
                d.add_stat(v, t if isinstance(t, Instant) else Instant(int(t)))
        out.append(LB.lists(d.bucket(LB.W)))
    return out


def _save_buckets(path, lm, outs):
    z = dict(np.load(path))
    z["bucket_w"], z["bucket_n"] = np.float64(LB.W), np.int64(LB.NB)
    for q, (m, o) in enumerate(zip(lm.models, outs)):
        z[f"p{q}_profiles"] = m.profiles if m.profiles is not None else np.zeros(0)
        z[f"p{q}_profile_table"] = m.profile_table if m.profile_table is not None else np.zeros(0)
        for b, ls in enumerate(_bucket_lists(m, o["objects"])):
            for f, v in ls.items():
                z[f"p{q}_bucket{b}_{f}"] = np.array(v, dtype=np.int64 if f == "counts" else np.float64)
    np.savez_compressed(path, **z)


def main():
    for name, (script, schedules) in LB.CASES.items():
        ps = script()
        plm = ps._linked
        kinds = {}
        for m, objs in zip(plm.models, plm.objects):
            for i, o in enumerate(objs):
                if int(m.entities["kind"][i]) == A.HS_ENT_SINK and hasattr(o, "data"):
                    kinds[m.names[i]] = "tp" if B._is_throughput(o) else "lat"
        seed, end_s = ps._seed, ps._end_ns / 1e9
        # the partitions without their FAULT rows: the fault generator appends them from the schedules
        lm = LinkedModel([_without_faults(m) for m in plm.models], list(plm.names), plm.links, window_s=plm.window_s,
                         n_streams=plm.n_streams)
        restore = _tracker_sinks(kinds)
        try:
            if schedules is None:
                outs, summ = RH.run_reference_linked(lm, seed=seed, end_ns=int(end_s * 1e9))
                path = os.path.join(HERE, f"{name}.npz")
                GL.save(path, lm, outs, summ, dict(seed=seed, end_s=end_s))
                flm = lm
            else:
                flm, outs, summ, extra = GF.run_case(lm, schedules, seed=seed, end_s=end_s, expect_tie=False)
                GF.save(name, flm, outs, summ, extra, dict(seed=seed, end_s=end_s))
                path = os.path.join(HERE, f"{name}.npz")
                os.replace(os.path.join(HERE, f"lfault_{name}.npz"), path)
        finally:
            restore()
        _save_buckets(path, flm, outs)
        print(f"{name}: {summ.total_windows} windows, {summ.total_cross_partition_events} delivered, "
              f"{[int(o['summaries']['events_processed'][0]) for o in outs]} events, "
              f"{[len(B.rows(m)) for m in flm.models]} bucketed rows")


def _without_faults(model):
    """``model`` without its FAULT rows (the fault generator derives them from the schedule again)"""
    import dataclasses
    keep = model.entities["kind"] != A.HS_ENT_FAULT
    if keep.all():
        return model
    m = dataclasses.replace(model, entities=model.entities[keep].copy(), names=[n for n, k in zip(model.names, keep) if k])
    m.outbox_cap, m.inbox_cap = model.outbox_cap, model.inbox_cap
    return m


if __name__ == "__main__":
    main()
