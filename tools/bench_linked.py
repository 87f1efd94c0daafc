"""Throughput of a linked ParallelSimulation ensemble on one GPU (DESIGN.md section 4.4): the tandem of the fixture
linked_tandem_const (A: Source -> Server -> [link, 50 ms] -> B: Server(c=2) -> Sink, 50 ms windows) and the three-partition
lossy fan-out, many replicas, timed with CUDA events around the whole window loop.

    python tools/bench_linked.py [--faults] [replicas ...]

--faults runs every configuration a second time with a node-fault schedule in every partition (fault_schedules):
the same ensemble then runs the LINKED | FAULTS kernels, and the two lines compare their throughput.
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import happysim_b200  # noqa: F401,E402
import golden_lib as G  # noqa: E402
import linked_fault_models as LF  # noqa: E402
from happysim_b200 import _abi as A  # noqa: E402
from happysim_b200.linked import LinkedRun  # noqa: E402


def fault_schedules(lm, end_s):
    """per partition that has a Source of its own: its first Server crashed from 25 % to 40 % of the run, and paused
    from 60 % to 70 %.  A partition without a Source is left alone: its only local events would be the fault events,
    so its first window would run its clock ahead to the first of them (the overshoot rule) and every delivery until
    then would wait in its heap, beyond what the device's event list holds (DESIGN.md section 4.2c)."""
    out = []
    for m in lm.models:
        kinds = [int(k) for k in m.entities["kind"]]
        tgt = next((i for i, k in enumerate(kinds) if k == A.HS_ENT_SERVER), None) if A.HS_ENT_SOURCE in kinds else None
        out.append([] if tgt is None else [("crash", m.names[tgt], 0.25 * end_s, 0.4 * end_s, False),
                                           ("pause", m.names[tgt], 0.6 * end_s, 0.7 * end_s, False)])
    return out


def main():
    args = sys.argv[1:]
    faults = "--faults" in args
    sizes = [int(a) for a in args if a != "--faults"] or [4096, 16384, 65536]
    for (name, end_s), with_faults in [(c, f) for c in (("linked_tandem_const", 20.0), ("linked_lossy_fanout", 10.0))
                                       for f in ((False, True) if faults else (False,))]:
        lm, kw, z = G.load_linked(name)
        if with_faults:
            lm = LF.linked_with_faults(lm, fault_schedules(lm, end_s))
        for n in sizes:
            run = LinkedRun(lm)
            try:
                end_ns = int(end_s * 1e9)
                run.run(seed=kw["seed"], end_ns=int(1e9), n_replicas=n, flags=0)            # warm-up (allocations, module load)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs, (delivered, lost, over) = run.run(seed=kw["seed"], end_ns=end_ns, n_replicas=n, flags=0)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                flags = [e.last_launch()["flags"] for e in run.engines]
            finally:
                run.close()
            ev = sum(int(o["summaries"]["events_processed"].sum()) for o in outs)
            bad = sum(int((o["summaries"]["status"] != 0).sum()) for o in outs)
            bits = 0
            for o in outs:
                for x in o["summaries"]["status"]:
                    bits |= int(x)
            who = [(q, int(r)) for q, o in enumerate(outs) for r in (o["summaries"]["status"] != 0).nonzero()[0][:3]]
            print(json.dumps({"model": name, "faults": with_faults, "kernel_flags": flags,
                              "partitions": lm.n_partitions, "replicas": n, "sim_s": end_s, "windows": run.windows,
                              "events": ev, "cross_partition_events": int(delivered.sum()), "lost": int(lost.sum()),
                              "inbox_overflows": int(over.sum()), "flagged": bad, "status_bits": bits, "flagged_where": who, "wall_ms": round(dt * 1e3, 2),
                              "events_per_s": round(ev / dt, 1), "us_per_window": round(dt * 1e6 / run.windows, 1)}), flush=True)


if __name__ == "__main__":
    main()
