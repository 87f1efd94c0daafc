"""Throughput of a linked ParallelSimulation ensemble on one GPU (DESIGN.md section 4.4): the tandem of the fixture
linked_tandem_const (A: Source -> Server -> [link, 50 ms] -> B: Server(c=2) -> Sink, 50 ms windows) and the three-partition
lossy fan-out, many replicas, timed with a host clock around LinkedRun.run ending in a device synchronise.

    python tools/bench_linked.py [--faults] [replicas ...]
    python tools/bench_linked.py --buckets W N [--percentiles] [--long] [replicas ...]
    python tools/bench_linked.py --sweep K [--rpc R] [--sim-s S]

--faults runs every configuration a second time with a node-fault schedule in every partition (fault_schedules):
the same ensemble then runs the LINKED | FAULTS kernels, and the two lines compare their throughput.

--buckets W N runs every configuration without and with time buckets (N buckets of W seconds, with --percentiles
also their p50 / p99), alternating, 5 rounds each, and prints the usual line for the bucketed run (its window loop,
the reads of the outputs taken off and reported as read_ms) with the bucket settings, the run without buckets, the
card and its power limit, read in the same process.  N must cover every configuration's end time (--long: 100 s, so
N > 100 / W).  --long adds the point a record-mode run could not hold: tandem_heavy
(500 req/s) for 100 s at 16 384 replicas, with buckets only (its recorder rings would need about 5 MB per
partition-replica, 165 GB in all).

--sweep K runs K configurations of linked_tandem_const (link latency 1x to 1.875x the window, mean service times 0.6x
to 1.4x), R replicas each (default 1), for S simulated seconds (default 20) in two ways, alternating, 5 rounds each: K
separate LinkedRuns, and one LinkedRun whose K sweep cells are the configurations (LinkedModel.from_cells, K * R
replicas).  Each is timed with a host clock that ends in a device synchronise, outputs read included; the line gives
both medians, whether every configuration's summaries came out the same both ways, and the card and its power limit.
"""
import json
import math
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
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


def card():
    """the card's name and power limit (nvidia-smi's query; None where it is not available)"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.splitlines()[torch.cuda.current_device()]
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), None


def timed(lm, seed, end_ns, n, **kw):
    """One LinkedRun.run after a warm-up: (window-loop seconds, seconds of the reads that follow it, outputs, counts,
    kernel flags per partition, windows).  LinkedRun.run ends with the reads of every partition's outputs (and of the
    bucket records, totals and percentiles): they are timed again on their own after the run and taken off, so the first
    figure is the window loop (launches, barriers, and a device synchronise)."""
    from happysim_b200 import buckets as B
    run = LinkedRun(lm)
    try:
        run.run(seed=seed, end_ns=int(1e9), n_replicas=n, flags=0, **kw)        # warm-up (allocations, module load)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs, counts = run.run(seed=seed, end_ns=end_ns, n_replicas=n, flags=0, **kw)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        bk = kw.get("buckets")
        bucketed = [q for q, m in enumerate(lm.models) if bk is not None and B.rows(m)]
        t1 = time.perf_counter()
        for q, e in enumerate(run.engines):
            e.read_outputs()
            if q in bucketed:                       # what LinkedRun.run reads after the last window
                B.read_outputs(e, bk, kw.get("bucket_sample_cap", 0), lm.models[q], [None] * lm.models[q].n_entities)
        reads = time.perf_counter() - t1
        return total - reads, reads, outs, counts, [e.last_launch()["flags"] for e in run.engines], run.windows
    finally:
        run.close()


def _line(name, lm, n, end_s, windows, outs, counts, flags, dt, faults=False):
    """the JSON fields every line of this tool carries"""
    delivered, lost, over = counts
    ev = sum(int(o["summaries"]["events_processed"].sum()) for o in outs)
    bits = 0
    for o in outs:
        bits |= int(np.bitwise_or.reduce(o["summaries"]["status"]))
    who = [(q, int(r)) for q, o in enumerate(outs) for r in (o["summaries"]["status"] != 0).nonzero()[0][:3]]
    return {"model": name, "faults": faults, "kernel_flags": flags, "partitions": lm.n_partitions, "replicas": n,
            "sim_s": end_s, "windows": windows, "events": ev, "cross_partition_events": int(delivered.sum()),
            "lost": int(lost.sum()), "inbox_overflows": int(over.sum()),
            "flagged": sum(int((o["summaries"]["status"] != 0).sum()) for o in outs), "status_bits": bits,
            "flagged_where": who, "wall_ms": round(dt * 1e3, 2), "events_per_s": round(ev / dt, 1),
            "us_per_window": round(dt * 1e6 / windows, 1)}


def bench_buckets(args):
    """--buckets W N [--percentiles] [--long]: without / with buckets, alternating, median of 5 rounds"""
    k = args.index("--buckets")
    w, nb = float(args[k + 1]), int(args[k + 2])
    pct = "--percentiles" in args
    rest = args[:k] + args[k + 3:]
    sizes = [int(a) for a in rest if not a.startswith("--")] or [4096, 16384, 65536]
    name_, limit = card()
    cases = [(c, n, True) for c in (("linked_tandem_const", 20.0), ("linked_lossy_fanout", 10.0)) for n in sizes]
    if "--long" in args:
        cases.append((("linked_tandem_heavy", 100.0), 16384, False))
    for (_, end_s), _, _ in cases:
        if math.floor(end_s / w) >= nb:
            sys.exit(f"--buckets {w} {nb}: {nb} buckets of {w} s end before the end time {end_s} s of a configuration; "
                     f"pass at least {math.floor(end_s / w) + 1}")
    cap = 128 if pct else 0         # holds every 0.1 s bucket of tandem_heavy (about 50 samples)
    for (name, end_s), n, both in cases:
        lm, kw, z = G.load_linked(name)
        end_ns = int(end_s * 1e9)
        bk = dict(buckets=(w, nb), bucket_sample_cap=cap)
        t_plain, t_bk, r_bk = [], [], []
        for _ in range(5):
            if both:
                t_plain.append(timed(lm, kw["seed"], end_ns, n)[0])
            dt, rd, outs, counts, flags, windows = timed(lm, kw["seed"], end_ns, n, **bk)
            t_bk.append(dt)
            r_bk.append(rd)
        line = _line(name, lm, n, end_s, windows, outs, counts, flags, statistics.median(t_bk))
        line.update({"bucket_width_s": w, "buckets": nb, "percentiles": pct, "bucket_sample_cap": cap,
                     "wall_ms_without_buckets": round(statistics.median(t_plain) * 1e3, 2) if t_plain else None,
                     "read_ms": round(statistics.median(r_bk) * 1e3, 2), "rounds": 5,
                     "timed": "window loop of LinkedRun.run (launches and barriers, device synchronise), reads excluded",
                     "card": name_, "power_limit": limit})
        print(json.dumps(line), flush=True)


def sweep_configs(lm, K):
    """K LinkedModels of lm's topology: server mean service times 0.6x to 1.4x, link latency 1x to 1.875x"""
    import dataclasses
    out = []
    for k in range(K):
        models = []
        for m in lm.models:
            E = m.entities.copy()
            srv = E["kind"] == A.HS_ENT_SERVER
            E["d0"][srv] = E["d0"][srv] * (0.6 + 0.8 * k / max(1, K - 1))
            models.append(dataclasses.replace(m, entities=E))
        links = [[dataclasses.replace(l, latency_mean_s=l.latency_mean_s * (1 + (k % 8) / 8)) for l in ls] for ls in lm.links]
        out.append(dataclasses.replace(lm, models=models, links=links))
    return out


def bench_sweep(args):
    """--sweep K [--rpc R] [--sim-s S]: K separate LinkedRuns against one celled LinkedRun, alternating, median of 5"""
    from happysim_b200.linked import LinkedModel
    opt = lambda f, d: type(d)(args[args.index(f) + 1]) if f in args else d      # noqa: E731
    K, rpc, end_s = opt("--sweep", 16), opt("--rpc", 1), opt("--sim-s", 20.0)
    name_, limit = card()
    lm, kw, z = G.load_linked("linked_tandem_const")
    cfgs = sweep_configs(lm, K)
    celled = LinkedModel.from_cells(cfgs)
    end_ns, seed = int(end_s * 1e9), kw["seed"]

    def separate():
        res = []
        for k, c in enumerate(cfgs):       # configuration k's replicas keep their global index, hence their draws
            run = LinkedRun(c)
            try:
                outs, counts = run.run(seed=seed, end_ns=end_ns, n_replicas=rpc, replica_index_base=k * rpc, flags=0)
            finally:
                run.close()
            res.append(outs)
        return res

    def one():
        run = LinkedRun(celled)
        try:
            return run.run(seed=seed, end_ns=end_ns, n_replicas=K * rpc, replicas_per_cell=rpc, flags=0)
        finally:
            run.close()

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    separate(), one()                # warm-up (module load, allocations)
    t_sep, t_one = [], []
    for _ in range(5):
        dt, sep = clock(separate)
        t_sep.append(dt)
        dt, (outs, counts) = clock(one)
        t_one.append(dt)
    same = all(outs[q]["summaries"][k * rpc:(k + 1) * rpc].tobytes() == sep[k][q]["summaries"].tobytes()
               for k in range(K) for q in range(lm.n_partitions))
    bits = 0
    for o in outs:
        bits |= int(np.bitwise_or.reduce(o["summaries"]["status"]))
    ev = sum(int(o["summaries"]["events_processed"].sum()) for o in outs)
    a, b = statistics.median(t_sep), statistics.median(t_one)
    print(json.dumps({"mode": "sweep", "model": "linked_tandem_const", "configs": K, "replicas_per_config": rpc,
                      "sim_s": end_s, "windows": len(lm.window_ends(end_ns)), "events": ev, "status_bits": bits,
                      "separate_runs_ms": round(a * 1e3, 2), "celled_run_ms": round(b * 1e3, 2),
                      "speedup": round(a / b, 2), "same_summaries": same, "rounds": 5,
                      "timed": "host clock around the runs (outputs read), ending in a device synchronise",
                      "card": name_, "power_limit": limit}), flush=True)


def main():
    args = sys.argv[1:]
    if "--buckets" in args:
        return bench_buckets(args)
    if "--sweep" in args:
        return bench_sweep(args)
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
