"""Device throughput of PriorityQueue servers against FIFO servers on the same farm: configs[2]'s Source(512/s) ->
LoadBalancer(RoundRobin) -> 64 x Server(1, Exp(0.1 s)) -> Sink, 16 384 replicas on the thread engine, once with FIFO
queues and once with two-class PriorityQueue servers (20 % of the keys priority 0, the rest 1).  The priority farm's
source draws a routing key (population 10, needed by PriorityByKey); the FIFO farm is run both without and with that
key draw, so the difference between the last two lines is the queue policy alone.

    python tools/bench_priority.py [--replicas N] [--sim-s S] [--reps R]

Prints one line per variant: best and median device time of R launches (CUDA events) and events per second, plus the
card's name and power limit."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import numpy as np                                   # noqa: E402

import happysim_b200 as hs                           # noqa: E402
from happysim_b200 import engine                     # noqa: E402


def farm(priority: bool, keyed: bool, n_servers=64, rate=512.0, K=10):
    b = hs.ModelBuilder()
    src = b.source(rate=rate, key_population=K if keyed else 0)
    table = [0.0, 0.0] + [1.0] * (K - 2)
    servers = [b.server(f"S{i}", mean_service_s=0.1, priorities=table if priority else None) for i in range(n_servers)]
    snk = b.sink()
    lb = b.load_balancer(backends=servers)
    b.set_target(src, lb)
    for s in servers:
        b.set_target(s, snk)
    return b.build()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=16384)
    ap.add_argument("--sim-s", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = "unknown"
    print(f"card: {card}; {a.replicas} replicas, {a.sim_s} simulated s, thread engine, {a.reps} timed launches after one warm-up")
    for name, model in (("FIFO, no routing key", farm(False, False)), ("FIFO, keyed source", farm(False, True)),
                        ("PriorityQueue, two classes", farm(True, True))):
        eng = engine.Engine(0)
        eng.upload(model)
        p = engine.make_params(seed=1234, end_ns=int(a.sim_s * 1e9), n_replicas=a.replicas, flags=0, engine=3, queue_ring=512)
        eng.run(p)
        eng.sync()
        ms = []
        for _ in range(a.reps):
            eng.run(p)
            eng.sync()
            ms.append(eng.last_run_ms())
        out = eng.read_outputs()
        ev = int(out["summaries"]["events_processed"].sum())
        bad = int((out["summaries"]["status"] != 0).sum())
        best, med = min(ms), float(np.median(ms))
        print(f"{name:28s} events={ev:.4e} best {best:9.2f} ms  median {med:9.2f} ms  spread {max(ms) - best:7.2f} ms  "
              f"{ev / best / 1e6:6.2f} Gev/s (best)  {ev / med / 1e6:6.2f} Gev/s (median)  flagged={bad}", flush=True)
        eng.close()


if __name__ == "__main__":
    main()
