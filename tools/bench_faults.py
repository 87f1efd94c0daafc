"""Cost of the node-fault path: python tools/bench_faults.py  -> one JSON line.

  farm     configs[2]-shaped: Source(512/s) -> LoadBalancer(RoundRobin) -> 64 x Server -> Sink, 16 384 replicas,
           10 s; once without faults and once with 8 backends crashed at 3-4.75 s and restarted at 6-7.75 s
  mm1      Source -> Server -> Sink with one crash (3 s) and restart (6 s) of the server, thread engine, 65 536 replicas
Device time of the kernel (CUDA events), best of 3, events/s; the card's name and power limit are reported with them."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import happysim_b200 as hs  # noqa: E402
from happysim_b200 import _abi as A, engine  # noqa: E402


def with_faults(m, targets, crash_s, restart_s):
    rows, k = [], len(m.ids_of(A.HS_ENT_SOURCE))
    for j, t in enumerate(targets):
        for at, crash in ((crash_s + 0.25 * j, 1), (restart_s + 0.25 * j, 0)):
            rows.append((A.HS_ENT_FAULT, t, 0, crash, 0, k, int(at * 1e9), 0.0, 0.0)); k += 1
    m.entities = np.array(list(m.entities.tolist()) + rows, dtype=A.ENTITY_DTYPE)
    m.names = list(m.names) + [f"fault{i}" for i in range(len(rows))]
    return m


def run(eng, model, n, end_s):
    eng.upload(model)
    best, ev = None, 0
    for _ in range(3):
        eng.run(engine.make_params(seed=1234, end_ns=int(end_s * 1e9), n_replicas=n, flags=0, engine=3))
        eng.sync()
        ms = eng.last_run_ms(); best = ms if best is None else min(best, ms)
    out = eng.read_outputs()
    ev = int(out["summaries"]["events_processed"].sum())
    return dict(events_per_s=ev / (best / 1e3), device_ms=best, events=ev, flags=eng.last_launch()["flags"],
                replicas_flagged=int((out["summaries"]["status"] != 0).sum()))


def main():
    eng = engine.Engine(0)
    farm = hs.lb_round_robin(64, 512.0)
    servers = farm.ids_of(A.HS_ENT_SERVER)
    res = {"farm_no_faults": run(eng, farm, 16384, 10.0)}
    res["farm_8_crash_restart"] = run(eng, with_faults(hs.lb_round_robin(64, 512.0), servers[::8], 3.0, 6.0), 16384, 10.0)
    mm1 = hs.mm1()
    res["mm1_crash_restart"] = run(eng, with_faults(mm1, [mm1.ids_of(A.HS_ENT_SERVER)[0]], 3.0, 6.0), 65536, 10.0)
    res["mm1_no_faults_thread"] = run(eng, hs.mm1(), 65536, 10.0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
