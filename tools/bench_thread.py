"""Thread-engine A/B on configs[2]/[3]: python tools/bench_thread.py  (HS_B200_LIB selects the library variant)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import happysim_b200 as hs
from happysim_b200 import engine

def run(name, model, n, end_s, **kw):
    eng = engine.Engine(0)
    eng.upload(model)
    best = None
    for _ in range(3):
        eng.run(engine.make_params(seed=1234, end_ns=int(end_s * 1e9), n_replicas=n, flags=0, engine=3, **kw))
        eng.sync()
        ms = eng.last_run_ms(); best = ms if best is None else min(best, ms)
    out = eng.read_outputs()
    ev = int(out["summaries"]["events_processed"].sum())
    print(f"{os.path.basename(os.environ.get('HS_B200_LIB', 'default')):14s} {name:30s} n={n:6d} ev={ev:.3e} {best:9.2f} ms {ev / best / 1e6:8.3f} Gev/s flagged={int((out['summaries']['status'] != 0).sum())}", flush=True)
    eng.close()

lb = hs.lb_round_robin(64, 512.0)
for n in (16384, 65536):
    run("configs[2] lb-rr64", lb, n, 10.0)
tab = hs.consistent_hash_table([f"S{i}" for i in range(1024)], 100, 10000)
ch = hs.lb_key_table(tab, 1024, rate=8192.0)
for n in (1024, 4096):
    run("configs[3] chash1024", ch, n, 2.0)
run("mm1 on thread engine", hs.mm1(), 65536, 50.0)
