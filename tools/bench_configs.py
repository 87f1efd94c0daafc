"""Device-time throughput of the BASELINE configs that run on the warp engine (context numbers for
DESIGN.md; the driver's bench is bench.py)."""
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
        eng.run(engine.make_params(seed=1234, end_ns=int(end_s * 1e9), n_replicas=n, flags=0, **kw))
        eng.sync()
        ms = eng.last_run_ms(); best = ms if best is None else min(best, ms)
    out = eng.read_outputs()
    ev = int(out["summaries"]["events_processed"].sum())
    bad = int((out["summaries"]["status"] != 0).sum())
    print(f"{name:34s} replicas={n:6d} sim={end_s:7.1f}s events={ev:.3e} {best:9.2f} ms {ev / best / 1e6:8.3f} Gev/s flagged={bad}", flush=True)
    eng.close()

if __name__ == "__main__":
    run("configs[1] mm1 lane engine", hs.mm1(), 65536, 1000.0)
    run("configs[1] mm1 on the WARP engine", hs.mm1(), 65536, 50.0, engine=1)
    run("configs[1] mm1 on the THREAD engine", hs.mm1(), 65536, 50.0, engine=3)
    for n in (4096, 16384, 65536, 262144):
        run("configs[2] lb-rr64 thread", hs.lb_round_robin(64, 512.0), n, 10.0, engine=3)
    run("configs[2] lb-rr 64 servers, warp", hs.lb_round_robin(64, 512.0), 16384, 10.0, engine=1)
    tab = hs.consistent_hash_table([f"S{i}" for i in range(1024)], 100, 10000)
    for n in (1024, 4096):
        run("configs[3] chash1024 thread", hs.lb_key_table(tab, 1024, rate=8192.0), n, 2.0, engine=3)
    run("configs[3] chash 1024 nodes, warp", hs.lb_key_table(tab, 1024, rate=8192.0), 1024, 2.0, engine=1)
    K = 10000
    b = hs.ModelBuilder()
    src = b.source(rate=512.0, key_population=K)
    servers = [b.server(f"S{i}", mean_service_s=0.1) for i in range(64)]
    hll = b.sketch_hll("uniques", precision=12, table=hs.hll_table(12, 1, K))
    cms = b.sketch_cms("freq", width=272, depth=5, table=hs.cms_table(272, 5, 2, K))
    lb = b.load_balancer(backends=servers)
    b.set_target(src, lb)
    for k, sv in enumerate(servers):
        b.set_target(sv, hll if k % 2 else cms)
    run("lb-rr64 -> HLL(p=12) | CMS(272x5) sinks", b.build(), 16384, 10.0, engine=3)
    m = hs.mmc_sweep()
    run("configs[4] M/M/c sweep 256 cells", m, 32768, 100.0, replicas_per_cell=128, queue_ring=4096)
