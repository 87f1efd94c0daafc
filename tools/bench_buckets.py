"""Cost of the time buckets (hs_set_buckets) and of their percentiles (hs_set_bucket_percentiles):
python tools/bench_buckets.py  -> one JSON line.

  configs1  65 536 M/M/1 replicas (Source.poisson(8) -> Server(Exponential(0.1)) -> Sink), summary mode, lane engine,
            200 sim-s
  configs2  16 384 replicas of Source(512/s) -> LoadBalancer(RoundRobin) -> 64 x Server -> Sink, thread engine, 10 sim-s
Each without buckets, with 100 and with 1 000 buckets (width = horizon / (n - 1)), and with both bucket counts plus
percentiles (a sample capacity of 64 for configs1, 256 for configs2: well above the largest bucket), the five
alternating within every round, 5 rounds.  Device time of the kernel alone (CUDA events; the cell reductions are
separate calls), best and median, events/s; the card's name and power limit are reported with them."""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import happysim_b200 as hs  # noqa: E402
from happysim_b200 import engine  # noqa: E402


def bench(eng, model, n, end_s, cap, rounds=5):
    eng.upload(model)
    variants = {"off": (0, 0), "buckets_100": (100, 0), "buckets_1000": (1000, 0), "pct_100": (100, cap),
                "pct_1000": (1000, cap)}
    ms = {k: [] for k in variants}
    events, flags = {}, {}
    for _ in range(rounds + 1):                      # the first round warms every variant up and is not counted
        for k, (nb, cap) in variants.items():
            eng.set_buckets(end_s / (nb - 1) if nb else 0.0, nb)
            eng.set_bucket_percentiles(cap)
            eng.run(engine.make_params(seed=1234, end_ns=int(end_s * 1e9), n_replicas=n, flags=0))
            eng.sync()
            ms[k].append(eng.last_run_ms())
            s = eng.read_outputs()["summaries"]
            events[k] = int(s["events_processed"].sum())
            flags[k] = eng.last_launch()
            assert not (s["status"] & hs._abi.HS_ST_BUCKET_OVERFLOW).any(), k
    eng.set_bucket_percentiles(0)
    eng.set_buckets(0.0, 0)
    assert len(set(events.values())) == 1, events
    res = {}
    for k in variants:
        t = ms[k][1:]
        res[k] = dict(best_ms=min(t), median_ms=statistics.median(t), events_per_s=events[k] / (min(t) / 1e3),
                      kernel=flags[k]["kernel"], flags=flags[k]["flags"])
    for k in ("buckets_100", "buckets_1000", "pct_100", "pct_1000"):
        res[k]["overhead_median"] = res[k]["median_ms"] / res["off"]["median_ms"] - 1.0
    for nb in (100, 1000):        # what the percentiles add to the same buckets
        res[f"pct_{nb}"]["over_buckets_median"] = res[f"pct_{nb}"]["median_ms"] / res[f"buckets_{nb}"]["median_ms"] - 1.0
    return res


def main():
    eng = engine.Engine(0)
    res = {"configs1": bench(eng, hs.mm1(8.0, 0.1), 65536, 200.0, 64),
           "configs2": bench(eng, hs.lb_round_robin(64, 512.0), 16384, 10.0, 256)}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
