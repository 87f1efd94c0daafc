"""bench.py's output contract: the committed line of the last GPU run carries every key the driver reads, and
the reference arm (the unmodified Python reference from oracle/_ref when installed, else the oracle port, on the
host cores -- runs without a GPU) prints exactly one JSON line."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config"}


def test_committed_bench_line_has_the_contract_keys():
    d = json.load(open(os.path.join(ROOT, "profiles", "h100_bench_n1.json")))
    assert BASE_KEYS | {"roofline", "cpu_baseline", "e2e", "gpu_launches", "clocks", "parity_sample"} <= set(d)
    assert d["metric"] == "simulated_events_per_second" and d["unit"] == "events/s"      # BASELINE.json: "simulated events/sec"
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(d["roofline"]) and d["roofline"]["bound"] == "hbm"
    assert abs(d["roofline"]["frac"] - d["roofline"]["achieved"] / d["roofline"]["peak"]) < 1e-12
    assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"]) and d["cpu_baseline"]["kind"] in ("reference", "port")
    assert d["cpu_baseline"]["cores"] <= d["cpu_baseline"]["core_accounting"]["affinity"]
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"]) and d["e2e"]["d2h_bytes_per_step"] > 0
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(d["clocks"]) and d["gpu_launches"] == d["steps"]
    assert "workload" in d["config"] and d["higher_is_better"] is True and d["scaling"] == "weak"
    assert abs(d["value"] - d["events_timed"] / (d["ms_per_step"] * d["steps"] * 1e-3)) / d["value"] < 1e-9
    # the timed run was checked against the CPU oracle inside the bench: raw rings, summaries, statistics
    ps = d["parity_sample"]
    assert ps["ok"] and ps["ok_all_ranks"] and ps["replicas"] >= 8 and "records" in ps["compared"] and ps["events_checked"] > 1e7


def test_committed_full_horizon_run_covers_the_whole_configuration():
    """BASELINE configs[1] is 65 536 replicas x 1e6 sim-s: one committed run covers all 100 windows, with the same sentinel."""
    d = json.load(open(os.path.join(ROOT, "profiles", "h100_bench_full_horizon.json")))
    assert d["steps"] + d["warmup"] == 100 and d["config"]["window_s"] * 100 == d["config"]["horizon_s"] == 1e6
    assert d["aggregate"]["events_processed"] > 3.9e12 and d["aggregate"]["replicas"] == 65536 and d["replicas_flagged"] == 0
    assert abs(d["aggregate"]["mean_latency_s"] - 0.5) < 1e-3                 # M/M/1, rho = 0.8: W = 1 / (mu - lambda)
    ps = d["parity_sample"]
    assert ps["ok"] and ps["windows"] == 100 and ps["sim_seconds_each"] == 1e6 and ps["events_checked"] > 4e8


def test_reference_arm_prints_one_json_line_without_a_gpu():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                         capture_output=True, text=True, timeout=300, env=dict(os.environ, HS_BENCH_REF_BUDGET_S="1.0"))
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert out.returncode == 0 and len(lines) == 1, out.stderr[-500:]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and BASE_KEYS <= set(d) and d["value"] > 0
    have_ref = os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "happysimulator"))
    assert d["cpu_baseline"]["kind"] == ("reference" if have_ref else "port") and d["cpu_baseline"]["value"] == d["value"]
    assert d["cpu_baseline"]["cores"] == len(os.sched_getaffinity(0)) or d["cpu_baseline"]["core_accounting"]["cgroup_quota_cpus"]
    assert d["cpu_baseline_port"]["kind"] == "port" and d["cpu_baseline_port"]["per_core"] > 1e6
    if have_ref:
        assert 2e4 < d["cpu_baseline"]["per_core"] < 2e6        # CPython: ~1.5e5 events/s per core
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def _bench_module():
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _synthetic_outputs(n, rng):
    import numpy as np
    from happysim_b200 import _abi as A
    out = {"summaries": np.zeros(n, A.SUMMARY_DTYPE), "entity_stats": np.zeros((n, 3), A.STATS_DTYPE),
           "records": np.zeros((n, 64), A.RECORD_DTYPE), "sink_samples": None, "service_samples": rng.random((n, 8)),
           "histograms": rng.integers(0, 1000, (n, 64)).astype(np.uint32)}
    for k in ("summaries", "entity_stats", "records"):
        for f in out[k].dtype.names:
            v = out[k][f]
            v[...] = rng.integers(-2**62, 2**63 - 1, v.shape, dtype=np.int64).astype(v.dtype) if v.dtype.kind in "iu" \
                else rng.random(v.shape)
    return out


def test_dump_outputs_names_size_and_exactness(tmp_path, monkeypatch):
    """--dump-outputs: the file names depend only on which outputs exist (64-bit integers are always split), every
    output stays within its byte budget (sampled replicas listed), and the values come back exactly."""
    import numpy as np
    b = _bench_module()
    monkeypatch.setattr(b, "DUMP_KEY_BYTES", 200_000)
    n = 3000
    small = _synthetic_outputs(n, np.random.default_rng(1))
    small["summaries"]["order_hash"] = 5                      # no value near 2^53: still split
    big = _synthetic_outputs(n, np.random.default_rng(2))
    total = b.dump_outputs(small, n, str(tmp_path / "a"))
    b.dump_outputs(big, n, str(tmp_path / "b"))
    names = sorted(os.listdir(tmp_path / "a"))
    assert names == sorted(os.listdir(tmp_path / "b"))
    assert "summaries.order_hash_hi.npy" in names and "summaries.order_hash.npy" not in names
    assert not any(f.startswith("sink_samples") for f in names)
    load = lambda d, f: np.load(tmp_path / d / f"{f}.npy")     # noqa: E731
    assert all(load("a", f[:-4]).dtype == np.float64 for f in names)
    assert total == sum(os.path.getsize(tmp_path / "a" / f) - 128 for f in names)
    for key in ("summaries", "entity_stats", "records", "service_samples", "histograms"):
        size = sum(load("b", f[:-4]).nbytes for f in names if f.split(".")[0] == key and f != key + ".replicas.npy")
        assert size <= 200_000, key
    idx = load("b", "records.replicas").astype(np.int64)
    assert 0 < len(idx) < n and (np.diff(idx) > 0).all()
    hi, lo = load("b", "records.time_ns_hi").astype(np.uint64), load("b", "records.time_ns_lo").astype(np.uint64)
    assert ((hi << np.uint64(32)) | lo).view(np.int64).tolist() == big["records"]["time_ns"][idx].tolist()
    assert load("b", "records.sort_index").tolist() == big["records"]["sort_index"][idx].tolist()
    assert load("b", "entity_stats.f2").tolist() == big["entity_stats"]["f2"][load("b", "entity_stats.replicas").astype(int)].tolist()
