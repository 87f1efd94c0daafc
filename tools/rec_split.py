"""Where the record-mode step's time goes: bench.py's headline (config 1, record mode: 65 536 M/M/1 replicas, record /
sample / service caps 1024 / 128 / 128, consecutive resumed 1e4-s windows) on variants of the lane kernel built from
patched copies of the engine sources:
    V0  the sources as they are
    V1  every recorder global store dead behind a runtime predicate that is always false (the record-line, sample-group
        and service-chunk flushes, the entry-by-entry paths, the epilogue); the values they would store are still
        loaded, so staging STS, ballots, __fns, shuffles and the flush LDS remain: the recorder's instructions without
        its HBM writes
    V2  V1 with the recorder pointers null at run time (same predicate): no staging, no flush loops, the record
        kernel's event loop and 8-slot draw buffers alone -- close to summary mode, the check that the split adds up
    sum summary mode (V0 library, no recorder caps), for comparison with V2
V0 - V1 is the time the event loop loses to the stores, V1 - V2 the recorder's own instruction cost.

    python tools/rec_split.py [--csrc DIR] [--libs DIR] [--reps 3] [--steps 5] [--warmup 3] [--build-only]

--csrc patches another copy of happy-simulator_b200/csrc (an A/B against an earlier commit).  The variant libraries are
built into --libs (default: a temporary directory) and reused from there when present.  Each (variant, repetition)
runs in a process of its own, variants alternating within a repetition; a step is the kernel time of one window
(CUDA events around the launch).  The tree is left as it was."""
import argparse
import os
import re
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

LANE = "hs_lane_engine.cuh"
DEAD = "(P.n_replicas == 0xffffffffu)"       # never true at run time, unknown to the compiler
# a recorder store made dead: the stored value is still computed (the asm consumes it), the store is not issued
KEEP = ("#define HS_SPLIT_KEEP4(V) do { const uint4 k4_ = (V); asm volatile(\"\" :: \"r\"(k4_.x), \"r\"(k4_.y), "
        "\"r\"(k4_.z), \"r\"(k4_.w)); } while (0)\n"
        "#define HS_SPLIT_KEEPD(V) do { const double kd_ = (V); asm volatile(\"\" :: \"d\"(kd_)); } while (0)\n"
        "#define HS_SPLIT_STCS(PTR, V) do { const uint4 v4_ = (V); HS_SPLIT_KEEP4(v4_); if " + DEAD +
        " __stcs((PTR), v4_); } while (0)\n")


def _sub(src, pat, rep, count, flags=0):
    out, n = re.subn(pat, rep, src, flags=flags)
    if n != count:
        raise SystemExit(f"rec_split: pattern {pat!r} matched {n} times, expected {count}: the sources changed")
    return out


def patch_v1(src):
    n = src.count("__stcs(")
    src = src.replace("__stcs(", "HS_SPLIT_STCS(")
    src = src.replace("#define HS_LANE_THREADS 64", KEEP + "#define HS_LANE_THREADS 64", 1)
    if n < 3:
        raise SystemExit("rec_split: fewer than three recorder flush stores found")
    # stores through plain assignment: Sink samples and service times entry by entry, and in the epilogue
    src = _sub(src, r"\*\(uint4 \*\)\((smp \+ [^;]*?)\) = ([^;]*);", r"{ HS_SPLIT_KEEP4(\2); if " + DEAD + r" *(uint4 *)(\1) = \2; }", 4)
    src = _sub(src, r"(svc_out\[[^\]]+\]) = ([^;]*);", r"{ HS_SPLIT_KEEPD(\2); if " + DEAD + r" \1 = \2; }", 3)
    return src


def patch_v2(src):
    src = patch_v1(src)
    for p in ("O.records", "O.samples", "O.service"):
        src = _sub(src, r"\(FLAGS & HS_LF_REC\) && " + re.escape(p) + r" \?", f"(FLAGS & HS_LF_REC) && {p} && {DEAD} ?", 1)
    return src


VARIANTS = {"V0": lambda s: s, "V1": patch_v1, "V2": patch_v2}


def build(csrc, libs, name):
    from happysim_b200.build import NVCC_FLAGS, _nvcc
    lib = os.path.join(libs, f"{name}.so")
    if os.path.exists(lib):
        return lib
    # the sources include ../../include/hs_b200.h: keep that layout in the copy
    top = os.path.join(libs, name)
    shutil.rmtree(top, ignore_errors=True)
    d = os.path.join(top, "pkg", "csrc")
    shutil.copytree(csrc, d)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(top, "include"))
    with open(os.path.join(d, LANE)) as f:
        src = f.read()
    with open(os.path.join(d, LANE), "w") as f:
        f.write(VARIANTS[name](src))
    r = subprocess.run([_nvcc(), *NVCC_FLAGS, "-Xptxas", "-v", "-o", lib + ".tmp",
                        os.path.join(d, "hs_engine.cu")], cwd=d, capture_output=True, text=True)
    if r.returncode:
        raise SystemExit(f"rec_split: {name} does not compile:\n{r.stderr[-4000:]}")
    lines = r.stderr.splitlines()
    with open(os.path.join(libs, f"{name}.ptxas.txt"), "w") as f:
        for i, line in enumerate(lines):   # the record-mode lane kernels: <2>, <3>, <10>, <11>
            if re.search(r"_Z\d+hs_lane_kernelILi(2|3|10|11)E", line) and "Compiling entry" in line:
                f.write("\n".join(lines[i:i + 4]) + "\n")
    os.replace(lib + ".tmp", lib)
    return lib


def worker(mode, steps, warmup):
    """One process, one library (HS_B200_LIB): warmup + steps windows of bench.py's config 1; prints ms per step."""
    import happysim_b200 as hs
    from happysim_b200 import engine
    from bench import RATE, MEAN
    n, win = 65536, int(1.0e4 * 1e9)
    caps = dict(record_cap=1024, sample_cap=128, service_cap=128) if mode == "record" else {}
    eng = engine.Engine(0)
    eng.upload(hs.mm1(RATE, MEAN))
    ms = []
    for k in range(warmup + steps):
        eng.run(engine.make_params(seed=1234, end_ns=int(1.0e6 * 1e9), window_end_ns=(k + 1) * win, n_replicas=n,
                                   resume=int(k > 0), **caps))
        eng.sync()
        if k >= warmup:
            ms.append(eng.last_run_ms())
    s = eng.read_outputs()["summaries"]
    print(f"RESULT {sum(ms) / len(ms):.2f} flagged {int((s['status'] != 0).sum())} events {int(s['events_processed'].sum())}")
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--csrc", default=os.path.join(ROOT, "happy-simulator_b200", "csrc"))
    ap.add_argument("--libs", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--worker", choices=["record", "summary"], default=None)
    a = ap.parse_args()
    if a.worker:
        worker(a.worker, a.steps, a.warmup)
        return
    tmp = None
    libs = a.libs
    if libs is None:
        tmp = tempfile.TemporaryDirectory()
        libs = tmp.name
    libs = os.path.abspath(libs)
    os.makedirs(libs, exist_ok=True)
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        lib = dict(zip(VARIANTS, ex.map(lambda v: build(a.csrc, libs, v), VARIANTS)))
    for v in VARIANTS:
        with open(os.path.join(libs, f"{v}.ptxas.txt")) as f:
            print(f"# {v} ptxas: " + " | ".join(l.strip() for l in f if "registers" in l or "stack" in l), flush=True)
    if a.build_only:
        return
    from bench import ClockSampler
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# card: {card}; kernel sources: {os.path.relpath(a.csrc, ROOT)}; {a.steps} timed windows after "
          f"{a.warmup}, kernel time per window (CUDA events), one process per run", flush=True)
    runs = [(v, "record") for v in VARIANTS] + [("sum", "summary")]
    res = {v: [] for v, _ in runs}
    clk = ClockSampler(0)
    clk.start()
    for rep in range(a.reps):
        for v, mode in runs:
            env = dict(os.environ, HS_B200_LIB=lib["V0" if v == "sum" else v])
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", mode, "--steps", str(a.steps),
                                  "--warmup", str(a.warmup)], env=env, capture_output=True, text=True, cwd=ROOT)
            m = re.search(r"RESULT (\S+) flagged (\d+) events (\d+)", out.stdout)
            if not m:
                raise SystemExit(f"rec_split: {v} failed:\n{out.stdout[-2000:]}\n{out.stderr[-4000:]}")
            res[v].append(float(m.group(1)))
            print(f"{v:3s} rep {rep + 1} {float(m.group(1)):8.2f} ms/step  flagged {m.group(2)}  events {m.group(3)}",
                  flush=True)
    print(f"# clocks while running: {clk.stop()}")
    med = {v: sorted(x)[len(x) // 2] for v, x in res.items()}
    for v, x in res.items():
        print(f"# {v:3s} median {med[v]:8.2f} ms/step (spread {min(x):.2f}-{max(x):.2f})")
    print(f"# V0 - V1 (loop time lost to the recorder's global stores) {med['V0'] - med['V1']:8.2f} ms/step")
    print(f"# V1 - V2 (the recorder's own instructions)                {med['V1'] - med['V2']:8.2f} ms/step")
    print(f"# V2 - summary                                             {med['V2'] - med['sum']:8.2f} ms/step")
    if tmp:
        tmp.cleanup()


if __name__ == "__main__":
    main()
