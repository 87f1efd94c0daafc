"""Build and run the recorder-store microbenchmark (tools/rec_store_bench.cu) on cuda:0, with the card's name,
power limit and the clocks / throttle reasons sampled while it runs:
    python tools/rec_store_bench.py [--events 3.96e10] [--reps 5] [--seed 1]
The binary is compiled into a temporary directory, so the tree is left as it was."""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
from bench import ClockSampler                           # noqa: E402
from happysim_b200.build import _nvcc                    # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "rec_store_bench")
        subprocess.check_call([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                               os.path.join(ROOT, "tools", "rec_store_bench.cu")])
        card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
        print(f"# card: {card}", flush=True)
        clk = ClockSampler(0)
        clk.start()
        rc = subprocess.call([exe, *sys.argv[1:]])
        print(f"# clocks while running: {clk.stop()}", flush=True)
    sys.exit(rc)


if __name__ == "__main__":
    main()
