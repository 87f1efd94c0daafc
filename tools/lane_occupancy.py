"""Build and run tools/lane_occupancy.cu on cuda:0: registers, shared and local memory and blocks per SM of the lane
kernel's record-mode instantiations, as the engine sources in the tree compile them:
    python tools/lane_occupancy.py [--csrc DIR]
--csrc compiles the kernel from another copy of happy-simulator_b200/csrc (an A/B against an earlier commit).  The
binary is compiled into a temporary directory, so the tree is left as it was."""
import argparse
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
from happysim_b200.build import _nvcc                    # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--csrc", default=os.path.join(ROOT, "happy-simulator_b200", "csrc"))
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "lane_occupancy")
        subprocess.check_call([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                               "-I", os.path.join(ROOT, "include"), "-I", a.csrc, "-o", exe,
                               os.path.join(ROOT, "tools", "lane_occupancy.cu")])
        card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit",
                               "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
        print(f"# card: {card}; kernel sources: {os.path.relpath(a.csrc, ROOT)}", flush=True)
        sys.exit(subprocess.call([exe]))


if __name__ == "__main__":
    main()
