"""Build the CUDA engine in-tree: happy-simulator_b200/libhs_b200.so (sm_90a, H100)."""
from __future__ import annotations

import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.environ.get("HS_B200_LIB") or os.path.join(PKG_DIR, "libhs_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def sources() -> list[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC))


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    inc = os.path.join(os.path.dirname(PKG_DIR), "include", "hs_b200.h")
    return any(os.path.getmtime(s) > t for s in sources() + [inc])


def build_cuda(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    cmd = [_nvcc(), *NVCC_FLAGS, *os.environ.get("HS_B200_DEFS", "").split(), "-o", LIB_PATH,
           os.path.join(CSRC, "hs_engine.cu")]
    if verbose:
        cmd[1:1] = ["-Xptxas", "-v"]
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB_PATH


if __name__ == "__main__":
    print(build_cuda(force=True, verbose=True))
