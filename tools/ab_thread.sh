#!/bin/bash
# A/B of thread-engine library variants on one GPU box: tools/ab_thread.sh <variant> ...   (libhs_<variant>.so, built with HS_B200_DEFS)
cd "$(dirname "$0")/.."
OUT="${HS_OUT_DIR:-${TMPDIR:-/tmp}/hs_gpu_out}"; mkdir -p "$OUT"
for v in "$@"; do
  HS_B200_LIB=$PWD/happy-simulator_b200/libhs_$v.so timeout 300 python tools/bench_thread.py
done 2>&1 | tee "$OUT"/ab_thread.txt
