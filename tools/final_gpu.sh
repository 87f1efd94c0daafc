#!/bin/bash
# round-end evidence on one GPU: smoke, GPU tests, the default bench line, configs[3] on one GPU's share, device
# throughput of the other configs, one ncu --set full capture of the thread engine.  Outputs under $HS_OUT_DIR (default $TMPDIR/hs_gpu_out).
cd "$(dirname "$0")/.."; OUT="${HS_OUT_DIR:-${TMPDIR:-/tmp}/hs_gpu_out}"; mkdir -p "$OUT"
python __graft_entry__.py smoke > "$OUT"/final_smoke.txt 2>&1; tail -1 "$OUT"/final_smoke.txt
timeout 500 python -m pytest tests -m gpu -q > "$OUT"/final_gputest.txt 2>&1; tail -1 "$OUT"/final_gputest.txt
timeout 600 python bench.py > "$OUT"/final_bench_n1.json 2> "$OUT"/final_bench_n1.err; tail -c 600 "$OUT"/final_bench_n1.json
timeout 300 python bench.py --config 3 --no-other-configs > "$OUT"/final_bench_config3_n1.json 2> "$OUT"/final_bench_config3_n1.err; tail -c 400 "$OUT"/final_bench_config3_n1.json
timeout 300 python tools/bench_thread.py > "$OUT"/final_thread.txt 2>&1; cat "$OUT"/final_thread.txt
timeout 300 python tools/bench_configs.py > "$OUT"/final_configs.txt 2>&1; cat "$OUT"/final_configs.txt
timeout 300 ncu --set full --clock-control none --import-source on -k regex:hs_thread_kernel --launch-skip 2 --launch-count 1 -f -o "$OUT"/r02c_thread python tools/ncu_target.py thread 10 16384 > "$OUT"/ncu_thread.log 2>&1; tail -2 "$OUT"/ncu_thread.log
