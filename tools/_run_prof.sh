#!/bin/bash
# Profiler captures and sanitizer runs of the hot kernels: tools/_run_prof.sh OUT_DIR (run from any directory).
O="${1:?usage: tools/_run_prof.sh OUT_DIR}"
mkdir -p "$O"
O="$(cd "$O" && pwd)"
cd "$(dirname "$0")/.."
# 1. the LK kernel, full capture (4 units x 2000 features, default work-item size)
LK_SPANS=2 timeout 900 ncu --set full --import-source on --clock-control none -k regex:k_lk_ring -s 3 -c 1 -f -o "$O/lk_r02" python tools/lk_ab.py 8 2000 1 > "$O/ncu_lk_r02.out" 2>&1
tail -1 "$O/ncu_lk_r02.out"
# 2. launch list of the bench command (cold-cache serialised times: compare shares)
VO_OPT_SM_PARTITION=0 timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 1500 --csv --log-file "$O/launches_bench_r02.csv" python bench.py --steps 2 --warmup 3 --cpu-seconds 0.3 --sweep 0 > "$O/launches_bench_r02.out" 2>&1
tail -c 300 "$O/launches_bench_r02.out"
# 3. launch list of the sequence mode
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file "$O/launches_seq_r02.csv" python tools/run_seq.py 6 > "$O/launches_seq_r02.out" 2>&1
# 4. sanitizers on the new kernels (small cases)
timeout 900 compute-sanitizer --tool memcheck python -m pytest tests/test_gpu_lk.py -q -x -k "empty or truncation or random" > "$O/memcheck_lk_r02.txt" 2>&1; tail -3 "$O/memcheck_lk_r02.txt"
VO_LK_SPAN=1 timeout 900 compute-sanitizer --tool racecheck python -m pytest tests/test_gpu_lk.py -q -x -k "empty or truncation" > "$O/racecheck_lk_r02.txt" 2>&1; tail -3 "$O/racecheck_lk_r02.txt"
timeout 900 compute-sanitizer --tool memcheck python -m pytest tests/test_gpu_stages.py -q -x -k "mono" > "$O/memcheck_ess_r02.txt" 2>&1; tail -3 "$O/memcheck_ess_r02.txt"
