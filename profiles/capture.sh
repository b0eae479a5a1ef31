#!/usr/bin/env bash
# Nsight Compute captures of a bench step, on a machine with an H100 and ncu. Run from the repo root:
#   bash profiles/capture.sh <tag>
# Writes under profile_out/<tag>/; afterwards:
#   python profiles/ncu_summary.py profile_out/<tag>/prof_str_scan.ncu-rep profile_out/<tag>/k_str_scan_ncu_details.txt
#   python profiles/ncu_source_hotspots.py profile_out/<tag>/prof_str_scan.ncu-rep > profile_out/<tag>/k_str_scan_source_hotspots.txt
# (same for prof_int_scan). Numbers printed by bench.py under ncu are never bench values.
set -u
tag="${1:-rXX}"
out="profile_out/${tag}"
mkdir -p "$out"
# 1. launch list of one bench step (cold-cache, serialised times: only the kernels' SHARE of the step is comparable)
ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file "$out/launches_url_like.csv" \
    python bench.py --steps 2 --warmup 3 --no-cpu-baseline > "$out/bench_under_ncu.log" 2>&1
# 2. full capture of the dominant kernel (LIKE scan), three launches after the warm-up ones
ncu --set full --clock-control none --import-source on -k regex:k_str_scan -s 4 -c 3 -o "$out/prof_str_scan" -f \
    python bench.py --steps 2 --warmup 3 --no-cpu-baseline > "$out/ncu_str.log" 2>&1
# 3. full capture of the integer scan on the narrow column (W = 17) and on l_shipdate (W = 12)
ncu --set full --clock-control none --import-source on -k regex:k_int_scan -s 6 -c 3 -o "$out/prof_int_scan" -f \
    python bench.py --workload int_filter --steps 2 --warmup 3 > "$out/ncu_int.log" 2>&1
# 4. the plain bench lines of the same library (these ARE bench values)
python bench.py --steps 20 --warmup 5 > "$out/bench_url_like.json" 2> "$out/bench_url_like.err"
python bench.py --workload int_filter --steps 20 --warmup 5 > "$out/bench_int_filter.json" 2> "$out/bench_int_filter.err"
python bench.py --workload shipdate --steps 10 --warmup 3 > "$out/bench_shipdate.json" 2> "$out/bench_shipdate.err"
python bench.py --workload clickbench_sweep --steps 12 --warmup 3 > "$out/bench_clickbench_sweep.json" 2> "$out/bench_clickbench_sweep.err"
ls -la "$out"
