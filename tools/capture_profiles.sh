#!/usr/bin/env bash
# Bench lines, Nsight Compute captures, in-kernel stage timing and the host pipeline profile of one build, written to
# ${PROFILE_DIR:-prof_out}/<name> (needs an H100 and Nsight Compute):
#   bash tools/capture_profiles.sh r03
set -u
R=${1:-rXX}
O=${PROFILE_DIR:-prof_out}/$R
mkdir -p "$O"
timeout 600 python bench.py --steps 5 --warmup 3 > "$O/bench.json" 2> "$O/bench.err"
timeout 300 python bench.py --impl reference --steps 2 --warmup 1 > "$O/bench_reference.json" 2>/dev/null
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file "$O/launches.csv" \
  python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-extras > /dev/null 2>&1
timeout 300 ncu --set full --clock-control none --import-source on -k regex:ar_persistent -s 1 -c 1 -o "$O/ar_full" \
  python tools/prof_ar.py 64 bf16 401 > /dev/null 2>&1
# the NAR refiner's tensor-core GEMMs (exact six-product split): GLU / FFN1 / FFN2 of the first block at 16 x 401 frames
timeout 300 ncu --set full --clock-control none -k regex:igemm_tc -c 3 -o "$O/nar_tc_full" \
  python tools/prof_nar.py 16 401 > /dev/null 2>&1
timeout 300 ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none --csv \
  --log-file "$O/mimi_dram.csv" python tools/prof_mimi.py 400 bf16_tc 25 1 > /dev/null 2>&1
timeout 200 python tools/gpu_stage_timing.py 64:bf16:0 1:bf16:0 > "$O/stage_timing.log" 2>&1
timeout 300 python tools/prof_e2e.py > "$O/prof_e2e.log" 2>&1
ls -la "$O"
