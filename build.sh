#!/usr/bin/env bash
# Builds the C-ABI shared library in-tree: sopro_b200/lib/libsopro_b200.so (sm_90a only).
# The translation units compile in parallel (objects and per-unit logs under sopro_b200/lib/obj), then link.
set -euo pipefail
cd "$(dirname "$0")"
mkdir -p sopro_b200/lib/obj
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH=(-gencode arch=compute_90a,code=sm_90a)
FLAGS=("${ARCH[@]}" -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr)
UNITS=(ar_engine mimi_engine nar_engine noise_host resample stretch loudness level longform flac align watermark ingest denoise)
OBJS=()
PIDS=()
for u in "${UNITS[@]}"; do
  OBJS+=("sopro_b200/lib/obj/$u.o")
  "$NVCC" "${FLAGS[@]}" -c "sopro_b200/csrc/$u.cu" -o "sopro_b200/lib/obj/$u.o" > "sopro_b200/lib/obj/$u.log" 2>&1 &
  PIDS+=($!)
done
rc=0
for i in "${!PIDS[@]}"; do
  wait "${PIDS[$i]}" || { rc=1; echo "nvcc failed: sopro_b200/csrc/${UNITS[$i]}.cu" >&2; }
done
for u in "${UNITS[@]}"; do cat "sopro_b200/lib/obj/$u.log"; done > sopro_b200/lib/build.log
if [ "$rc" -ne 0 ]; then
  grep -E "error" sopro_b200/lib/build.log >&2 || true
  exit 1
fi
"$NVCC" "${ARCH[@]}" -shared -o sopro_b200/lib/libsopro_b200.so "${OBJS[@]}"
grep -E "error|warning|spill|registers" sopro_b200/lib/build.log | sort | uniq -c | sort -rn | head -40 || true
echo "built sopro_b200/lib/libsopro_b200.so"
