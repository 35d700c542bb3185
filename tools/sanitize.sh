#!/bin/bash
# compute-sanitizer passes over the small encode + decode (tools/sanitize_small.py); logs -> gpurun_out/
# Run on a machine with a GPU and compute-sanitizer:  bash tools/sanitize.sh
mkdir -p gpurun_out
for tool in memcheck racecheck synccheck; do
  timeout 240 compute-sanitizer --tool $tool --print-limit 20 python tools/sanitize_small.py > gpurun_out/sanitize_$tool.log 2>&1
  echo "$tool exit=$?" >> gpurun_out/sanitize_$tool.log
  tail -4 gpurun_out/sanitize_$tool.log
done
