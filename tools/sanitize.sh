#!/bin/bash
# compute-sanitizer passes over the library's kernels (GPU box only; SURVEY.md section 5 asks for
# them).  Not part of the timed or tested path -- run by hand on a GPU machine:
#     bash tools/sanitize.sh
# memcheck / racecheck slow kernels down by 10-100x: the bounded waits of the wgmma kernels trap
# after ~3e9 cycles, so the small configurations of tests/gpu_checks.py are used, one process per
# check (a trap poisons the CUDA context).  SAN_MEMCHECK / SAN_RACECHECK override the check lists,
# SAN_TIMEOUT the per-check limit in seconds.
set -u
OUT=gpurun_out/sanitizer
mkdir -p "$OUT"
MEM=${SAN_MEMCHECK:-"warp_hrflow_s4 warp_lrflow_bd4 pool_upsample module_ops downsample_bd conv_tc_halo_64 conv_tc_tap_convT epilogues_tc step_golden_g1"}
RACE=${SAN_RACECHECK:-"warp_lrflow_bd4 conv_tc_halo_64 conv_tc_tap_convT epilogues_tc"}
TMO=${SAN_TIMEOUT:-600}
for tool in memcheck racecheck; do
  if [ $tool = memcheck ]; then LIST=$MEM; else LIST=$RACE; fi
  for c in $LIST; do
    timeout $TMO /usr/local/cuda/bin/compute-sanitizer --tool $tool --error-exitcode 9 \
      python tests/gpu_diag.py --one $c > "$OUT/${tool}_$c.log" 2>&1
    echo "$tool $c rc=$? $(grep 'ERROR SUMMARY' "$OUT/${tool}_$c.log" | tail -1)" | tee -a "$OUT/summary.txt"
  done
done
