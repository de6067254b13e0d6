#!/bin/bash
# Nsight Compute on an H100: launch list + `--set full` captures of one diffusion step for BASELINE configs 1-3, reduced to
# raw-page CSVs (the .ncu-rep files are ~40 MB each; only config 1's is kept).
#   bash tools/ncu_capture.sh <tag> [out_dir]
set -u
TAG=${1:-r02}
OUT=${2:-ncu_out}
mkdir -p $OUT
export LDM_GRAPH=0      # stream launches (one graph node per kernel would be profiled just the same; this keeps the launch order explicit)
M="gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed,dram__bytes_read.sum,dram__bytes_write.sum,gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed,lts__t_sector_hit_rate.pct,lts__throughput.avg.pct_of_peak_sustained_elapsed,sm__warps_active.avg.pct_of_peak_sustained_active,launch__registers_per_thread,sm__throughput.avg.pct_of_peak_sustained_elapsed,l1tex__throughput.avg.pct_of_peak_sustained_elapsed"
# launch list of the third step (config 1: 1 fill kernel + 2 x 23 launches skipped)
ncu --metrics gpu__time_duration.sum --clock-control none -s 47 -c 23 --csv --log-file $OUT/${TAG}_launches_step.csv python tools/profile_step.py --steps 3 > $OUT/${TAG}_ncu_list.log 2>&1
for CFG in 1 2 3; do
  SKIP=23; [ $CFG = 1 ] && SKIP=24
  ncu --set full --clock-control none --import-source on -s $SKIP -c 23 -f -o $OUT/prof_${TAG}_cfg$CFG python tools/profile_step.py --config $CFG --steps 2 > $OUT/${TAG}_ncu_full_cfg$CFG.log 2>&1
  ncu -i $OUT/prof_${TAG}_cfg$CFG.ncu-rep --page raw --csv --metrics $M > $OUT/${TAG}_cfg${CFG}_raw.csv 2>/dev/null
  [ $CFG != 1 ] && rm -f $OUT/prof_${TAG}_cfg$CFG.ncu-rep
  tail -1 $OUT/${TAG}_ncu_full_cfg$CFG.log
done
ls -la $OUT
