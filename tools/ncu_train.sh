#!/bin/bash
# ncu pass over the kernels of one training step (bench config 3 or 5): duration, DRAM bytes, tensor / issue / L1 / L2
# utilisation per kernel -> $OUT/r2_train_kernels_cfg$1.csv (summarised by tools/ncu_summary.py).
# usage (on an H100 machine with Nsight Compute): bash tools/ncu_train.sh 5
set -u
cd "$(dirname "$0")/.."
OUT=${OUT:-tool_out}          # reports go here (git-ignored)
mkdir -p "$OUT"
CFG=${1:-5}
M=gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,dram__throughput.avg.pct_of_peak_sustained_elapsed
M=$M,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active,sm__issue_active.avg.pct_of_peak_sustained_active
M=$M,l1tex__throughput.avg.pct_of_peak_sustained_elapsed,lts__throughput.avg.pct_of_peak_sustained_elapsed
M=$M,sm__warps_active.avg.pct_of_peak_sustained_active,launch__registers_per_thread,smsp__inst_executed.sum
ncu --metrics $M --clock-control none -k regex:"field_kernel|field_mlp_bwd|deform_bwd|deform_dw|hash_bwd|hash_expand|table_step|composite|losses_|march_occ|vis_compact|depth_" --launch-skip 120 -c 40 --csv --log-file $OUT/r2_train_kernels_cfg$CFG.csv \
    python tools/train_profile.py $CFG > $OUT/r2_train_ncu_cfg$CFG.log 2>&1
python tools/ncu_summary.py $OUT/r2_train_kernels_cfg$CFG.csv
