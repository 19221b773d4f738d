#!/bin/bash
# Per-launch device times of ONE bench step (ncu, cold-cache, serialised: compare SHARES).
# usage (under gpurun): bash tools/launch_list.sh <tag> <launches_per_step> [extra bench args]
TAG=${1:-r01}; NPER=${2:-97}; shift; shift
mkdir -p gpurun_out
SKIP=$((NPER * 3))
ncu --metrics gpu__time_duration.sum --clock-control none \
    -k regex:"conv_tc_kernel|conv3x3_tc_kernel|conv_simt_kernel|dcn_tc_kernel|head_tc_kernel|stem_kernel|maxpool_kernel|dwdeconv_add_kernel|dwdeconv_add_fast_kernel|upsample_add_kernel|dwconv_kernel|dwconv_tiled_kernel|stem_tc_kernel|stem_tc_h_kernel|conv_sp_kernel|avgpool_kernel|scale_add_kernel|decode_kernel|sigmoid_kernel" \
    -s ${SKIP} -c ${NPER} --csv --log-file gpurun_out/launches_${TAG}.csv \
    python bench.py --steps 1 --warmup 3 --no-cpu-baseline "$@" > gpurun_out/launches_${TAG}.log 2>&1
python tools/summarize_launches.py gpurun_out/launches_${TAG}.csv > gpurun_out/launches_${TAG}_summary.txt
head -60 gpurun_out/launches_${TAG}_summary.txt
