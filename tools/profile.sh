#!/bin/bash
# Profiling recipe (ONE GPU). Outputs land in out/.
#   1) launch list of one graph-replayed UNet step (device time per launch, no cache flush)
#   2) ncu --set full of the 96x96 320->320 implicit-GEMM conv and of the 9216-token flash attention
set -u
TAG=${1:-r01}
mkdir -p out
STEP="python tools/step_only.py 3"
timeout 500 ncu --metrics gpu__time_duration.sum --clock-control none --cache-control none -c 3000 --csv \
    --log-file out/${TAG}_launches.csv $STEP > out/${TAG}_launches.log 2>&1
# first eager UNet step: launch #57 is select_step; conv_in is gemm #1, the first resnet's conv1 (72x2 CTAs, K=2880) gemm #2
timeout 500 ncu --set full --clock-control none --import-source on -k regex:gemm_tc_kernel -s 1 -c 2 \
    -o out/${TAG}_gemm -f $STEP > out/${TAG}_gemm.log 2>&1
timeout 500 ncu --set full --clock-control none --import-source on -k regex:flash_attn64 -s 0 -c 1 \
    -o out/${TAG}_attn -f $STEP > out/${TAG}_attn.log 2>&1
ls -la out/ | tail -8
