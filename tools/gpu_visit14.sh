#!/usr/bin/env bash
# Round-2 visit 14 (1 GPU): where the C4 update+cull stage stands after the fallback skip and the fold rework — ncu launch list,
# full captures of the main level and of the fold; the in-order-fold variant test.
set -u
OUT=gpurun_out
TAG=r02r
mkdir -p $OUT
echo "[v14] variant test"; timeout 900 python -m pytest tests/test_gpu_variants.py -m gpu -q -x -k "fold_in_stream" 2>&1 | tail -3
K='regex:k_update_level|k_update_subforest|k_fold|k_palette|k_skin|k_snapshot|k_cull|k_scatter_trs'
B="--no-c5 --no-parity --no-cpu-baseline --no-device-animation"
echo "[v14] launch list"
timeout 400 ncu --metrics gpu__time_duration.sum --clock-control none -k "$K" --csv --log-file $OUT/${TAG}_launches_C4.csv \
    python bench.py --steps 2 --warmup 1 $B > $OUT/${TAG}_launches.log 2>&1
echo "[v14] full captures"
timeout 400 ncu --set full --clock-control none --import-source on -k regex:k_update_level --launch-skip 3 -c 1 -o $OUT/${TAG}_full_c4_update \
    python bench.py --workload C4 --steps 2 --warmup 1 $B > $OUT/${TAG}_full_a.log 2>&1
timeout 400 ncu --set full --clock-control none --import-source on -k 'regex:k_fold' --launch-skip 1 -c 1 -o $OUT/${TAG}_full_c4_fold \
    python bench.py --workload C4 --steps 2 --warmup 1 $B > $OUT/${TAG}_full_b.log 2>&1
ls -la $OUT/${TAG}_*.ncu-rep
echo "[v14] done"
