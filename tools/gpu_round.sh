#!/usr/bin/env bash
# One GPU-box visit that produces everything a round needs (box acquisition is the expensive part of a gpurun call):
#   tests -> bench (default = C4 + strong C5 + parity; C2, target, C3) -> reference arm -> ncu launch list of the default bench
#   command -> ncu --set full of the hot kernels ON C4 (traffic) -> N2 / N3 tools.  Everything lands in gpurun_out/<tag>_*;
#   summaries: tools/make_profiles.py / tools/ncu_summary.py.
#   usage (from the repo root, on the GPU box):  bash tools/gpu_round.sh r02 [quick]
# "quick" skips the ncu captures.  Every step has its own timeout so that a hang cannot eat the budget.
set -u
TAG=${1:-rXX}
MODE=${2:-full}
OUT=gpurun_out
mkdir -p $OUT
log() { echo "[gpu_round] $*"; }
summ() {
python - "$1" <<'PY'
import json, sys
try:
    d = json.load(open(sys.argv[1]))
    st = {k: (round(v["ms"], 4), round(v["frac"], 3)) for k, v in d["roofline"]["stages"].items()}
    print("   ms/frame", round(d["ms_per_step"], 4), "e2e", round(d["e2e"]["ms_per_step"], 4), st, "launches", d["gpu_launches"], "parity", (d.get("parity") or {}).get("ok"))
    c5 = (d.get("modes") or {}).get("strong_C5")
    if c5:
        print("   strong C5:", {k: c5.get(k) for k in ("ms_per_step", "e2e_ms_per_step", "value")}, "parity", (c5.get("parity") or {}).get("ok"))
except Exception as ex:
    print("   (no JSON line)", ex)
PY
}

log "tests"
timeout 2400 python -m pytest tests -m gpu -q 2>&1 | tail -15 > $OUT/${TAG}_tests.log
tail -3 $OUT/${TAG}_tests.log

log "sanitizer (memcheck, racecheck) over the small parity tests"
SMALL='test_update_matches_oracle_on_generated_scenes or test_incremental_update or test_cull_six_cube_faces or test_palette_and_skinning or test_render_prep_one_call or test_pipelined_frames or test_skinned_mesh_box_quirk or test_blend_shapes'
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -q -x -k "$SMALL" > $OUT/${TAG}_memcheck.log 2>&1; echo "rc=$?" >> $OUT/${TAG}_memcheck.log; tail -3 $OUT/${TAG}_memcheck.log
timeout 900 compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -q -x -k "$SMALL" > $OUT/${TAG}_racecheck.log 2>&1; echo "rc=$?" >> $OUT/${TAG}_racecheck.log; tail -3 $OUT/${TAG}_racecheck.log

for w in C4 C2 target C3; do
    extra="--no-cpu-baseline --no-device-animation --no-c5"
    [ "$w" = "C4" ] && extra=""   # the default command, complete (C5 strong + CPU baseline included)
    log "bench $w"
    timeout 900 python bench.py --workload $w $extra > $OUT/${TAG}_bench_$w.json 2> $OUT/${TAG}_bench_$w.err
    summ $OUT/${TAG}_bench_$w.json
done

log "reference arm (bounded sample + one full-workload frame)"
timeout 900 python bench.py --impl reference --steps 3 --warmup 1 > $OUT/${TAG}_bench_reference.json 2> $OUT/${TAG}_bench_reference.err
python -c "import json; d=json.load(open('$OUT/${TAG}_bench_reference.json')); print('   ', d['value'], d.get('full_workload_frame'))" 2>/dev/null

log "N3 / N2 tools"
timeout 200 python tools/drawprep_bench.py > $OUT/${TAG}_drawprep.json 2> $OUT/${TAG}_drawprep.err
cat $OUT/${TAG}_drawprep.json

if [ "$MODE" != "quick" ]; then
    K='regex:k_update_level|k_update_subforest|k_fold|k_palette|k_skin|k_snapshot|k_cull|k_scatter_trs|k_anim|k_inst|k_lod|k_peer'
    B="--no-c5 --no-parity --no-cpu-baseline --no-device-animation"
    log "ncu launch list of the default bench workload (C4)"
    timeout 400 ncu --metrics gpu__time_duration.sum --clock-control none -k "$K" --csv --log-file $OUT/${TAG}_launches_C4.csv \
        python bench.py --steps 2 --warmup 1 $B > $OUT/${TAG}_launches.log 2>&1
    log "ncu --set full on C4: main level of the fused update+cull, k_skin (traffic measured on C4), palette, fold"
    timeout 400 ncu --set full --clock-control none --import-source on -k regex:k_update_level --launch-skip 3 -c 1 -o $OUT/${TAG}_full_c4_update \
        python bench.py --workload C4 --steps 2 --warmup 1 $B > $OUT/${TAG}_full_a.log 2>&1
    timeout 400 ncu --set full --clock-control none --import-source on -k 'regex:k_skin|k_palette|k_fold' --launch-skip 3 -c 3 -o $OUT/${TAG}_full_c4_skin \
        python bench.py --workload C4 --steps 2 --warmup 1 $B > $OUT/${TAG}_full_b.log 2>&1
    ls -la $OUT/${TAG}_*.ncu-rep 2>/dev/null
fi
log "done"
