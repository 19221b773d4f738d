#!/bin/bash
# Validation on ONE GPU: GPU tests, smoke, the default bench line, the other backbones in both tensor-core precisions,
# the reference arm.  usage: bash tools/final_check.sh <tag> [outdir]   -> <outdir>/bench_*_<tag>.json
TAG=${1:-v1}
OUT=${2:-check_out}
mkdir -p "$OUT"
timeout 900 python -m pytest tests -m gpu -x -q 2>&1 | tail -3
timeout 200 python -c "import __graft_entry__ as g; g.smoke(); print('SMOKE OK')" 2>&1 | tail -3
timeout 400 python bench.py 2>$OUT/bench_full_${TAG}.err | tail -1 > $OUT/bench_full_${TAG}.json
for a in res_50:16 hrnet:16 mobilenetv3:64; do
  arch=${a%%:*}; b=${a##*:}
  for p in fp16x2 bf16; do
    timeout 200 python bench.py --arch $arch --batch $b --precision $p --no-extras --no-cpu-baseline 2>/dev/null | tail -1 > $OUT/bench_${arch}_${p}_${TAG}.json
  done
done
timeout 300 python bench.py --impl reference --steps 2 --warmup 1 2>/dev/null | tail -1 > $OUT/bench_reference_arm_${TAG}.json
python - "$TAG" "$OUT" <<'PY'
import glob, json, sys
tag, out = sys.argv[1], sys.argv[2]
for f in sorted(glob.glob(f"{out}/bench_*_{tag}.json")):
    try:
        d = json.load(open(f)); print(f, round(d["value"], 2), round(d["ms_per_step"], 3), round(d["e2e"]["value"], 1), d.get("gpu_launches"))
    except Exception as e:
        print(f, "ERR", e)
d = json.load(open(f"{out}/bench_full_{tag}.json"))
print(json.dumps(d["roofline"].get("dominant_kernel"))[:1600])
print(d["parity"]["head_maps_rel_l2"], d["parity"]["rows_all_56_values_within_1e-3"], d["fast_mode"]["value"], d["decode"], d["cpu_baseline"]["value"], d["clocks"])
PY
tail -3 $OUT/bench_full_${TAG}.err
