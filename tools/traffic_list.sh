#!/bin/bash
# Per-kernel time + DRAM traffic of ONE bench step (ncu; compare SHARES, not absolutes).
# usage (under gpurun): bash tools/traffic_list.sh <tag> <launches_per_step> [extra bench args]
TAG=${1:-r02}; NPER=${2:-96}; shift; shift
mkdir -p gpurun_out
SKIP=$((NPER * 3))
ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none \
    -k regex:"avgpool_kernel|conv3x3_tc_kernel|conv_simt_kernel|conv_sp_kernel|conv_tc_kernel|convert_from_split_kernel|convert_to_split_kernel|decode_kernel|dwconv_kernel|dwconv_tiled_kernel|dwdeconv_add_fast_kernel|dwdeconv_add_kernel|flip_merge_kernel|maxpool_kernel|scale_add_kernel|sigmoid_kernel|soft_nms_kernel|stem_kernel|stem_tc_h_kernel|stem_tc_kernel|upsample_add_kernel" \
    -s ${SKIP} -c ${NPER} --csv --log-file gpurun_out/traffic_${TAG}.csv \
    python bench.py --steps 1 --warmup 3 --no-cpu-baseline --no-extras "$@" > gpurun_out/traffic_${TAG}.log 2>&1
python - gpurun_out/traffic_${TAG}.csv <<'PY' > gpurun_out/traffic_${TAG}_summary.txt
import csv, sys
from collections import defaultdict
lines = [l for l in open(sys.argv[1]) if not l.startswith("==")]
t = defaultdict(float); r = defaultdict(float); w = defaultdict(float); n = defaultdict(int); order = {}; per = defaultdict(dict)
for row in csv.DictReader(lines):
    name = row["Kernel Name"].split("(")[0].replace("void <unnamed>::", "").replace("<unnamed>::", "").replace("void ", "")
    order.setdefault(row["ID"], name)
    v = float(row["Metric Value"].replace(",", "")); u = row.get("Metric Unit", "")
    m = row["Metric Name"]
    if m == "gpu__time_duration.sum":
        us = v / 1000.0 if u in ("ns", "nsecond") else (v if u in ("us", "usecond") else v * 1000.0)
        t[name] += us; n[name] += 1; per[row["ID"]]["us"] = us
    else:
        scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
        (r if m == "dram__bytes_read.sum" else w)[name] += v * scale
        per[row["ID"]]["rd" if m == "dram__bytes_read.sum" else "wr"] = v * scale
print("# kernel, launches, time_us, dram_read_MB, dram_write_MB")
for k in sorted(t, key=lambda k: -t[k]):
    print(f"{k:58s} {n[k]:4d} {t[k]:10.1f} {r[k] / 1e6:10.1f} {w[k] / 1e6:10.1f}")
print("# ---- launches in program order: index, kernel, time_us, dram_read_MB, dram_write_MB")
for i, k in enumerate(sorted(order, key=lambda x: int(x))):
    p = per[k]
    print(f"{i:3d} {order[k]:58s} {p.get('us', 0):9.1f} {p.get('rd', 0) / 1e6:9.1f} {p.get('wr', 0) / 1e6:9.1f}")
print(f"# total: {sum(n.values())} launches, {sum(t.values()):.1f} us, read {sum(r.values()) / 1e6:.1f} MB, write {sum(w.values()) / 1e6:.1f} MB, "
      f"sum {(sum(r.values()) + sum(w.values())) / 1e9:.3f} GB")
PY
cat gpurun_out/traffic_${TAG}_summary.txt
