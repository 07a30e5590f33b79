#!/bin/bash
# Round-end evidence in ONE run on one GPU: gpu tests, smoke, the default bench line, the reference
# arm, the bench table of DESIGN.md §7 and the ncu launch lists for profiles/. Outputs under gpurun_out/.
set -u
TAG=${1:-r1_final}
mkdir -p gpurun_out
echo "== pytest -m gpu"; timeout 600 python -m pytest tests -q -m gpu 2>&1 | tail -4
echo "== smoke"; timeout 200 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -2
echo "== bench (default)"; timeout 400 python bench.py 2>/dev/null | grep '^{' | tail -1 | tee gpurun_out/${TAG}_bench_default.json | cut -c1-400
echo "== bench --impl reference"; timeout 300 python bench.py --impl reference --steps 2 --warmup 1 2>/dev/null | grep '^{' | tail -1 | tee gpurun_out/${TAG}_bench_reference.json | cut -c1-300
: > gpurun_out/${TAG}_bench_table.jsonl
for spec in rmat24:clustering grid256:clustering rgg20:clustering rmat22:refinement grid256:refinement rmat22:contraction grid256:contraction; do
  w=${spec%%:*}; m=${spec##*:}
  extra="--no-cpu-baseline"; [ "$spec" = "rmat22:contraction" ] && extra=""
  timeout 400 python bench.py --workload $w --mode $m $extra 2>/dev/null | grep '^{' | tail -1 >> gpurun_out/${TAG}_bench_table.jsonl
done
python - <<PY
import json
for ln in open("gpurun_out/${TAG}_bench_table.jsonl"):
    d = json.loads(ln); c = d["config"]; e = d.get("e2e") or {}
    print(c["workload"], c["mode"], "ms", round(d["ms_per_step"], 2), "value %.3g" % d["value"], "e2e %.3g" % e.get("value", 0), "frac", round(d["roofline"]["frac"], 4), "launches", d["gpu_launches"])
PY
echo "== ncu launch lists"
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:"sweep_|commit_|k_[a-z]" -c 4000 --csv \
  --log-file gpurun_out/${TAG}_launches_rmat22.csv python bench.py --steps 1 --warmup 1 --no-cpu-baseline --no-e2e > gpurun_out/prof_a.log 2>&1
timeout 300 ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none \
  -k regex:"k_contract|k_coarse|k_map|k_flag|RadixSort|ReduceByKey|DeviceScan" -c 200 --csv \
  --log-file gpurun_out/${TAG}_contraction_launches_rmat22.csv python bench.py --mode contraction --steps 1 --warmup 0 --no-cpu-baseline --no-e2e > gpurun_out/prof_d.log 2>&1
ls -la gpurun_out | tail -8
