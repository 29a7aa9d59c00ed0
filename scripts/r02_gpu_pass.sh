#!/bin/bash
# Round-2 measurement pass (one gpurun call, one GPU).  Everything lands in gpurun_out/<TAG>_*; the summaries that are
# judged are copied into profiles/ afterwards (scripts/ncu_summary.py, scripts/launch_share.py) and committed.
#   TAG=r02a STAGES="tests bench ref probes ncu full" bash scripts/r02_gpu_pass.sh
cd "$(dirname "$0")/.."
TAG=${TAG:-r02a}
STAGES=${STAGES:-"tests bench ref probes ncu full"}
O=gpurun_out
mkdir -p $O
has() { [[ " $STAGES " == *" $1 "* ]]; }
echo "== $(nvidia-smi -L | head -1) / nproc $(nproc) / tag $TAG / stages $STAGES"

if has tests; then
  timeout 1500 python -m pytest tests -m gpu -q -p no:cacheprovider -x --timeout 900 > $O/${TAG}_pytest_gpu.log 2>&1
  echo "--- pytest -m gpu: rc=$?"; tail -n 15 $O/${TAG}_pytest_gpu.log | cut -c1-220
  timeout 300 python __graft_entry__.py smoke > $O/${TAG}_smoke.log 2>&1; echo "--- smoke rc=$?"; tail -n 2 $O/${TAG}_smoke.log | cut -c1-200
fi
if has bench; then
  timeout 900 python bench.py --steps 20 --warmup 5 > $O/${TAG}_bench.json 2> $O/${TAG}_bench.err
  echo "--- bench rc=$?"; python - <<PY
import json
try:
    d = json.loads(open("$O/${TAG}_bench.json").read().strip().splitlines()[-1])
    k = {n: round(v["ms_per_step"], 3) for n, v in d["kernels"].items()}
    print(json.dumps({"ms_per_step": d["ms_per_step"], "value": d["value"], "e2e": d["e2e"], "roofline": d["roofline"], "kernels": k,
                      "launches": d["gpu_launches"], "measured": d["workload_measured"], "clocks": d["clocks"],
                      "forward_only": d.get("forward_only"), "reference_gpu": d.get("reference_gpu"), "cpu_baseline": d.get("cpu_baseline")}))
except Exception as e:
    print("bench parse failed:", e); print(open("$O/${TAG}_bench.err").read()[-1500:])
PY
fi
if has ref; then
  timeout 600 python bench.py --impl reference --steps 3 --warmup 1 > $O/${TAG}_bench_ref.json 2> $O/${TAG}_bench_ref.err
  echo "--- bench --impl reference rc=$?"; tail -c 1200 $O/${TAG}_bench_ref.json
fi
if has configs; then
  for C in free nerf360 big20 big22; do
    timeout 600 python bench.py --config $C --steps 20 --warmup 5 --no-cpu-baseline > $O/${TAG}_bench_$C.json 2> $O/${TAG}_bench_$C.err
    echo "--- bench --config $C rc=$?"; tail -c 600 $O/${TAG}_bench_$C.json | cut -c1-600; echo
  done
fi
if has probes; then
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/red scripts/microbench_red.cu && timeout 120 /tmp/red > $O/${TAG}_red_rate.json
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/gather scripts/microbench_gather.cu && timeout 120 /tmp/gather > $O/${TAG}_gather_rate.json
  timeout 300 python scripts/level_probe.py > $O/${TAG}_level_probe.json 2> $O/${TAG}_level_probe.err
  timeout 300 python scripts/mlp_probe.py > $O/${TAG}_mlp_probe.json 2> $O/${TAG}_mlp_probe.err
  timeout 300 python scripts/timeline.py --steps 6 > $O/${TAG}_timeline.json 2> $O/${TAG}_timeline.err
  for f in red_rate gather_rate level_probe mlp_probe; do echo "--- $f"; head -c 1500 $O/${TAG}_$f.json; echo; done
  echo "--- timeline"; head -c 2500 $O/${TAG}_timeline.json; echo
fi
if has ncu; then
  timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 800 --csv --log-file $O/${TAG}_launches.csv \
    python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-ref-gpu > $O/${TAG}_bench_ncu.log 2>&1
  echo "--- ncu launch list rc=$?"; wc -l $O/${TAG}_launches.csv
fi
if has full; then
  RE=${NCU_RE:-'march16|hash_bwd|field_fwd|mlp_fwd_tc|mlp_bwd|shader_prep_bwd|composite_bwd|composite_fwd|compact|mark_visit|early_stop'}
  timeout 1200 ncu --set full --import-source on --clock-control none -k "regex:$RE" -c ${NCU_CNT:-16} --launch-skip ${NCU_SKIP:-0} -f -o $O/prof_$TAG \
    python bench.py --steps 1 --warmup 1 --no-cpu-baseline --no-ref-gpu > $O/${TAG}_ncu_full.log 2>&1
  echo "--- ncu --set full rc=$?"; tail -n 2 $O/${TAG}_ncu_full.log | cut -c1-200; ls -la $O/prof_$TAG.ncu-rep
fi
du -sh $O
