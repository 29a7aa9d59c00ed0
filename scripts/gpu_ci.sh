#!/bin/bash
# One GPU-box pass: parity tests, reference parity, sanitizer on the end-to-end step, bench.  Logs (small) -> $O (default ci_logs/).
O=${O:-ci_logs}
mkdir -p "$O"
echo "== gpu: $(nvidia-smi -L) / nproc $(nproc)"
timeout 900 python -m pytest tests -m gpu -q --deselect tests/test_ref_parity.py -p no:cacheprovider -k "not tc and not fused" > $O/pytest_gpu.log 2>&1
tail -n 40 $O/pytest_gpu.log
# tensor-core kernels in their own processes (a faulting kernel must not poison the other tests)
for K in "tc-0" "tc-1" "fused" "tiles"; do
  timeout 300 python -m pytest tests/test_gpu_parity.py -m gpu -q -p no:cacheprovider -k "$K" > $O/pytest_$K.log 2>&1
  echo "--- -k $K"; tail -n 25 $O/pytest_$K.log | cut -c1-250
done
timeout 600 python -m pytest tests/test_ref_parity.py -m gpu -q -p no:cacheprovider > $O/pytest_ref.log 2>&1
tail -n 60 $O/pytest_ref.log
if [ "${SANITIZE:-0}" = "1" ]; then
  timeout 900 compute-sanitizer --tool memcheck --print-limit 8 python -m pytest "tests/test_gpu_render.py::test_render_train_step_matches_oracle" -q -x -p no:cacheprovider -k "64" > $O/sanitizer.log 2>&1
  grep -E "Invalid|at 0x|by thread|Address|in /|\.cu:|=========     at|ERROR SUMMARY" $O/sanitizer.log | head -40
fi
timeout 300 python __graft_entry__.py smoke 2>&1 | tail -n 2
timeout 500 python bench.py --steps ${STEPS:-5} --warmup 3 > $O/bench.json 2> $O/bench.err
tail -c 4000 $O/bench.json; tail -n 5 $O/bench.err
du -sh "$O"
if [ "${NCU:-0}" = "1" ]; then
  timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file $O/launches.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-ref-gpu > $O/bench_ncu.log 2>&1
  tail -n 3 $O/bench_ncu.log | cut -c1-300; wc -l $O/launches.csv
fi
