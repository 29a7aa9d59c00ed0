#!/bin/bash
# One GPU-box pass: parity tests, reference parity, sanitizer on the end-to-end step, bench.  Logs (small) -> $O (default ci_logs/).
# Selections are files and node ids, not -k substrings (-k also matches "matches", "prefetched", "unfused" and module names).
# The tensor-core and fused-kernel tests each run in a process of their own: a faulting kernel must not poison the other tests.
# So does the trained-checkpoint module (tests/test_gpu_checkpoint.py): it trains ngp_fox with the reference program once.
# And the training-with-octree-maintenance module (tests/test_gpu_train_maintenance.py): eight fused TRAIN steps per case.
# And the C++-host training-steps module (tests/test_gpu_cpp_host_steps.py): it runs the reference program for ten iterations per arm.
# And the float64-autograd gradient module (tests/test_gpu_grad_autograd.py): 48 TRAIN steps, each with a float64 twin on the device.
# And the C++ operator module (tests/test_gpu_cpp_ops_reference.py): it runs both reference binaries over 16 operator cases.
# And the geometry module (tests/test_gpu_geometry.py): the tensor-core point query, and a 300-iteration ngp_fox training.
# And the normals module (tests/test_gpu_normals.py): the tensor-core gradient kernel, and a 300-iteration ngp_fox training.
# And the reference-configs module (tests/test_gpu_ref_configs.py): both reference binaries, three arms on free, big20 and big22.
P=tests/test_gpu_parity.py
OWN=("$P::test_mlp_fwd_bwd" "$P::test_mlp_tc_tiles_and_f32_output" "$P::test_mlp_bwd_recompute_equals_saved"
     "$P::test_fused_epilogues_match_operator_sequence" "$P::test_fused_field_matches_unfused" "$P::test_shader_prep_bwd_fused_f16"
     tests/test_gpu_bwd_fused.py tests/test_gpu_shade_fused.py tests/test_gpu_checkpoint.py tests/test_gpu_train_maintenance.py
     tests/test_gpu_cpp_host_steps.py tests/test_gpu_grad_autograd.py tests/test_gpu_cpp_ops_reference.py tests/test_gpu_geometry.py tests/test_gpu_normals.py)
MAIN=(tests -m gpu --ignore=tests/test_ref_parity.py --ignore=tests/test_gpu_bwd_reference.py --ignore=tests/test_gpu_fwd_reference.py
      --ignore=tests/test_gpu_mlp_fwd_reference.py --ignore=tests/test_gpu_bwd_fused.py --ignore=tests/test_gpu_shade_fused.py --ignore=tests/test_gpu_checkpoint.py
      --ignore=tests/test_gpu_train_maintenance.py --ignore=tests/test_gpu_cpp_host_steps.py --ignore=tests/test_gpu_grad_autograd.py
      --ignore=tests/test_gpu_cpp_ops_reference.py --ignore=tests/test_gpu_geometry.py --ignore=tests/test_gpu_normals.py
      --ignore=tests/test_gpu_ref_configs.py)
for T in "${OWN[@]}"; do case "$T" in *::*) MAIN+=(--deselect "$T");; esac; done
if [ "${1:-}" = "--list" ]; then                 # print each pytest selection, one per line (collect with -m gpu --collect-only)
  echo "${MAIN[*]}"; for T in "${OWN[@]}"; do echo "$T"; done; echo tests/test_gpu_bwd_reference.py; echo tests/test_gpu_fwd_reference.py
  echo tests/test_gpu_mlp_fwd_reference.py; echo tests/test_ref_parity.py; echo tests/test_gpu_ref_configs.py
  exit 0
fi
O=${O:-ci_logs}
mkdir -p "$O"
echo "== gpu: $(nvidia-smi -L) / nproc $(nproc)"
timeout 1800 python -m pytest "${MAIN[@]}" -q -p no:cacheprovider > $O/pytest_gpu.log 2>&1
tail -n 40 $O/pytest_gpu.log
for T in "${OWN[@]}"; do
  L=${T##*/}; L=$O/pytest_${L//.py/}.log; L=${L//::/_}
  timeout 600 python -m pytest "$T" -m gpu -q -p no:cacheprovider > "$L" 2>&1
  echo "--- $T"; tail -n 25 "$L" | cut -c1-250
done
# the backward kernels against float64 / CPU-oracle references (multi-tile schedules, ~1 M-sample sizes)
timeout 1200 python -m pytest tests/test_gpu_bwd_reference.py -m gpu -q -p no:cacheprovider --durations=10 > $O/pytest_bwd_reference.log 2>&1
echo "--- tests/test_gpu_bwd_reference.py"; tail -n 40 $O/pytest_bwd_reference.log | cut -c1-250
# the slot-layout forward kernels and the fused forward renderer against the CPU oracle (planned ray lengths and early stops)
timeout 900 python -m pytest tests/test_gpu_fwd_reference.py -m gpu -q -p no:cacheprovider --durations=10 > $O/pytest_fwd_reference.log 2>&1
echo "--- tests/test_gpu_fwd_reference.py"; tail -n 40 $O/pytest_fwd_reference.log | cut -c1-250
# the packed tensor-core forwards, their epilogues and the casts against float64 / ATen references (tensor-core kernels: own process)
timeout 900 python -m pytest tests/test_gpu_mlp_fwd_reference.py -m gpu -q -p no:cacheprovider --durations=10 > $O/pytest_mlp_fwd_reference.log 2>&1
echo "--- tests/test_gpu_mlp_fwd_reference.py"; tail -n 40 $O/pytest_mlp_fwd_reference.log | cut -c1-250
timeout 600 python -m pytest tests/test_ref_parity.py -m gpu -q -p no:cacheprovider > $O/pytest_ref.log 2>&1
tail -n 60 $O/pytest_ref.log
# the free / big20 / big22 configs against the reference program in three arms (nine reference-program runs); -rs lists skips
timeout 1800 python -m pytest tests/test_gpu_ref_configs.py -m gpu -q -rs -p no:cacheprovider --durations=10 > $O/pytest_ref_configs.log 2>&1
echo "--- tests/test_gpu_ref_configs.py"; tail -n 40 $O/pytest_ref_configs.log | cut -c1-250
cp "$(python -c 'import tempfile; print(tempfile.gettempdir())')"/f2b_test_diag/refcfg_*.json "$O"/ 2>/dev/null   # measured margins
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
