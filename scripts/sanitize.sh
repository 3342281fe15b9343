# compute-sanitizer over a slice of the GPU parity suite (interpreter AND specialised kernels): memcheck for out-of-bounds /
# misaligned accesses, racecheck for shared-memory hazards in the tile pipeline (TMA stages, dictionary, look-back) and synccheck.
# Logs land in $OUT.  Every run is bounded (200 s).
OUT=gpurun_out/evidence; mkdir -p $OUT
R=${ROUND:-r02}
SEL='test_projection and 1000 or test_filter and 5000 and not two_pass or test_aggregate_single and 1000 or test_two_phase_aggregate or test_divide_by_zero or test_aggregate_batches_differ and alternating'
REL='test_hash_join_unique_build and 50-500 or test_hash_join_duplicate_build_keys or test_hash_join_string_keys or test_sort and 5000 or test_hash_repartition and 2 or test_row_round_robin_reference_kat or test_substr or test_nested_loop or test_sort_preserving_merge and 2-None or test_topk_selection and 10-keys0 or test_semi_anti_join_with_residual_filter and False'
run() {   # tool, name, env assignment, test file, selection
  local log=$OUT/${R}_sanitizer_$1_$2.log
  env $3 timeout 200 compute-sanitizer --tool $1 --error-exitcode 1 --launch-timeout 0 python -m pytest $4 -m gpu -x -q -k "$5" > $log 2>&1
  echo "exit=$?" >> $log
  echo "== $log"; grep -E "ERROR SUMMARY|passed|failed|exit=" $log | tail -3
}
run memcheck pipeline_jit SAILGPU_JIT_MIN_ROWS=0 tests/test_gpu_pipeline.py "$SEL"
run memcheck pipeline_vm SAILGPU_JIT=0 tests/test_gpu_pipeline.py "$SEL"
run memcheck relational SAILGPU_JIT_MIN_ROWS=0 tests/test_gpu_relational.py "$REL"
run racecheck pipeline_jit SAILGPU_JIT_MIN_ROWS=0 tests/test_gpu_pipeline.py "$SEL"
run racecheck pipeline_vm SAILGPU_JIT=0 tests/test_gpu_pipeline.py "$SEL"
run synccheck pipeline_jit SAILGPU_JIT_MIN_ROWS=0 tests/test_gpu_pipeline.py "test_aggregate_single and 1000 or test_two_phase_aggregate"
