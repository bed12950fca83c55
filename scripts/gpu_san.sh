#!/bin/bash
# compute-sanitizer over the parity tests that exercise every kernel (agg FLAT / per-block / gather, GAP merge, slab gather, scan, shift, blob decode, rs v2)
# + one full-set ncu capture of the two kernels the other capture scripts do not reach
mkdir -p gpurun_out
P=tests/test_gpu_parity.py
T="$P::test_aggregate_vs_golden $P::test_gap_stream_and_gather_paths_agree $P::test_flat_window_all_gap_styles $P::test_pipeline_batch $P::test_edge_cases $P::test_large_groups_chunked_classification $P::test_rs_index_vs_oracle_including_full_and_edges $P::test_rs_index_rank_select_vs_golden $P::test_gap_flat_and_raw_formats $P::test_scan_vs_golden $P::test_shift_right_and_vs_oracle $P::test_deserialize_to_device_vs_golden_and_oracle $P::test_binop_result_kinds_vs_reference $P::test_upload_slabs_dma_plus_device_gather_equals_host_packing $P::test_sharded_rs_device_callables_two_shards_one_gpu"
timeout 1500 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest $T -x -q 2>&1 | grep -E "ERROR SUMMARY|passed|failed|Invalid|at .*bmb200" | head -20 | tee gpurun_out/sanitizer_memcheck.log
timeout 600 compute-sanitizer --tool racecheck --print-limit 5 python -m pytest $P::test_binop_result_kinds_vs_reference $P::test_rs_index_vs_oracle_including_full_and_edges $P::test_flat_window_all_gap_styles -x -q 2>&1 | grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed|hazard|bmb200" | head -10 | tee gpurun_out/sanitizer_racecheck.log
# the plane-search kernels with several columns per CTA (the smallest grid-scale configuration: one CTA per SM, three launches)
G="tests/test_plane_search_grid.py::test_scan_unsigned[ctas1-1]"
for tool in racecheck synccheck; do
  timeout 1200 compute-sanitizer --tool $tool --print-limit 5 python -m pytest "$G" -x -q -m gpu 2>&1 | grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed|hazard|bmb200" | head -10
done
timeout 300 ncu --set full --clock-control none -k regex:"gap_merge_kernel|slab_gather_kernel" -c 8 -f -o gpurun_out/prof_rest3 \
   python -m pytest $P::test_binop_result_kinds_vs_reference $P::test_upload_slabs_dma_plus_device_gather_equals_host_packing -q > gpurun_out/ncu_rest3.log 2>&1
ncu -i gpurun_out/prof_rest3.ncu-rep --page raw --csv > gpurun_out/ncu_rest3_raw.csv 2>/dev/null
rm -f gpurun_out/prof_rest3.ncu-rep
tail -2 gpurun_out/ncu_rest3.log
