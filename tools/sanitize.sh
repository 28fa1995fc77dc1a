#!/bin/bash
# compute-sanitizer passes over the small GPU tests (every kernel family, tiny shapes): memcheck, then racecheck,
# synccheck and initcheck on the same selection.  Usage (through gpurun): bash tools/sanitize.sh [tools...]
set +e
out=gpurun_out/sanitize; mkdir -p $out
sel='goldens and not mid or other_class_counts or in_kernel or fused_epilogue or misaligned or status_codes or zero_points or generic_points or unaligned or daf_forward_backward or daf_matches or feature_maps or fused_forward or batched_launch or shared_points'
tools=${@:-memcheck racecheck synccheck initcheck}
for tool in $tools; do
  timeout 1500 compute-sanitizer --tool $tool --error-exitcode 7 --print-limit 30 --log-file $out/$tool.log \
      python -m pytest tests/test_splat_gpu.py tests/test_cabi_gpu.py tests/test_batch_fused_gpu.py tests/test_daf_gpu.py -m gpu -q -x -k "$sel" > $out/$tool.pytest.log 2>&1
  echo "$tool rc=$? : $(tail -1 $out/$tool.pytest.log)"
  grep -E "ERROR SUMMARY|RACECHECK SUMMARY" $out/$tool.log | tail -2
  grep -E "^=========     at|Invalid|Uninitialized|hazard|Barrier error" $out/$tool.log | sort | uniq -c | sort -rn | head -12
done
