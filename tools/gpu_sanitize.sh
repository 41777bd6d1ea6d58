#!/bin/bash
# compute-sanitizer over a selection of the gpu-marked tests on the hardware: memcheck (out-of-bounds / misaligned accesses of the
# real SASS), racecheck (shared-memory hazards between warps: the shared-tile barriers of scan_kernel<SUB, ..>, stage B's
# commit), synccheck.  Summary in gpurun_out/r02_sanitizer.txt, full logs beside it.
mkdir -p gpurun_out
SEL="ragged_and_tiny or one_segment_per_buffer or few_survivors or timestamp_discontinuity or modeac_with_empty or golden or dense_tile or modeac_matches"
for tool in memcheck racecheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 9 python -m pytest tests/test_gpu_edges.py tests/test_gpu_parity.py -m gpu -x -q -k "$SEL" > gpurun_out/sanitize_$tool.log 2>&1
  echo "$tool rc=$?"; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed" gpurun_out/sanitize_$tool.log | tail -3
done | tee gpurun_out/r02_sanitizer.txt
