#!/bin/bash
# compute-sanitizer racecheck (shared-memory hazards) over the kernels that use shared memory: K1 (TMA ring + aux),
# the persistent Cholesky (tiles, named barriers), the KA kernel (dense H / vectors), IRLS, dense SIFT (staged halo, E / P),
# batched query BA (shared projected rows and warp partials at 2 500 blocks and 18 columns).
set -u
run() {
  echo "=== $*"
  timeout 1200 compute-sanitizer --tool racecheck --error-exitcode 99 --print-limit 5 python -m pytest "$@" -q -m gpu -x 2>&1 | grep -E "RACECHECK SUMMARY|passed|failed|hazard" | head -8
}
run tests/test_gpu_ba_parity.py -k "residual_blocks or tile_dag"
run tests/test_gpu_ka.py -k "matches_oracle"
run tests/test_gpu_refs.py
run tests/test_gpu_dsift.py -k "oracle or bit_for_bit"
run tests/test_gpu_query_refinement_reference.py -k "linearisation and (b2500 or b257_full_opencv_all)"
