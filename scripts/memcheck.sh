#!/bin/bash
# compute-sanitizer memcheck over a representative slice of the GPU tests (on a machine with a GPU):
#   scripts/memcheck.sh > memcheck.log 2>&1
# Every kernel family is touched once: K0/K1 (all dtypes), build, Schur, persistent Cholesky, PCG dense + block-sparse,
# inner iterations, reference extraction, cost maps, KA (edge and query mode), dense SIFT, batched query BA (2 500 blocks,
# 18 columns), triangulation (verification, RANSAC tracks, evaluation), S2DNet.
set -u
run() {
  echo "=== $*"
  timeout 900 compute-sanitizer --tool memcheck --error-exitcode 99 --print-limit 5 python -m pytest "$@" -q -m gpu -x 2>&1 | grep -E "ERROR SUMMARY|passed|failed|Invalid|out of bounds|=========.*(Invalid|Error)" | head -12
}
run tests/test_gpu_ba_parity.py -k "residual_blocks or full_solve or tile_dag or block_sparse or iterative_schur_pcg"
run tests/test_gpu_refs.py
run tests/test_gpu_costmaps.py -k "extraction_matches or fused or full_solve"
run tests/test_gpu_ka.py
run tests/test_gpu_edge_cases.py -k "triangulation or single_free or clamped"
run tests/test_gpu_dsift.py -k "not past_2_to_the_31"
run tests/test_gpu_s2dnet.py -k "not past_2_to_the_31"
run tests/test_gpu_query_refinement_reference.py -k "b2500_full_opencv_all or b257_full_opencv_all"
run tests/test_gpu_triangulation.py
