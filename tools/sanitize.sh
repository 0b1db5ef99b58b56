#!/bin/bash
# compute-sanitizer pass over the single-GPU kernel tests (SURVEY.md section 5: race detection / sanitizers).
#   tools/sanitize.sh [memcheck|racecheck|synccheck|initcheck] [pytest -k expression]
# Lock mode is the deterministic oracle for the (intentionally racy) Hogwild mode, so racecheck is only meaningful
# on the lock-mode and single-kernel tests.
TOOL=${1:-memcheck}
EXPR=${2:-"cast_transpose or softmax or mse or argmax or gemm_plain or push_matches or pull_copies"}
mkdir -p bench_out
SPARKFLOW_NO_PDL=1 timeout ${SANITIZE_TIMEOUT:-600} compute-sanitizer --tool "$TOOL" --error-exitcode 9 --print-limit 20 \
  --log-file bench_out/sanitize_$TOOL.log python -m pytest tests/test_gpu_kernels.py -m gpu -x -q -k "$EXPR" -p no:cacheprovider
RC=$?
echo "compute-sanitizer $TOOL exit code: $RC"
tail -5 bench_out/sanitize_$TOOL.log
exit $RC
