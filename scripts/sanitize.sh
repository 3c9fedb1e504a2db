#!/bin/bash
# Memory / race checks (run on a GPU box).  The shard rows are intentionally racy (asynchronous
# Hogwild updates through atomics), so racecheck is scoped to the control structures (rings, credit
# counter) and memcheck to the kernels with non-trivial addressing.
set -x
LOG=${LOG_DIR:-${TMPDIR:-/tmp}/fps_sanitize}
mkdir -p "$LOG"
export PYTHONUNBUFFERED=1
timeout 600 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_kernels.py -x -q \
  -k "pull_push_dot or matches_reference or packed64 or wide_rows or item_cache" > $LOG/sanitize_memcheck_kernels.log 2>&1
echo "memcheck kernels rc=$?"; tail -3 $LOG/sanitize_memcheck_kernels.log
timeout 600 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_topk.py tests/test_gpu_pa.py tests/test_gpu_sketch.py -x -q \
  > $LOG/sanitize_memcheck_topk_pa_sketch.log 2>&1
echo "memcheck topk/pa/sketch rc=$?"; tail -3 $LOG/sanitize_memcheck_topk_pa_sketch.log
