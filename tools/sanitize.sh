#!/usr/bin/env bash
# compute-sanitizer targets for the hand-written kernels (the reference ships no sanitizer usage, SURVEY §5.2).
# Run on one GPU:   bash tools/sanitize.sh memcheck
#   memcheck  : out-of-bounds / misaligned global+shared accesses (TMA boxes, swizzled staging, peer stores)
#   racecheck : shared-memory hazards between the producer / consumer / epilogue roles (mbarrier-ordered hand-offs)
#   synccheck : invalid barrier usage (named barriers of the GEMM epilogue)
# The kernel tests are tiny shapes, so a run is minutes even at sanitizer speed.  Multi-GPU flag protocols
# (st.release.sys / ld.acquire.sys) are covered functionally by tests/test_gpu_multi.py; racecheck does not model
# cross-GPU traffic.
set -euo pipefail
tool="${1:-memcheck}"
out="gpurun_out/sanitize_${tool}.log"
mkdir -p gpurun_out
compute-sanitizer --tool "$tool" --print-limit 20 --error-exitcode 1 \
    python -m pytest tests/test_gpu_kernels.py -x -q -k "gemm or layernorm or attention or cross_entropy" 2>&1 | tee "$out" | tail -15
