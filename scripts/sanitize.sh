#!/bin/bash
# Race / memory checking (the reference has none in-tree, SURVEY.md §5.2).
#   control plane : the native selftest (unit tables, live Lighthouse + ManagerServer, hostile raw traffic)
#                   under ThreadSanitizer and AddressSanitizer+UBSan             -- CPU only
#   CUDA kernels  : compute-sanitizer memcheck + racecheck + synccheck over the GPU kernel tests -- needs a GPU
set -euo pipefail
cd "$(dirname "$0")/.."
python - <<'PY'
from torchft_b200 import _build
for s in ("thread", "address"):
    print(_build.build_selftest(sanitize=s))
PY
TSAN_OPTIONS="halt_on_error=1 second_deadlock_stack=1" bin/torchft_b200_selftest_tsan
ASAN_OPTIONS="detect_leaks=1" UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1" bin/torchft_b200_selftest_asan
if python -c "import torch,sys; sys.exit(0 if torch.cuda.is_available() else 1)"; then
  for tool in memcheck racecheck synccheck; do
    compute-sanitizer --tool $tool --error-exitcode 1 --launch-timeout 120 \
      python -m pytest tests/test_kernels_gpu.py tests/test_heal_exact_gpu.py::test_heal_copy -x -q -m gpu -k "rmsnorm or swiglu or rope or cross_entropy or adamw or q8_roundtrip or heal_copy"
  done
fi
