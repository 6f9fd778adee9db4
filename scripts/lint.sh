#!/bin/bash
# Static checks that need nothing beyond the toolchain in the image.
set -euo pipefail
cd "$(dirname "$0")/.."
python -m compileall -q torchft_b200 tests bench examples bench.py train_ddp.py train_diloco.py __graft_entry__.py
# every CUDA source must at least pass the front-end + ptxas for sm_90a
for f in torchft_b200/csrc/kernels/*.cu; do
  nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a -ccbin /usr/bin/g++ \
       $(python -m pybind11 --includes) -I torchft_b200/csrc/kernels -c "$f" -o /dev/null
done
python scripts/lint_unused.py
