# Build + test image. The control plane is plain C++17 (no Rust/protoc toolchain as in the reference's
# maturin image); the kernels need nvcc >= 12.0 for sm_90a.
FROM nvidia/cuda:12.9.0-devel-ubuntu24.04
RUN apt-get update && apt-get install -y --no-install-recommends python3 python3-pip python3-dev g++ git && rm -rf /var/lib/apt/lists/*
RUN pip install --break-system-packages torch pybind11 numpy pytest pytest-timeout
WORKDIR /workspace/torchft_b200
COPY . .
RUN python3 -m torchft_b200._build
CMD ["python3", "-m", "torchft_b200.lighthouse", "--min_replicas", "1"]
