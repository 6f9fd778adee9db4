"""HSDPTrainer (FSDP2 inside a replica group x fault-tolerant all-reduce across groups) on one GPU: 1 group x 1 shard
still runs FSDP2's all-gather / reduce-scatter / all-reduce-hook machinery against the fused model ops.
Reference wiring: upstream torchft/fsdp_test.py:57-72."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a GPU")
@pytest.mark.parametrize("backend", ["b200", "nccl"])
def test_hsdp_one_group_trains_with_finite_gradients(backend):
    env = dict(os.environ, MASTER_PORT=str(29655 + (backend == "nccl")))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gpu", "hsdp_debug.py"), "llama3_debug", backend],
                         capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert out.returncode == 0 and "HSDP_DEBUG ok" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
