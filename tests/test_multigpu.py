"""GPU, >= 2 devices (skipped on a machine with fewer): data-parallel equivalence of the training step's gradient exchange."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_gradients_equal_single_gpu_whole_batch():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29631", os.path.join(ROOT, "tools", "dp_equivalence.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "DP_EQUIV_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
