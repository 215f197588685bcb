"""-m gpu, needs >= 2 GPUs on the box: grouped-query attention over the native rings (NCCL, copy engine,
hierarchical at W >= 4), one process per GPU under torchrun (tests/ring_check_gqa.py)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_gqa_ring_parity_all_visible_gpus():
    n = min(torch.cuda.device_count(), 8)
    n = 1 << (n.bit_length() - 1)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr", "127.0.0.1", "--master-port", "29547", os.path.join(ROOT, "tests", "ring_check_gqa.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ))
    sys.stdout.write(res.stdout[-4000:])
    sys.stderr.write(res.stderr[-4000:])
    assert res.returncode == 0
