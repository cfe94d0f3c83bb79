"""Multi-GPU tests (need >= 2 CUDA devices: `python -m pytest tests/test_gpu_multi.py -m gpu` on a machine with two or
more GPUs; skipped on a single GPU)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_fused_nvlink_allreduce_world2():
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
           '127.0.0.1', '--master-port', '29533', os.path.join(ROOT, 'tests', 'dist_fused_allreduce.py')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and 'DIST OK world=2' in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
