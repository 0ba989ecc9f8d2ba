"""GPU, needs >= 2 devices: cluster-sharded solve over NCCL vs the single-GPU solve."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_matches_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29617",
           os.path.join(ROOT, "tests", "mgpu_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    print(out.stdout[-3000:], out.stderr[-3000:])
    assert out.returncode == 0 and "MGPU_CHECK OK" in out.stdout


def test_consensus_over_subbands():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29618",
           os.path.join(ROOT, "tests", "consensus_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    print(out.stdout[-3000:], out.stderr[-3000:])
    assert out.returncode == 0 and "CONSENSUS_CHECK OK" in out.stdout
