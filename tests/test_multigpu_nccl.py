"""GPU, two or more devices: the gradient exchange of the view-sharded step over NCCL (SURVEY.md 8e).  Skipped on a
machine with one GPU; run `python -m pytest tests/test_multigpu_nccl.py -m gpu -q` on one with two or more."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def test_compact_exchange_equals_allreduce_over_nccl():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least two GPUs")
    world = 2
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(29600 + os.getpid() % 300), os.path.join(ROOT, "tests", "nccl_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stderr[-3000:]
