"""N > 1: the time-sharded solver (replicated and distributed reduced solve over NCCL) against the unsharded oracle.
Needs >= 2 GPUs on the machine; skipped otherwise."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_two_gpu_sharded_lm_matches_oracle():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29577", os.path.join(ROOT, "tests", "multi", "check_sharded.py")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "all sharded x2 cases ok" in r.stdout and r.stdout.count("sharded x2 ok") == 5
