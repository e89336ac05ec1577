"""GPU (>= 2 devices): append for FITC, DTC and SoR with the observations sharded over 2 ranks, each rank appending its own
rows (none on one rank in one step), against a one-rank model on the union.  Skipped on 1-GPU boxes."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu


def test_multi_gpu_append():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29687", os.path.join(here, "mgpu_fitc_append_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    sys.stdout.write(r.stdout[-4000:]); sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0 and "MGPU_RESULT PASS" in r.stdout
