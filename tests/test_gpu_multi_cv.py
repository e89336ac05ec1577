"""GPU (>= 2 devices): cross-validation on row-sharded storage over NCCL ranks ("shard" = 1) against a single-GPU GPE on the
full data.  Skipped on 1-GPU boxes."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu


def _ngpu():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_sharded_cv(world):
    if _ngpu() < world:
        pytest.skip("needs %d GPUs" % world)
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29731 + world), os.path.join(here, "mgpu_cv_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    sys.stdout.write(r.stdout[-4000:]); sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0 and "MGPU_CV_RESULT PASS" in r.stdout
