"""Worker for the multi-GPU inducing-point gradient test: torchrun --nproc-per-node R tests/mgpu_inducing_worker.py
Every rank holds its slice of the observations and the same Xu; dmll/dXu of the distributed FITC must equal the single-GPU
value on the full data set within 1e-10 relative."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))


def main():
    import torch
    import torch.distributed as dist
    import gpb200

    rank = int(os.environ["RANK"]); local = int(os.environ["LOCAL_RANK"]); world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rng = np.random.default_rng(91)
    N, M, d = 6000, 140, 3
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-1.5, 1.5, (M, d))
    kf = gpb200.SEArd([-0.4, -0.6, -0.5], 0.1)
    lo, hi = rank * N // world, (rank + 1) * N // world
    ok = True
    for mode in ("FITC", "DTC", "SoR"):
        cls = getattr(gpb200, mode)
        gd = cls(X[lo:hi].T, Xu.T, y[lo:hi], gpb200.MeanConst(0.1), kf, -1.0, device=local, distributed=True)
        gd.update_dmll(inducing=True)
        gs = cls(X.T, Xu.T, y, gpb200.MeanConst(0.1), kf, -1.0, device=local)
        gs.update_dmll(inducing=True)
        nu = Xu.size
        err = np.max(np.abs(gd.dmll[-nu:] - gs.dmll[-nu:])) / np.max(np.abs(gs.dmll[-nu:]))
        m_ok = err <= 1e-10
        print("MGPU rank %d %s dmll/dXu over %d ranks: max rel err %.3e -> %s" % (rank, mode, world, err, "OK" if m_ok else "FAIL"),
              flush=True)
        t = torch.tensor([1.0 if m_ok else 0.0], dtype=torch.float64, device="cuda"); dist.all_reduce(t, op=dist.ReduceOp.MIN)
        ok = ok and t.item() > 0.5
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_RESULT", "PASS" if ok else "FAIL", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
