"""Worker for the multi-GPU cross-validation test: torchrun --nproc-per-node R tests/mgpu_cv_worker.py
Each rank builds the same GPE, joins the NCCL communicator with row-sharded storage ("shard" = 1) and compares the LOO and
k-fold values and gradients, and the K^-1 / M_j sub-blocks, with a single-GPU GPE on the full data."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def main():
    import torch
    import torch.distributed as dist
    import gpb200

    rank = int(os.environ["RANK"]); local = int(os.environ["LOCAL_RANK"]); world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ok = True
    for (N, rb, kern) in [
        (1500, 2, gpb200.Mat52Iso(0.3, 0.1) + gpb200.fix(gpb200.SEIso(-0.2, 0.3), "lσ")),
        (3000, 4, gpb200.Mat32Iso(0.2, 0.1) + gpb200.RQIso(0.4, -0.3, 0.2)),
    ]:
        rng = np.random.default_rng(N)
        X = rng.standard_normal((N, 2)); y = np.sin(X.sum(axis=1)) + 0.1 * rng.standard_normal(N)
        folds = [np.arange(128 * rb - 60, 128 * rb + 70), np.sort(rng.choice(np.arange(700, N), 150, replace=False))]
        gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), kern, -0.7, device=local)
        gp._eng.set_option("shard", 1)
        gp._eng.set_option("shard_rb", rb)
        gp.init_distributed(p2p=False)
        ref = gpb200.GPE(X.T, y, gpb200.MeanZero(), kern, -0.7, device=local)        # single GPU
        mu, s2 = gp.predict_LOO(); mr, sr = ref.predict_LOO()
        g, gr = gp.dlogp_LOO(), ref.dlogp_LOO()
        gf, gfr = gp.dlogp_CVfold(folds), ref.dlogp_CVfold(folds)
        lf, lfr = gp.logp_CVfold(folds), ref.logp_CVfold(folds)
        j = int(gp._exposed[0])
        za, dz = gp._eng.cv_param(j); zr, dr = ref._eng.cv_param(j)
        B1, B1r = gp._eng.cv_block(1, folds[0]), ref._eng.cv_block(1, folds[0])
        info = gp._eng.storage_info()
        good = (info["sharded"] and info["bytes_cv"] > 0 and _rel(mu, mr) < 1e-9 and _rel(s2, sr) < 1e-9
                and np.allclose(g, gr, rtol=1e-7, atol=1e-9) and np.allclose(gf, gfr, rtol=1e-6, atol=1e-8)
                and abs(lf - lfr) <= 1e-8 * abs(lfr) and _rel(za, zr) < 1e-8 and _rel(dz, dr) < 1e-8
                and np.array_equal(B1, B1.T) and _rel(B1, B1r) < 1e-8)
        print("MGPU_CV rank %d world %d N %d (rb %d): dlogp_LOO %s vs %s -> %s"
              % (rank, world, N, info["rb"], g, gr, "OK" if good else "FAIL"), flush=True)
        t = torch.tensor([1.0 if good else 0.0], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        ok = ok and t.item() > 0.5
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_CV_RESULT", "PASS" if ok else "FAIL", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
