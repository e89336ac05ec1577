"""Worker for the multi-GPU append test: torchrun --nproc-per-node R tests/mgpu_append_worker.py
Each rank builds the same ElasticGPE, joins the NCCL communicator with row-sharded storage ("shard" = 1), appends points in
three steps and compares mll, alpha, gradient and predictions with a single-GPU GPE refitted on the full data."""
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
    ok = True
    for (N0, steps, rb, kern) in [
        (1500, (1, 200, 300), 2, gpb200.SEIso(0.3, 0.1)),
        (3000, (64, 1000), 4, gpb200.Mat32Iso(0.2, 0.1) + gpb200.RQIso(0.4, -0.3, 0.2)),
    ]:
        Nt = N0 + sum(steps)
        rng = np.random.default_rng(N0)
        X = rng.standard_normal((Nt, 3)); y = np.sin(X.sum(axis=1)) + 0.1 * rng.standard_normal(Nt)
        Xs = rng.standard_normal((50, 3))
        gp = gpb200.ElasticGPE(X[:N0].T, y[:N0], gpb200.MeanConst(0.2), kern, -0.5, capacity=Nt, device=local)
        gp._eng.set_option("shard", 1)
        gp._eng.set_option("shard_rb", rb)
        gp.init_distributed(p2p=False)
        n = N0
        for k in steps:
            gp.append(X[n:n + k].T, y[n:n + k])
            n += k
        gp.update_dmll()
        mu, s2 = gp.predict_f(Xs.T)
        info = gp._eng.storage_info()
        ref = gpb200.GPE(X.T, y, gpb200.MeanConst(0.2), kern, -0.5, device=local)        # single GPU, batch fit
        ref.update_target_and_dtarget()
        mr, vr = ref.predict_f(Xs.T)
        good = (info["sharded"] and gp.nobs == Nt and abs(gp.mll - ref.mll) <= 1e-10 * abs(ref.mll)
                and np.max(np.abs(gp.alpha - ref.alpha)) <= 1e-10 * np.max(np.abs(ref.alpha))
                and np.allclose(gp.dmll, ref.dmll, rtol=1e-8, atol=1e-10)
                and np.max(np.abs(mu - mr)) <= 1e-10 * np.max(np.abs(mr)) and np.max(np.abs(s2 - vr)) <= 1e-10 * np.max(np.abs(vr)))
        print("MGPU_APPEND rank %d world %d N0 %d -> %d (rb %d): mll %.15g vs %.15g -> %s"
              % (rank, world, N0, Nt, info["rb"], gp.mll, ref.mll, "OK" if good else "FAIL"), flush=True)
        t = torch.tensor([1.0 if good else 0.0], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        ok = ok and t.item() > 0.5
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_APPEND_RESULT", "PASS" if ok else "FAIL", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
