"""Worker for the multi-GPU training-input gradient test: torchrun --nproc-per-node R tests/mgpu_inputs_worker.py
Every rank builds the same GPE and joins the NCCL communicator, once with replicated storage and once row-sharded
("shard" = 1); dmll/dX must equal the single-GPU value within 1e-12 of its largest entry (only the cross-rank sum order
differs) and repeat bitwise."""
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
    rng = np.random.default_rng(93)
    N, d = 5000, 3
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    kern = gpb200.SEIso(0.2, 0.1) + gpb200.RQIso(0.3, 0.0, 0.2)
    ref = gpb200.GPE(X.T, y, gpb200.MeanLin([0.2, 0.1, -0.3]), kern, -1.0, device=local)
    ref.update_dmll(noise=False, domean=False, kern=False, inputs=True)
    ok = True
    for storage in ("replicated", "sharded"):
        gp = gpb200.GPE(X.T, y, gpb200.MeanLin([0.2, 0.1, -0.3]), kern, -1.0, device=local)
        if storage == "sharded":
            gp._eng.set_option("shard", 1)
        gp.init_distributed(p2p=False)
        gp.update_dmll(noise=False, domean=False, kern=False, inputs=True)
        a = gp.dmll.copy()
        gp.update_dmll(noise=False, domean=False, kern=False, inputs=True)
        err = np.max(np.abs(a - ref.dmll)) / np.max(np.abs(ref.dmll))
        m_ok = err <= 1e-12 and np.array_equal(a, gp.dmll) and gp._eng.storage_info()["sharded"] == (storage == "sharded")
        print("MGPU rank %d %s dmll/dX over %d ranks: max rel err %.3e -> %s" % (rank, storage, world, err, "OK" if m_ok else "FAIL"),
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
