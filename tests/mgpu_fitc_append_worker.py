"""Worker for the multi-GPU append test: torchrun --nproc-per-node R tests/mgpu_fitc_append_worker.py
Every rank holds its slice of the observations and the same Xu, and appends its own new rows in three collective steps (in
the second, rank 1 appends none).  The mll and the predictions of the distributed FITC, DTC and SoR after each step must
equal those of a one-rank model built on the union within 1e-9 relative, the bound mgpu_worker.py holds alpha to."""
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
    N0, M, d = 4000, 120, 3
    steps = [(300, 200), (150, 0), (1, 700)]                    # new rows of rank 0 and of the other ranks per step
    N = N0 + sum(a + b * (world - 1) for a, b in steps)
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-1.5, 1.5, (M, d))
    xs = rng.standard_normal((200, d))
    ok = True
    for mode in ("FITC", "DTC", "SoR"):
        cls = getattr(gpb200, mode)
        lo, hi = rank * N0 // world, (rank + 1) * N0 // world
        gd = cls(X[lo:hi].T, Xu.T, y[lo:hi], gpb200.MeanConst(0.1), gpb200.SEIso(-0.4, 0.1), -1.0, device=local, distributed=True)
        seen = list(range(N0))
        r0 = N0
        for a, b in steps:
            counts = [a] + [b] * (world - 1)
            mine = np.arange(r0 + sum(counts[:rank]), r0 + sum(counts[:rank + 1]))
            gd.append(X[mine].T, y[mine])
            seen += list(range(r0, r0 + sum(counts)))
            r0 += sum(counts)
            gs = cls(X[seen].T, Xu.T, y[seen], gpb200.MeanConst(0.1), gpb200.SEIso(-0.4, 0.1), -1.0, device=local)
            md, ms = gd.predict_f(xs.T)[0], gs.predict_f(xs.T)[0]
            err_m = abs(gd.mll - gs.mll) / abs(gs.mll)
            err_p = np.max(np.abs(md - ms)) / np.max(np.abs(ms))
            m_ok = err_m <= 1e-9 and err_p <= 1e-9
            print("MGPU rank %d %s N=%d over %d ranks: mll rel err %.3e, mean %.3e -> %s" % (
                rank, mode, len(seen), world, err_m, err_p, "OK" if m_ok else "FAIL"), flush=True)
            t = torch.tensor([1.0 if m_ok else 0.0], dtype=torch.float64, device="cuda"); dist.all_reduce(t, op=dist.ReduceOp.MIN)
            ok = ok and t.item() > 0.5
            gs._eng.close()
        gd._eng.close()
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_RESULT", "PASS" if ok else "FAIL", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
