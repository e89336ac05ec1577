"""Worker for the multi-GPU training-input gradient test: torchrun --nproc-per-node R tests/mgpu_fitc_inputs_worker.py
Every rank holds its slice of the observations and the same Xu; the dmll/dX rows of the distributed FITC, DTC and SoR must
equal the matching rows of the single-GPU value on the full data set within 1e-9 relative (the bound mgpu_worker.py holds
alpha to, which they are linear in), and dmll/dXu within 1e-10.  The noise
and kernel entries and the mean entries (summed over the ranks) are held to mgpu_worker.py's rtol 1e-7, atol 1e-8."""
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
    rng = np.random.default_rng(92)
    N, M, d = 6000, 140, 3
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-1.5, 1.5, (M, d))
    kf = gpb200.SEArd([-0.4, -0.6, -0.5], 0.1) + gpb200.LinIso(0.5)
    lo, hi = rank * N // world, (rank + 1) * N // world
    ok = True
    for mode in ("FITC", "DTC", "SoR"):
        cls = getattr(gpb200, mode)
        gd = cls(X[lo:hi].T, Xu.T, y[lo:hi], gpb200.MeanLin([0.2, -0.1, 0.3]), kf, -1.0, device=local, distributed=True)
        gd.update_dmll(inducing=True, inputs=True)
        gs = cls(X.T, Xu.T, y, gpb200.MeanLin([0.2, -0.1, 0.3]), kf, -1.0, device=local)
        gs.update_dmll(inducing=True, inputs=True)
        nx, nu, nm = (hi - lo) * d, Xu.size, 3
        # [noise; mean (3); kernel; Xu; X]: the X rows are the rank's own; the mean-parameter gradient is a sum over the rank's
        # own rows (as in mgpu_worker.py), so the slices are added up before the comparison
        gx_d, gx_s = gd.dmll[-nx:], gs.dmll[-N * d:].reshape(N, d)[lo:hi].ravel()
        gu_d, gu_s = gd.dmll[-nx - nu:-nx], gs.dmll[-N * d - nu:-N * d]
        head_d, head_s = gd.dmll[:-nx - nu], gs.dmll[:-N * d - nu]
        tm = torch.tensor(head_d[1:1 + nm], dtype=torch.float64, device="cuda"); dist.all_reduce(tm)
        mean_d = tm.cpu().numpy()
        err_x = np.max(np.abs(gx_d - gx_s)) / np.max(np.abs(gx_s))
        err_u = np.max(np.abs(gu_d - gu_s)) / np.max(np.abs(gu_s))
        nk = np.r_[0, np.arange(1 + nm, head_s.size)]                   # noise and kernel entries
        # the X rows are linear in this rank's alpha, which mgpu_worker.py holds to 1e-9 of the single-GPU alpha
        m_ok = (head_d.size == head_s.size and err_x <= 1e-9 and err_u <= 1e-10
                and np.allclose(head_d[nk], head_s[nk], rtol=1e-7, atol=1e-8)
                and np.allclose(mean_d, head_s[1:1 + nm], rtol=1e-7, atol=1e-8))
        print("MGPU rank %d %s rows %d..%d over %d ranks: dmll/dX max rel err %.3e, dmll/dXu %.3e -> %s" % (
            rank, mode, lo, hi, world, err_x, err_u, "OK" if m_ok else "FAIL"), flush=True)
        t = torch.tensor([1.0 if m_ok else 0.0], dtype=torch.float64, device="cuda"); dist.all_reduce(t, op=dist.ReduceOp.MIN)
        ok = ok and t.item() > 0.5
        try:
            gd.optimize(inputs=True)
            ok = False
        except ValueError:
            pass
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("MGPU_RESULT", "PASS" if ok else "FAIL", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
