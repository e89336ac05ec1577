"""Times cross-validation on the sparse engine (FITC, mode 0) next to the kernel gradient on the same handle:

  N = 10^6, d = 8, M = 4096 inducing points, SEIso; inverse_diag, cv_param for every parameter (noise and the two SEIso
  parameters) and a sweep of cv_block over 64 folds (which = 0 and which = 1), next to factorize / mll / grad_kernel.

  python profiles/tools/fitc_cv_bench.py --out DIR [--n 1000000] [--m 4096] [--folds 64] [--repeats 3]

Every library call ends in a device synchronise, so a host clock around it times the device work.  Per phase: one warm-up
call, then `--repeats` timed calls.  The per-parameter time is compared with the flop count of the schedule's DMMA GEMMs:
pass 1 runs C = K_fu K_uu^-1, G = dK_fu - 1/2 K_fu Dp, R += K_uf L^-1 G and H += K_uf L^-1 Delta L^-1 K_fu, pass 2 runs
G again, K_fu S^-1 and Ch Q: seven N x M x M products, 14 N M^2 flop per FITC kernel parameter (the noise direction has
G = 0 and runs H, K_fu S^-1 and Ch Q only: 6 N M^2).  The library's in-run FP64 issue-rate probe (fp64_peak) is recorded
beside the numbers, with the card name and power limit read in the same run.  Writes DIR/h100_fitc_cv.json."""
import argparse, json, math, os, statistics, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))


def timed(fn, repeats):
    fn()
    out = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return {"ms": out, "ms_median": statistics.median(out)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--m", type=int, default=4096)
    ap.add_argument("--d", type=int, default=8)
    ap.add_argument("--folds", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    import gpb200
    from gpb200.capi import FitcEngine
    from gpb200.kernels import flatten

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(0)
    N, M, d = args.n, args.m, args.d
    X = rng.uniform(-2.0, 2.0, (N, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.choice(N, M, replace=False)]
    kern = gpb200.SEIso(math.log(0.8), 0.0)
    ops, dims, theta, _ = flatten(kern, d)
    ln = -1.0
    folds = np.array_split(rng.permutation(N), args.folds)
    Mpad = -(-M // 128) * 128
    res = {"card": card, "device": torch.cuda.get_device_name(0), "config": {"N": N, "M": M, "d": d, "kernel": "SEIso",
           "mode": "FITC", "folds": args.folds, "fold_size": int(folds[0].size), "repeats": args.repeats}}
    e = FitcEngine(0)
    e.set_data(X, Xu)
    e.set_kernel(ops, dims, theta.size)
    r = {"factorize": timed(lambda: e.factorize(theta, ln), args.repeats)}
    r["mll"] = timed(lambda: e.mll(y), args.repeats)
    r["grad_kernel"] = timed(lambda: e.grad_kernel(), args.repeats)
    r["inverse_diag"] = timed(lambda: e.inverse_diag(), args.repeats)
    for p in [-1] + list(range(theta.size)):
        r["cv_param[%d]" % p] = timed(lambda: e.cv_param(p), args.repeats)
    def sweep(which):                                              # one fold block at a time: each is |V|^2 doubles on the host
        for V in folds:
            e.cv_block(which, V)
    r["cv_block_sweep_which0"] = timed(lambda: sweep(0), 1)
    e.cv_param(0)
    r["cv_block_sweep_which1"] = timed(lambda: sweep(1), 1)
    for k, v in r.items():
        print("%-22s %10.1f ms" % (k, v["ms_median"]), flush=True)
    peak = gpb200.Engine(0).fp64_peak()
    est = {}
    for p in [-1] + list(range(theta.size)):
        fl = (6.0 if p < 0 else 14.0) * N * Mpad * Mpad
        ms = r["cv_param[%d]" % p]["ms_median"]
        est["cv_param[%d]" % p] = {"gemm_flops": fl, "tflops_effective": fl / (ms * 1e-3) * 1e-12,
                                   "share_of_dmma_peak": fl / (ms * 1e-3) * 1e-12 / peak["dmma_tflops"],
                                   "estimate_9NM2_ms_at_peak": 9.0 * N * M * M / (peak["dmma_tflops"] * 1e12) * 1e3}
        print("cv_param[%d]: %.1f ms, %.1f TFLOP/s effective over the GEMM flops (%.0f%% of DMMA peak %.1f)"
              % (p, ms, est["cv_param[%d]" % p]["tflops_effective"], 100 * est["cv_param[%d]" % p]["share_of_dmma_peak"],
                 peak["dmma_tflops"]), flush=True)
    res["phases"] = r
    res["cv_param_vs_gemm_flops"] = est
    res["fp64_peak"] = peak
    res["cv_param_over_grad_kernel"] = r["cv_param[0]"]["ms_median"] / r["grad_kernel"]["ms_median"]
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_fitc_cv.json"), "w") as f:
        json.dump(res, f, indent=1)
    e.close()


if __name__ == "__main__":
    main()
