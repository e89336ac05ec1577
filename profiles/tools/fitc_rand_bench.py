"""Times posterior draws of the sparse engine (gpb200_fitc_rand, FITC mode 0):

  N = 10^6, d = 8, M = 4096 inducing points, SEIso; Ms in {4096, 16384, 32768} test points, nsamp in {16, 256} draws.

  python profiles/tools/fitc_rand_bench.py --out DIR [--n 1000000] [--m 4096] [--ms 4096,16384,32768] [--nsamp 16,256]
                                           [--repeats 3]

Per (Ms, nsamp): one warm-up call (it sizes the Ms x Ms sub-engine and the draw staging), then `--repeats` timed calls.
Reported per call: the host time (the call ends in a device synchronise, and includes the copies of z and the samples) and
the library's device-event split -- Sigma* build (cross-Gram, two whitening TRSMs, K** and the two NT GEMMs), make_posdef! +
Cholesky of Sigma* + nugget I, unwhiten! (one triangular NT GEMM) + mu -- as medians.  The flop counts beside them are the
algorithm's: Sigma* = K** - A A' + B B' with A, B = K*u L^-T is 2 Ms M^2 (TRSMs) + 4 Ms^2 M (two GEMMs), the Cholesky
Ms^3 / 3, unwhiten! nsamp Ms^2.  The library's in-run FP64 issue-rate probe (fp64_peak) is recorded beside the numbers, with
the card name and power limit read in the same run.  Writes DIR/h100_fitc_rand.json."""
import argparse, json, math, os, statistics, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--m", type=int, default=4096)
    ap.add_argument("--d", type=int, default=8)
    ap.add_argument("--ms", default="4096,16384,32768")
    ap.add_argument("--nsamp", default="16,256")
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
    res = {"card": card, "device": torch.cuda.get_device_name(0),
           "config": {"N": N, "M": M, "d": d, "kernel": "SEIso", "mode": "FITC", "nugget": 1e-6, "repeats": args.repeats}}
    e = FitcEngine(0)
    e.set_data(X, Xu)
    e.set_kernel(ops, dims, theta.size)
    e.factorize(theta, ln)
    e.mll(y)
    peak = gpb200.Engine(0).fp64_peak()
    rows = []
    for Ms in [int(v) for v in args.ms.split(",")]:
        xs = rng.uniform(-2.0, 2.0, (Ms, d))
        for ns in [int(v) for v in args.nsamp.split(",")]:
            z = rng.standard_normal((ns, Ms))
            e.rand(xs, z, nugget=1e-6)
            host, split = [], []
            for _ in range(args.repeats):
                t0 = time.perf_counter()
                e.rand(xs, z, nugget=1e-6)
                host.append((time.perf_counter() - t0) * 1e3)
                split.append(e.rand_timings().tolist())
            med = [statistics.median(s[i] for s in split) for i in range(3)]
            fl = {"sigma_build": 2.0 * Ms * M * M + 4.0 * Ms * Ms * M, "cholesky": Ms ** 3 / 3.0, "unwhiten": float(ns) * Ms * Ms}
            row = {"Ms": Ms, "nsamp": ns, "host_ms": host, "host_ms_median": statistics.median(host),
                   "sigma_build_ms": med[0], "cholesky_ms": med[1], "unwhiten_ms": med[2], "flops": fl,
                   "tflops": {k: fl[k] / (ms * 1e-3) * 1e-12 for k, ms in zip(("sigma_build", "cholesky", "unwhiten"), med)}}
            rows.append(row)
            print("Ms %6d nsamp %4d: host %9.1f ms | Sigma* %8.1f ms (%5.1f TFLOP/s)  Cholesky %8.1f ms (%5.1f TFLOP/s)  "
                  "unwhiten %7.1f ms (%5.1f TFLOP/s)" % (Ms, ns, row["host_ms_median"], med[0], row["tflops"]["sigma_build"], med[1],
                                                          row["tflops"]["cholesky"], med[2], row["tflops"]["unwhiten"]), flush=True)
    res["runs"] = rows
    res["fp64_peak"] = peak
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_fitc_rand.json"), "w") as f:
        json.dump(res, f, indent=1)
    e.close()


if __name__ == "__main__":
    main()
