"""Times the Full Scale Approximation (sparse engine mode 3) against FITC on the same data, and the grouped tile GEMM that
carries FSA's block-diagonal work:

  N = 10^6, d = 8, M = 4096 inducing points, SEIso; training blocks = consecutive runs of 512 points in the order of a
  1-D projection of x; a 4096-point predict_fsa whose test points are paired with the block of their projection.

  python profiles/tools/fsa_bench.py --out DIR [--n 1000000] [--m 4096] [--block 512] [--repeats 3]

Every library call ends in a device synchronise, so a host clock around it times the device work.  Per phase: one warm-up
call, then `--repeats` timed calls.  A separate torch.profiler pass over one FSA factorize sums the device time of the
grouped GEMM (fsa_gemm_kernel); its flops are computed here from the block sizes (2 * 128 * 128 * K per work item, the
same lists gpb200_fitc_set_blocks builds) and compared with the library's in-run FP64 issue-rate probe (fp64_peak).
Writes DIR/h100_fsa.json with the card name and power limit read in the same run."""
import argparse, json, math, os, statistics, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))


def grouped_gemm_flops_factorize(sizes, Mpad):
    """flops of the grouped-GEMM items of one FSA factorize (Schur term, batched Cholesky + inverse, W')"""
    items_k = 0
    for b in sizes:
        T = -(-b // 128)
        items_k += T * (T + 1) // 2 * Mpad                                   # Lambda_i -= V_i V_i'
        for k in range(T):
            items_k += (T - 1 - k) * 128                                     # panel
            items_k += (T - 1 - k) * (T - k) // 2 * 128                      # trailing update
            items_k += sum((k - j) * 128 for j in range(k))                  # inverse: T'
            items_k += 2 * k * 128                                           # inverse: X_kj and X_jk'
        items_k += (Mpad // 128) * sum((r + 1) * 128 for r in range(T))      # W' = K_uf X'
    return 2.0 * 128 * 128 * items_k


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
    ap.add_argument("--block", type=int, default=512)
    ap.add_argument("--ntest", type=int, default=4096)
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
    w = rng.standard_normal(d)
    proj = X @ w
    order = np.argsort(proj, kind="stable")
    blocks = [order[i:i + args.block] for i in range(0, N, args.block)]
    sizes = [b.size for b in blocks]
    block_ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    Xs = rng.uniform(-2.0, 2.0, (args.ntest, d))
    edges = proj[order[block_ptr[1:-1]]]                                      # first projection value of blocks 1..
    block_of = np.searchsorted(edges, Xs @ w, side="right").astype(np.int64)
    kern = gpb200.SEIso(math.log(0.8), 0.0)
    ops, dims, theta, _ = flatten(kern, d)
    ln = -1.0
    res = {"card": card, "device": torch.cuda.get_device_name(0), "config": {"N": N, "M": M, "d": d, "kernel": "SEIso",
           "block": args.block, "nblocks": len(blocks), "ntest": args.ntest, "repeats": args.repeats}}

    def engine(mode):
        e = FitcEngine(0)
        e.set_mode(mode)
        e.set_data(X, Xu)
        e.set_kernel(ops, dims, theta.size)
        return e

    phases = {}
    for name, mode in (("fsa", 3), ("fitc", 0)):
        e = engine(mode)
        if mode == 3:
            t0 = time.perf_counter()
            e.set_blocks(block_ptr, np.concatenate(blocks))
            phases["fsa_set_blocks_ms"] = (time.perf_counter() - t0) * 1e3
        r = {"factorize": timed(lambda: e.factorize(theta, ln), args.repeats)}
        r["mll"] = timed(lambda: e.mll(y), args.repeats)
        r["grad_noise"] = timed(lambda: e.grad_noise(), args.repeats)
        r["grad_kernel"] = timed(lambda: e.grad_kernel(), args.repeats)
        if mode == 3:
            r["predict_fsa"] = timed(lambda: e.predict_fsa(Xs, block_of), args.repeats)
        else:
            r["predict"] = timed(lambda: e.predict(Xs), args.repeats)
        for k, v in r.items():
            print("%-4s %-12s %10.1f ms" % (name, k, v["ms_median"]), flush=True)
        phases[name] = r
        if mode == 3:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                e.factorize(theta, ln)
            us = sum(ev.device_time_total for ev in prof.key_averages() if "fsa_gemm_kernel" in ev.key)
            n = sum(ev.count for ev in prof.key_averages() if "fsa_gemm_kernel" in ev.key)
            fl = grouped_gemm_flops_factorize(sizes, -(-M // 128) * 128)
            phases["grouped_gemm_factorize"] = {"launches": n, "device_ms": us * 1e-3, "flops": fl,
                                                "tflops": fl / (us * 1e-6) * 1e-12 if us else None}
            print("grouped GEMM in one factorize: %d launches, %.1f ms, %.2f TFLOP/s"
                  % (n, us * 1e-3, phases["grouped_gemm_factorize"]["tflops"] or 0.0), flush=True)
        e.close()
        del e
    step = lambda p: sum(p[k]["ms_median"] for k in ("factorize", "mll", "grad_noise", "grad_kernel"))
    phases["fsa_over_fitc_mll_and_gradient"] = step(phases["fsa"]) / step(phases["fitc"])
    peak = gpb200.Engine(0).fp64_peak()
    phases["fp64_peak"] = peak
    gg = phases["grouped_gemm_factorize"]
    if gg["tflops"]:
        gg["share_of_dmma_peak"] = gg["tflops"] / peak["dmma_tflops"]
    res["phases"] = phases
    print("FSA / FITC (factorize + mll + gradients): %.2f ; fp64_peak DMMA %.1f TFLOP/s"
          % (phases["fsa_over_fitc_mll_and_gradient"], peak["dmma_tflops"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_fsa.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
