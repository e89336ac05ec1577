"""Times one GPA step (update_target_and_dtarget of a Bernoulli GPA) against the GPE step (update_target_and_dtarget) on
the same inputs, alternating the two in one call:

  N = 32768, d = 8, kernel SEIso + Noise, MeanConst; GPA: BernLik, logNoise = -20 (GPA.jl:111-114); GPE: logNoise = -1.

  python profiles/tools/gpa_bench.py --out DIR [--n 32768] [--repeats 3]

Every library call ends in a device synchronise, so a host clock around a step times the device work plus the O(N) host
likelihood.  The per-phase device times come from the engine's CUDA events (gpb200_get_timings): Gram, Cholesky, the
inverse merges, the scans, the S = W'Z GEMM and the trace.  The S GEMM's rate counts N^3/3 flop and is compared with the
library's in-run FP64 issue-rate probe (fp64_peak).  Both steps do N^3 flop (GPE: Cholesky + merges + W'W; GPA: Cholesky +
merges + W'Z).  Writes DIR/h100_gpa.json with the card name and power limit read in the same run."""
import argparse, json, math, os, statistics, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=32768)
    ap.add_argument("--d", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    import gpb200 as g

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(0)
    N, d = args.n, args.d
    X = 2 * np.pi * rng.random((N, d))
    f = np.sin(X).sum(axis=1) / d
    y = rng.random(N) < np.abs(f)
    kern = lambda: g.SEIso(math.log(1.5), 0.0) + g.Noise(-1.0)
    gpa = g.GPA(X.T, y, g.MeanConst(0.1), kern(), g.BernLik())
    p = gpa.get_params()
    p[:N] = 0.5 * rng.standard_normal(N)
    gpa.set_params(p)
    gpe = g.GPE(X.T, y.astype(np.float64), g.MeanConst(0.1), kern(), -1.0)
    steps = {"gpa": gpa.update_target_and_dtarget, "gpe": gpe.update_target_and_dtarget}
    for fn in steps.values():                                        # warm-up
        fn()
    times = {k: [] for k in steps}
    phases = {k: [] for k in steps}
    for _ in range(args.repeats):
        for name, fn in steps.items():
            t0 = time.perf_counter()
            fn()
            times[name].append((time.perf_counter() - t0) * 1e3)
            t = (gpa if name == "gpa" else gpe)._eng.timings()
            ph = dict(gram=t["gram"], cholesky=t["cholesky"], merges=t["inverse"], trace=t["trace"])
            if name == "gpa":
                ph.update(scan=t["gpa_scan"], s_gemm=t["gpa_product"])
            else:
                ph["inverse_incl_WtW"] = ph.pop("merges")
            phases[name].append(ph)
            print("%s step %9.1f ms  %s" % (name, times[name][-1], "  ".join("%s %.2f" % kv for kv in ph.items())), flush=True)
    peak = g.Engine(0).fp64_peak()
    s_ms = statistics.median(ph["s_gemm"] for ph in phases["gpa"])
    s_tflops = N ** 3 / 3.0 / (s_ms * 1e-3) * 1e-12
    res = {"card": card, "device": torch.cuda.get_device_name(0),
           "config": {"N": N, "d": d, "kernel": "SEIso + Noise", "mean": "MeanConst", "lik": "BernLik", "repeats": args.repeats},
           "step_ms": times, "step_ms_median": {k: statistics.median(v) for k, v in times.items()},
           "phases_ms": phases, "s_gemm": {"ms_median": s_ms, "flop": N ** 3 / 3.0, "tflops": s_tflops,
                                           "share_of_dmma_peak": s_tflops / peak["dmma_tflops"]},
           "fp64_peak": peak, "algorithmic_flop_per_step": float(N) ** 3}
    print("GPA %.1f ms, GPE %.1f ms; S GEMM %.2f ms = %.1f TFLOP/s = %.2f of the in-run DMMA peak (%.1f)"
          % (res["step_ms_median"]["gpa"], res["step_ms_median"]["gpe"], s_ms, s_tflops, s_tflops / peak["dmma_tflops"],
             peak["dmma_tflops"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_gpa.json"), "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
