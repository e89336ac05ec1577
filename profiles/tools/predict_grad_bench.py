"""Times predictive gradients (gpb200_predict_grad) against plain predictions (gpb200_predict) on the same handle:

  N = 32768, d = 8: SEIso at M in {128, 4096}; Mat32Iso + RQIso (the generic kernel program) at M = 4096.

  python profiles/tools/predict_grad_bench.py --out DIR [--n 32768] [--repeats 3]

Per case: one warm-up call of each, then `--repeats` rounds alternating predict and predict_grad; medians of the host times
(each call ends in a device synchronise).  The library's device-event split of predict_grad is recorded: cross-Gram + mean,
V' = K*' L^-T + variance, L' into F's upper tiles, W' = V' L^-1, gradient contraction.  Each TRSM's rate is 2 N^2 Mpad / 2
= N^2 Mpad flop (a triangular solve of Mpad right-hand sides) over its device time, beside the in-run FP64 probe (fp64_peak),
with the card name and power limit read in the same run.  Writes DIR/h100_predict_grad.json."""
import argparse, json, math, os, statistics, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))

CASES = [("SEIso", 8, 128), ("SEIso", 8, 4096), ("Mat32Iso+RQIso", 8, 4096)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=32768)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    import gpb200

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(0)
    N = args.n
    res = {"card": card, "device": torch.cuda.get_device_name(0), "config": {"N": N, "repeats": args.repeats}}
    rows, gps = [], {}
    for kname, d, M in CASES:
        if (kname, d) not in gps:
            X = rng.uniform(-2.0, 2.0, (N, d))
            y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
            kern = gpb200.SEIso(math.log(0.8), 0.0) if kname == "SEIso" else gpb200.Mat32Iso(0.2, 0.0) + gpb200.RQIso(0.4, -0.3, 0.1)
            gps[(kname, d)] = gpb200.GPE(X.T, y, gpb200.MeanZero(), kern, -1.0)
        e = gps[(kname, d)]._eng
        xs = rng.uniform(-2.0, 2.0, (M, d))
        e.predict(xs)
        e.predict_grad(xs)
        tp, tg, split = [], [], []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            e.predict(xs)
            tp.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            e.predict_grad(xs)
            tg.append((time.perf_counter() - t0) * 1e3)
            t = e.timings()
            split.append([t["pgrad_crossgram"], t["pgrad_trsm"], t["pgrad_transpose"], t["pgrad_trsm_right"], t["pgrad_contract"]])
        med = [statistics.median(s[i] for s in split) for i in range(5)]
        Mpad = (M + 127) // 128 * 128
        Npad = (N + 127) // 128 * 128
        trsm_flop = float(Npad) * Npad * Mpad
        row = {"kernel": kname, "d": d, "M": M, "predict_ms": tp, "predict_grad_ms": tg,
               "predict_ms_median": statistics.median(tp), "predict_grad_ms_median": statistics.median(tg),
               "split_ms": dict(zip(("crossgram_mean", "trsm_variance", "transpose", "trsm_right", "contraction"), med)),
               "trsm_tflops": trsm_flop / (med[1] * 1e-3) * 1e-12, "trsm_right_tflops": trsm_flop / (med[3] * 1e-3) * 1e-12}
        rows.append(row)
        print("%-15s d=%d M=%5d: predict %8.1f ms  predict_grad %8.1f ms | split %s | TRSM %.1f / %.1f TFLOP/s" % (
            kname, d, M, row["predict_ms_median"], row["predict_grad_ms_median"],
            " ".join("%.1f" % v for v in med), row["trsm_tflops"], row["trsm_right_tflops"]), flush=True)
    res["runs"] = rows
    res["fp64_peak"] = gpb200.Engine(0).fp64_peak()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_predict_grad.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
