"""Times append on the sparse engine against a refit of the grown data:

  FITC, SEIso, d = 8, N0 = 10^6 rows, M = 4096 inducing points; k in {1, 128, 4096} new rows

  python profiles/tools/fitc_append_bench.py --out DIR [--n 1000000] [--m 4096] [--repeats 3]

Per k and round, alternated after a warm-up of both: the append handle is reset to the N0 rows (set_data + factorize + mll,
not timed), then `append` of k rows + `predict` of 4096 points is timed, then a second append of k more rows + predict (the
first append after a factorize also rebuilds Sigma_QR as L_s L_s' and sums r'Lambda^-1 r and log Lambda over every row; the
second does neither; the predict after it is also timed alone).  The refit handle holds the N0 + k rows (set_data not timed) and times factorize + mll + predict.
Every library call ends in a device synchronise, so a host clock around it times the device work.  Medians of the rounds
with the spread; the card name and power limit are read in the same run.  Writes DIR/h100_fitc_append.json."""
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
    ap.add_argument("--ks", default="1,128,4096")
    ap.add_argument("--npred", type=int, default=4096)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    import gpb200
    from gpb200.capi import FitcEngine
    from gpb200.kernels import flatten

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    ks = [int(v) for v in args.ks.split(",")]
    rng = np.random.default_rng(0)
    N0, M, d = args.n, args.m, args.d
    X = rng.uniform(-2.0, 2.0, (N0 + 2 * max(ks), d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(X.shape[0])
    Xu = X[rng.choice(N0, M, replace=False)]
    xs = rng.uniform(-2.0, 2.0, (args.npred, d))
    ops, dims, theta, _ = flatten(gpb200.SEIso(math.log(0.8), 0.0), d)
    ln = -1.0

    def engine(n):
        e = FitcEngine(0)
        e.set_mode(0)
        e.set_data(X[:n], Xu)
        e.set_kernel(ops, dims, theta.size)
        return e

    def clock(fn):
        t0 = time.perf_counter(); out = fn(); return (time.perf_counter() - t0) * 1e3, out

    res = {"card": card, "device": torch.cuda.get_device_name(0),
           "config": {"strategy": "FITC", "N0": N0, "M": M, "d": d, "kernel": "SEIso", "npred": args.npred,
                      "repeats": args.repeats}, "k": {}}
    ea = engine(N0)
    for k in ks:
        eb = engine(N0 + k)
        t1, t2, tr, tps, mll_a, mll_b = [], [], [], [], None, None
        for rnd in range(args.repeats + 1):                             # round 0 is the warm-up
            ea.set_data(X[:N0], Xu)
            ea.factorize(theta, ln)
            ea.mll(y[:N0])
            ta, (mll_a, _) = clock(lambda: ea.append(X[N0:N0 + k], y[N0:N0 + k]))
            ta += clock(lambda: ea.predict(xs))[0]
            tb, _ = clock(lambda: ea.append(X[N0 + k:N0 + 2 * k], y[N0 + k:N0 + 2 * k]))
            tp = clock(lambda: ea.predict(xs))[0]
            tb += tp

            def refit():
                eb.factorize(theta, ln)
                return eb.mll(y[:N0 + k])[1]
            tc, mll_b = clock(refit)
            tc += clock(lambda: eb.predict(xs))[0]
            if rnd:
                t1.append(ta); t2.append(tb); tr.append(tc); tps.append(tp)
        eb.close()
        r = {"first_append_predict_ms": t1, "second_append_predict_ms": t2, "refit_predict_ms": tr,
             "first_append_predict_ms_median": statistics.median(t1), "second_append_predict_ms_median": statistics.median(t2),
             "refit_predict_ms_median": statistics.median(tr), "predict_ms": tps, "predict_ms_median": statistics.median(tps), "refit_over_first_append": statistics.median(tr) / statistics.median(t1),
             "mll_append": mll_a, "mll_refit": mll_b, "mll_rel_diff": abs(mll_a - mll_b) / abs(mll_b)}
        res["k"][str(k)] = r
        print("k=%5d  append+predict first %8.1f ms  second %8.1f ms  refit+predict %8.1f ms  predict %6.1f ms  (spread %.1f / %.1f / %.1f)  mll rel diff %.1e"
              % (k, r["first_append_predict_ms_median"], r["second_append_predict_ms_median"], r["refit_predict_ms_median"], r["predict_ms_median"],
                 max(t1) - min(t1), max(t2) - min(t2), max(tr) - min(tr), r["mll_rel_diff"]), flush=True)
    ea.close()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_fitc_append.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(card)


if __name__ == "__main__":
    main()
