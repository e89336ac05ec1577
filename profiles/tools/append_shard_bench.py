"""Times ElasticGPE append! on row-sharded storage against a refit of the same group and against the single-GPU append, on
one GPU (the group's ranks are virtual ranks of gpb200_group_create sharing the device):

  N0 in {16384, 32768}, k in {1, 64, 1024}, groups R in {2, 4} (ownership block chosen by the engine), d = 8,
  kernel SEIso, logNoise = -1, capacity N0 + 1024.

  python profiles/tools/append_shard_bench.py --out DIR [--n0 16384 32768] [--repeats 3]

Per (N0, R, k) and repeat, three timed calls alternate: `append` = gpb200_append of k points onto the factor of N0 points, then
mll on the N0 + k targets (the group); `refit` = factorize + mll of the same N0 + k points on the same group; `single` = the
single-GPU append + mll.  The untimed set_data / factorize that restore the N0-point factor run before each timed call.
Every library call ends in a device synchronise, so a host clock around the calls times the device work.  Writes
DIR/h100_append_shard.json with the card name, power limit and clocks read in the same run."""
import argparse, json, math, os, statistics, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))

KS = (1, 64, 1024)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n0", type=int, nargs="+", default=[16384, 32768])
    ap.add_argument("--groups", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--d", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    import gpb200 as g

    def smi():
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    card_before = smi()
    d, ln = args.d, -1.0
    kern = g.SEIso(math.log(1.5), 0.0)
    rows = []
    for N0 in args.n0:
        rng = np.random.default_rng(N0)
        Nt = N0 + max(KS)
        X = 2 * np.pi * rng.random((Nt, d))
        y = np.sin(X).sum(axis=1) / d + 0.1 * rng.standard_normal(Nt)
        for R in args.groups:
            engines = {"group": g.LocalGroupEngine(R), "single": g.Engine(0)}
            for e in engines.values():
                gp = g.GPE(X[:N0].T, y[:N0], g.MeanZero(), kern, ln, capacity=Nt, engine=e)      # builds data + kernel program
                th = gp._theta_full()
                del gp
            info = engines["group"].engines[0].storage_info()

            def restore(e, n):
                e.set_data(X[:n])
                e.factorize(th, ln)

            def timed(fn):
                t0 = time.perf_counter()
                fn()
                return (time.perf_counter() - t0) * 1e3

            for k in KS:
                calls = {
                    "append": (lambda: restore(engines["group"], N0),
                               lambda: (engines["group"].append(X[N0:N0 + k]), engines["group"].mll(y[:N0 + k]))),
                    "refit": (lambda: engines["group"].set_data(X[:N0 + k]),
                              lambda: (engines["group"].factorize(th, ln), engines["group"].mll(y[:N0 + k]))),
                    "single": (lambda: restore(engines["single"], N0),
                               lambda: (engines["single"].append(X[N0:N0 + k]), engines["single"].mll(y[:N0 + k]))),
                }
                for prep, fn in calls.values():                     # warm-up of every shape
                    prep(); fn()
                ms = {name: [] for name in calls}
                mll = {}
                for _ in range(args.repeats):
                    for name, (prep, fn) in calls.items():
                        prep()
                        ms[name].append(timed(fn))
                        e = engines["group"] if name != "single" else engines["single"]
                        mll[name] = e.mll(y[:N0 + k])[1]
                med = {name: statistics.median(v) for name, v in ms.items()}
                row = {"N0": N0, "R": R, "rb": info["rb"], "k": k, "ms": ms, "ms_median": med,
                       "refit_over_append": med["refit"] / med["append"], "single_over_append": med["single"] / med["append"],
                       "mll": mll}
                rows.append(row)
                print("N0 %6d R %d rb %d k %5d: append+mll %8.1f ms  refit+mll %8.1f ms  single-GPU append+mll %8.1f ms  (x%.1f)"
                      % (N0, R, info["rb"], k, med["append"], med["refit"], med["single"], med["refit"] / med["append"]), flush=True)
            for e in engines.values():
                e.close()
            torch.cuda.empty_cache()
    res = {"card_before": card_before, "card_after": smi(), "device": torch.cuda.get_device_name(0),
           "config": {"d": d, "kernel": "SEIso", "logNoise": ln, "capacity": "N0 + %d" % max(KS), "repeats": args.repeats,
                      "group": "gpb200_group_create: R virtual ranks on the one device"},
           "rows": rows}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_append_shard.json"), "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
