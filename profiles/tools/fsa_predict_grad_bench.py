"""Times FSA's predictive gradients (predict_fsa_grad) against the predictions alone (predict_fsa) on the same inputs:

  N = 10^6, d = 8, M = 4096 inducing points, SEIso, training blocks = consecutive runs of 512 points in the order of a 1-D
  projection of x (fsa_bench.py's setup), and three sets of test points:
    1. 4096 points, two per training block (four on the first 94 of the 1954 blocks; every test tile padded from 2 or 4
       to 128 rows: the worst case)
    2. 4096 points in 32 blocks (128 per block)
    3. 128 points in one block

  python profiles/tools/fsa_predict_grad_bench.py --out DIR [--n 1000000] [--m 4096] [--repeats 3]

Every library call ends in a device synchronise, so a host clock around it times the device work.  Per case: one warm-up
call of each, then `--repeats` rounds alternating predict_fsa and predict_fsa_grad; medians are reported, with the
device-event split of the gradient call (gpb200_fitc_get_timings slots 3-6) of its last timed call.  The card name and
power limit are read in the same run.  Writes DIR/h100_fsa_predict_grad.json."""
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
    ap.add_argument("--block", type=int, default=512)
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
    proj = X @ rng.standard_normal(d)
    order = np.argsort(proj, kind="stable")
    blocks = [order[i:i + args.block] for i in range(0, N, args.block)]
    nb = len(blocks)
    block_ptr = np.concatenate([[0], np.cumsum([b.size for b in blocks])]).astype(np.int64)
    kern = gpb200.SEIso(math.log(0.8), 0.0)
    ops, dims, theta, _ = flatten(kern, d)
    e = FitcEngine(0)
    e.set_mode(3)
    e.set_data(X, Xu)
    e.set_kernel(ops, dims, theta.size)
    e.set_blocks(block_ptr, np.concatenate(blocks))
    e.factorize(theta, -1.0)
    e.mll(y)

    def near(b, k):                                           # k test points near the inputs of training block b
        return X[blocks[b][rng.choice(blocks[b].size, k, replace=False)]] + 0.01 * rng.standard_normal((k, d))

    c1 = [b % nb for b in range(2048)]                         # N = 10^6: 1954 blocks, 94 of them get four points
    c2 = [b * (nb // 32) for b in range(32)]
    cases = {
        "4096 points, 2 per block": (np.vstack([near(b, 2) for b in c1]), np.repeat(c1, 2)),
        "4096 points in 32 blocks": (np.vstack([near(b, 128) for b in c2]), np.repeat(c2, 128)),
        "128 points in 1 block": (near(nb // 2, 128), np.full(128, nb // 2)),
    }
    res = {"card": card, "device": torch.cuda.get_device_name(0),
           "config": {"N": N, "M": M, "d": d, "kernel": "SEIso", "block": args.block, "nblocks": nb, "repeats": args.repeats},
           "cases": {}}
    for name, (Xs, bo) in cases.items():
        Xs = np.ascontiguousarray(Xs)
        bo = np.ascontiguousarray(bo, dtype=np.int64)
        e.predict_fsa(Xs, bo)
        e.predict_fsa_grad(Xs, bo)
        tp, tg = [], []
        for _ in range(args.repeats):
            t0 = time.perf_counter(); e.predict_fsa(Xs, bo); tp.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter(); e.predict_fsa_grad(Xs, bo); tg.append((time.perf_counter() - t0) * 1e3)
        split = e.predict_fsa_grad_timings()
        r = {"ntest": int(Xs.shape[0]), "paired_blocks": int(np.unique(bo).size),
             "predict_fsa_ms": tp, "predict_fsa_grad_ms": tg,
             "predict_fsa_ms_median": statistics.median(tp), "predict_fsa_grad_ms_median": statistics.median(tg),
             "ratio": statistics.median(tg) / statistics.median(tp),
             "grad_split_ms": {"predict_fsa_launches": split[0], "s_and_second_sweep": split[1],
                               "kuu_trsms": split[2], "contraction": split[3]}}
        res["cases"][name] = r
        print("%-26s predict_fsa %9.1f ms  predict_fsa_grad %9.1f ms  ratio %.2f  split %s"
              % (name, r["predict_fsa_ms_median"], r["predict_fsa_grad_ms_median"], r["ratio"],
                 np.array2string(split, precision=1)), flush=True)
    e.close()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_fsa_predict_grad.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(card)


if __name__ == "__main__":
    main()
