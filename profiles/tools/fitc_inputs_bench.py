"""Times the joint kernel + training-input gradient (grad_kernel_inputs) against the kernel gradient alone (grad_kernel)
on the same handle:

  N = 10^6, d = 8, M = 4096 inducing points, SEIso;  FITC, and FSA on the same data with training blocks = consecutive
  runs of 512 points in the order of a 1-D projection of x (fsa_bench.py's setup)

  python profiles/tools/fitc_inputs_bench.py --out DIR [--n 1000000] [--m 4096] [--repeats 3]

Every library call ends in a device synchronise, so a host clock around it times the device work.  Per strategy: one
warm-up call of each, then `--repeats` rounds alternating grad_kernel and grad_kernel_inputs; medians are reported with
the spread, and the X contractions' own device time (gpb200_fitc_get_timings slot 9, summed over their launches: one row
contraction per staging chunk, FSA also one block contraction) and the joint call's device time (slot 10) of every timed
joint call.  The card name and power limit are read in the same run.  Writes DIR/h100_fitc_inputs.json."""
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
    order = np.argsort(X @ rng.standard_normal(d), kind="stable")
    blocks = [order[i:i + args.block] for i in range(0, N, args.block)]
    block_ptr = np.concatenate([[0], np.cumsum([b.size for b in blocks])]).astype(np.int64)
    ops, dims, theta, _ = flatten(gpb200.SEIso(math.log(0.8), 0.0), d)
    res = {"card": card, "device": torch.cuda.get_device_name(0),
           "config": {"N": N, "M": M, "d": d, "kernel": "SEIso", "fsa_block": args.block, "repeats": args.repeats},
           "strategies": {}}
    for name, mode in (("FITC", 0), ("FSA", 3)):
        e = FitcEngine(0)
        e.set_mode(mode)
        e.set_data(X, Xu)
        e.set_kernel(ops, dims, theta.size)
        if mode == 3:
            e.set_blocks(block_ptr, np.concatenate(blocks))
        e.factorize(theta, -1.0)
        e.mll(y)
        gk = e.grad_kernel()
        gk2, _, _ = e.grad_kernel_inputs()
        assert np.array_equal(gk, gk2)
        tk, tj, tc, tcall = [], [], [], []
        for _ in range(args.repeats):
            t0 = time.perf_counter(); e.grad_kernel(); tk.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter(); e.grad_kernel_inputs(); tj.append((time.perf_counter() - t0) * 1e3)
            c, call = e.grad_inputs_timings()
            tc.append(float(c)); tcall.append(float(call))
        mk, mj, mc = statistics.median(tk), statistics.median(tj), statistics.median(tc)
        r = {"grad_kernel_ms": tk, "grad_kernel_inputs_ms": tj, "contraction_ms": tc, "joint_call_device_ms": tcall,
             "grad_kernel_ms_median": mk, "grad_kernel_inputs_ms_median": mj, "contraction_ms_median": mc,
             "grad_kernel_spread_ms": max(tk) - min(tk), "grad_kernel_inputs_spread_ms": max(tj) - min(tj),
             "joint_minus_kernel_ms": mj - mk, "joint_minus_kernel_minus_contraction_ms": mj - mk - mc,
             "contraction_derivative_evals_per_s": N * M / (mc * 1e-3)}
        res["strategies"][name] = r
        print("%-5s grad_kernel %8.1f ms  joint %8.1f ms  contraction %7.1f ms  joint - kernel - contraction %+6.1f ms  (spread %.1f / %.1f)"
              % (name, mk, mj, mc, mj - mk - mc, r["grad_kernel_spread_ms"], r["grad_kernel_inputs_spread_ms"]), flush=True)
        e.close()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_fitc_inputs.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(card)


if __name__ == "__main__":
    main()
