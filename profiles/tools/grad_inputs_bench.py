"""Times the training-input gradient (gpb200_grad_inputs) against the kernel gradient (gpb200_grad_kernel) on the same
resident K^-1:

  SEIso, N = 32768, d = 8: grad_kernel, grad_inputs through the SEIso specialisation, and through the kernel program
    (option "gram_fast" = 0)
  Mat32Iso + RQIso, N = 32768, d = 8: grad_kernel and grad_inputs (kernel program)
  SEIso, N = 16384, d = 8 on a row-sharded in-process group of 4 virtual ranks on the one GPU

  python profiles/tools/grad_inputs_bench.py --out DIR [--n 32768] [--n-group 16384] [--repeats 3]

Every library call ends in a device synchronise; the device times are the calls' own CUDA events (gpb200_get_timings slot 4
for the trace, slot 16 for grad_inputs).  Per case: one warm-up call of each variant, then `--repeats` rounds alternating
the variants; medians are reported with the spread.  grad_inputs reads every stored entry of the lower triangle twice, so
its bytes are 2 * 8 * N (N + 1) / 2; the HBM bound is those bytes over 3.35 TB/s (H100 SXM data sheet), the derivative rate
N^2 / time.  The card name, power limit and clocks are read in the same run.  Writes DIR/h100_grad_inputs.json."""
import argparse, json, math, os, statistics, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))

HBM = 3.35e12


def _data(N, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, (N, d))
    return X, np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)


def _time(variants, repeats):
    """variants: name -> (call, device-ms getter).  Warm-up, then alternating rounds; medians and spreads"""
    for call, _ in variants.values():
        call()
    host = {k: [] for k in variants}
    dev = {k: [] for k in variants}
    for _ in range(repeats):
        for k, (call, dms) in variants.items():
            t0 = time.perf_counter()
            call()
            host[k].append((time.perf_counter() - t0) * 1e3)
            dev[k].append(float(dms()))
    return {k: {"host_ms": host[k], "device_ms": dev[k], "device_ms_median": statistics.median(dev[k]),
                "host_ms_median": statistics.median(host[k]), "device_spread_ms": max(dev[k]) - min(dev[k])} for k in variants}


def _rates(r, N):
    byts = 2.0 * 8.0 * N * (N + 1) / 2.0
    for k, v in r.items():
        if not k.startswith("grad_inputs"):
            continue
        t = v["device_ms_median"] * 1e-3
        v.update(bytes_read=byts, achieved_bytes_per_s=byts / t, hbm_bound_ms=byts / HBM * 1e3,
                 share_of_hbm_bound=(byts / HBM) / t, derivatives_per_s=N * N / t, ps_per_derivative=t / (N * N) * 1e12)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=32768)
    ap.add_argument("--n-group", type=int, default=16384)
    ap.add_argument("--d", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    import gpb200

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    N, d = args.n, args.d
    res = {"card": card, "device": torch.cuda.get_device_name(0), "hbm_bytes_per_s_datasheet": HBM,
           "config": {"N": N, "d": d, "N_group": args.n_group, "repeats": args.repeats}, "cases": {}}
    X, y = _data(N, d, 0)
    for name, kern in (("SEIso", gpb200.SEIso(math.log(0.8), 0.0)),
                       ("Mat32Iso+RQIso", gpb200.Mat32Iso(math.log(0.8), 0.0) + gpb200.RQIso(0.0, -0.5, 0.0))):
        gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), kern, -1.0)
        e = gp._eng
        e.grad_prepare()
        tm = lambda k: (lambda: e.timings()[k])
        variants = {"grad_kernel": (lambda: e.grad_kernel(), tm("trace"))}

        def generic():
            e.set_option("gram_fast", 0)
            try:
                return e.grad_inputs()
            finally:
                e.set_option("gram_fast", 1)
        if name == "SEIso":
            variants["grad_inputs_fast"] = (lambda: e.grad_inputs(), tm("grad_inputs"))
            fast, gen = e.grad_inputs(), generic()
            res.setdefault("checks", {})["fast_vs_generic_rel"] = float(np.max(np.abs(fast - gen)) / np.max(np.abs(gen)))
        variants["grad_inputs_generic"] = (generic, tm("grad_inputs"))
        r = _time(variants, args.repeats)
        _rates(r, N)
        res["cases"][name] = r
        for k, v in r.items():
            extra = ("  %.2f of the HBM bound (%.2f ms)  %.1f ps/derivative" % (v["share_of_hbm_bound"], v["hbm_bound_ms"],
                                                                                 v["ps_per_derivative"])) if "bytes_read" in v else ""
            print("%-15s %-20s device %9.2f ms (spread %.2f)%s" % (name, k, v["device_ms_median"], v["device_spread_ms"], extra),
                  flush=True)
        del gp, e
        torch.cuda.empty_cache()
    Ng = args.n_group
    Xg, yg = _data(Ng, d, 1)
    grp = gpb200.LocalGroupEngine(4)
    gs = gpb200.GPE(Xg.T, yg, gpb200.MeanZero(), gpb200.SEIso(math.log(0.8), 0.0), -1.0, engine=grp)
    grp.grad_prepare()
    single = gpb200.GPE(Xg.T, yg, gpb200.MeanZero(), gpb200.SEIso(math.log(0.8), 0.0), -1.0)
    single._eng.grad_prepare()
    a, b = grp.grad_inputs(), single._eng.grad_inputs()
    res.setdefault("checks", {})["group4_vs_single_rel"] = float(np.max(np.abs(a - b)) / np.max(np.abs(b)))
    r = _time({"grad_kernel_group4": (lambda: grp.grad_kernel(), lambda: grp.timings()["trace"]),
               "grad_inputs_group4": (lambda: grp.grad_inputs(), lambda: grp.timings()["grad_inputs"]),
               "grad_inputs_single": (lambda: single._eng.grad_inputs(), lambda: single._eng.timings()["grad_inputs"])},
              args.repeats)
    _rates(r, Ng)
    res["cases"]["SEIso_group4_N%d" % Ng] = r
    for k, v in r.items():
        print("group of 4, N=%d %-20s device %9.2f ms (spread %.2f)" % (Ng, k, v["device_ms_median"], v["device_spread_ms"]), flush=True)
    grp.close()
    print(json.dumps(res["checks"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_grad_inputs.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(card)


if __name__ == "__main__":
    main()
