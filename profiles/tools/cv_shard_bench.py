"""Times cross-validation per hyper-parameter (gpb200_cv_param) on row-sharded storage against a single-GPU handle, on one GPU
(the groups' ranks are virtual ranks of gpb200_group_create sharing the device):

  N = 16384, d = 3, kernel Mat32Iso + RQIso, logNoise = -0.5; paths: single GPU, groups of R = 2 and 4 (ownership block
  chosen by the engine).

  python profiles/tools/cv_shard_bench.py --out DIR [--n 16384] [--repeats 3]

Per path: factorize + mll + grad_prepare (untimed), one warm-up cv_param(0), then `repeats` rounds of cv_param(0) alternate
between the paths.  On groups the first cv_param(0) after a new grad_prepare also symmetrises the distributed K^-1 once:
after the timed rounds each group refactorises, and `sym_ms` = that first call - the median of the steady calls.  Every library call ends in a device
synchronise, so a host clock around the call times the device work.  Rates: 4 N^3 flop per cv_param on one GPU (two full
GEMMs), 3 N^3 on a group (Y' full, M_j lower triangle only).  The largest differences of Z_j alpha / diag(Z_j K^-1) and of a
cv_block(1) sub-block against the single-GPU path are recorded.  One extra profiled cv_param on the 2-rank group records
whether the K^-1 panel copies of the broadcasts actually overlap the M_j GEMMs.  Writes DIR/h100_cv_shard.json with the card
name, power limit and clocks read in the same run."""
import argparse, json, os, statistics, subprocess, sys, tempfile, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "gaussianprocesses.jl_b200"))


def overlap_of_copies_and_gemms(fn, tmp):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = os.path.join(tmp, "cv_trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    iv = lambda e: (float(e["ts"]), float(e["ts"]) + float(e.get("dur", 0.0)))
    copies = [iv(e) for e in ev if "Memcpy DtoD" in e.get("name", "")]
    gemms = [iv(e) for e in ev if e.get("cat") == "kernel" and "dgemm_nt" in e.get("name", "")]
    busy = []                                                       # union of the GEMM intervals (the ranks' GEMMs may overlap)
    for b0, b1 in sorted(gemms):
        if busy and b0 <= busy[-1][1]:
            busy[-1][1] = max(busy[-1][1], b1)
        else:
            busy.append([b0, b1])
    ov = sum(max(0.0, min(a1, b1) - max(a0, b0)) for a0, a1 in copies for b0, b1 in busy)
    return {"copies": len(copies), "copy_us": sum(b - a for a, b in copies), "gemms": len(gemms),
            "gemm_busy_us": sum(b - a for a, b in busy), "copy_time_under_gemms_us": ov}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--groups", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    import gpb200 as g

    def smi():
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    card_before = smi()
    N, d, ln = args.n, 3, -0.5
    rng = np.random.default_rng(N)
    X = rng.standard_normal((N, d))
    y = np.sin(X.sum(axis=1)) + 0.1 * rng.standard_normal(N)
    kern = g.Mat32Iso(0.2, 0.1) + g.RQIso(0.4, -0.3, 0.2)
    paths = {"single": g.Engine(0)}
    for R in args.groups:
        paths["group%d" % R] = g.LocalGroupEngine(R)
    gps = {}

    def timed(fn):
        t0 = time.perf_counter()
        out = fn()
        return (time.perf_counter() - t0) * 1e3, out

    first = {}
    for name, e in paths.items():
        gp = g.GPE(X.T, y, g.MeanZero(), kern, ln, engine=e)
        gp.update_target_and_dtarget()
        gps[name] = gp
        first[name] = timed(lambda: e.cv_param(0))[0]
    ms = {name: [] for name in paths}
    outs = {}
    for name, e in paths.items():                                   # warm-up
        e.cv_param(0)
    for _ in range(args.repeats):
        for name, e in paths.items():
            t, out = timed(lambda: e.cv_param(0))
            ms[name].append(t)
            outs[name] = out
    for name, e in paths.items():                                   # refactorise: the next call symmetrises K^-1 again
        if name != "single":
            gps[name].update_mll()
            e.grad_prepare()
            first[name] = timed(lambda: e.cv_param(0))[0]
    V = np.arange(N // 2 - 300, N // 2 + 300)
    blocks = {name: e.cv_block(1, V) for name, e in paths.items()}
    med = {name: statistics.median(v) for name, v in ms.items()}
    rows = {}
    for name in paths:
        flop = (4.0 if name == "single" else 3.0) * float(N) ** 3
        za, dz = outs[name]
        zs, ds = outs["single"]
        info = paths[name].storage_info() if name == "single" else paths[name].engines[0].storage_info()
        rows[name] = {"ms": ms[name], "ms_median": med[name], "first_call_ms": first[name],
                      "sym_ms": (first[name] - med[name]) if name != "single" else None,
                      "flop_per_call": flop, "tflops": flop / (med[name] * 1e-3) / 1e12, "rb": info["rb"],
                      "bytes_cv_rank0": info["bytes_cv"],
                      "max_rel_diff_vs_single": {
                          "Zj_alpha": float(np.max(np.abs(za - zs)) / np.max(np.abs(zs))),
                          "diag_ZjKinv": float(np.max(np.abs(dz - ds)) / np.max(np.abs(ds))),
                          "cv_block_1": float(np.max(np.abs(blocks[name] - blocks["single"])) / np.max(np.abs(blocks["single"])))}}
        print("%-8s cv_param %9.1f ms (first %9.1f ms)  %6.2f TFLOP/s over %dN^3  diff vs single %.2e"
              % (name, med[name], first[name], rows[name]["tflops"], 4 if name == "single" else 3,
                 max(rows[name]["max_rel_diff_vs_single"].values())), flush=True)
    overlap = None
    if "group2" in paths:
        with tempfile.TemporaryDirectory() as tmp:
            overlap = overlap_of_copies_and_gemms(lambda: paths["group2"].cv_param(0), tmp)
        print("group2 profiled cv_param: %s" % overlap, flush=True)
    for e in paths.values():
        e.close()
    res = {"card_before": card_before, "card_after": smi(), "device": torch.cuda.get_device_name(0),
           "config": {"N": N, "d": d, "kernel": "Mat32Iso + RQIso", "logNoise": ln, "param": 0, "repeats": args.repeats,
                      "group": "gpb200_group_create: R virtual ranks on the one device",
                      "timing": "host clock around cv_param (ends in a device synchronise); median after one warm-up, paths alternate"},
           "paths": rows, "group2_copy_gemm_overlap": overlap}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_cv_shard.json"), "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
