"""Times the DMMA NT GEMM (TMA loader, Engine.dgemm_nt_device) at the shape classes of one mll+gradient step at C2, so
that two builds of the library can be compared kernel for kernel:

  M=N=K=16384           top-level Schur update and top-level inverse merge
  M=16384, N=K=1024     mid-recursion Schur update
  M=32640, N=K=128      leaf panel TRSM

  python profiles/tools/gemm_ab.py --root TREE --out DIR [--seconds 1.0] [--repeats 3]

TREE is a source tree whose gaussianprocesses.jl_b200/lib/libgpb200.so has been built.  Per shape: warm-up, then
`--repeats` timed windows of at least `--seconds` of back-to-back launches each (CUDA events, one synchronise per
window).  Writes DIR/gemm_ab.json with ms per launch and TFLOP/s (2MNK flop per launch) of every window, their median,
and the library's in-run FP64 issue-rate probe (fp64_peak)."""
import argparse, json, math, os, statistics, sys

SHAPES = [(16384, 16384, 16384), (16384, 1024, 1024), (32640, 128, 128)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", required=True, help="tree whose gpb200 package (and built library) to import")
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--seconds", type=float, default=1.0, help="minimum GEMM time per timed window")
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, os.path.join(root, "gaussianprocesses.jl_b200"))
    import torch
    import gpb200
    if not os.path.realpath(gpb200.LIB_PATH).startswith(os.path.realpath(root) + os.sep):
        raise SystemExit("gpb200 was imported from outside --root: %s" % gpb200.LIB_PATH)

    eng = gpb200.Engine(0)
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    res = {"root": root, "lib": gpb200.LIB_PATH, "device": torch.cuda.get_device_name(0), "shapes": []}
    for M, N, K in SHAPES:
        A = torch.randn(M, K, dtype=torch.float64, device="cuda:0", generator=gen)
        B = torch.randn(N, K, dtype=torch.float64, device="cuda:0", generator=gen)
        C = torch.zeros(M, N, dtype=torch.float64, device="cuda:0")
        run = lambda reps: eng.dgemm_nt_device(0, M, N, K, -1.0, A.data_ptr(), K, B.data_ptr(), K, 1.0, C.data_ptr(), N,
                                               reps=reps)
        run(2)                                                       # module load, first-touch
        reps = max(1, math.ceil(args.seconds / (run(1) * 1e-3)))
        run(reps)                                                    # warm-up at the timed length
        ms = [run(reps) / reps for _ in range(args.repeats)]
        tf = [2.0 * M * N * K / (m * 1e-3) * 1e-12 for m in ms]
        res["shapes"].append({"M": M, "N": N, "K": K, "launches_per_window": reps, "ms_per_launch": ms,
                              "tflops": tf, "ms_median": statistics.median(ms), "tflops_median": statistics.median(tf)})
        print("M=%5d N=%5d K=%5d  %9.3f ms  %6.2f TFLOP/s  (%d launches x %d windows)"
              % (M, N, K, statistics.median(ms), statistics.median(tf), reps, args.repeats), flush=True)
        del A, B, C
        torch.cuda.empty_cache()
    res["fp64_peak"] = eng.fp64_peak()
    print("fp64_peak: DMMA %.1f  DFMA %.1f TFLOP/s" % (res["fp64_peak"]["dmma_tflops"], res["fp64_peak"]["dfma_tflops"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gemm_ab.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
