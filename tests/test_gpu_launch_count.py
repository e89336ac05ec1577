"""GPU: gpb200_launch_count / gpb200_fitc_launch_count against the device.  Every workload runs under torch.profiler with
CUDA activities; the kernels the profiler records in the window (copies and memsets left out) must equal the growth of the
handle's launch counter over the same calls.  Small sizes, but several predict chunks, FITC row chunks and FSA staging
chunks / test sub-chunks, since a miscount in a per-chunk loop only shows when the loop runs more than once."""
import json

import numpy as np
import pytest

from conftest import make_data

pytestmark = pytest.mark.gpu


def _device_kernels(fn, tmp_path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = tmp_path / "launches.pt.trace.json"
    prof.export_chrome_trace(str(path))
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    return sum(1 for e in events if e.get("cat") == "kernel" and not e.get("name", "").startswith(("Memcpy", "Memset")))


def _check(what, counter, steps, tmp_path):
    rows = []
    for name, fn in steps:
        c0 = counter()
        kernels = _device_kernels(fn, tmp_path)
        rows.append((name, counter() - c0, kernels))
    for name, counted, kernels in rows:
        print("launch count %-12s %-14s counted %6d  device %6d" % (what, name, counted, kernels))
    assert all(counted == kernels for _, counted, kernels in rows), rows


def test_profiler_sees_one_kernel_per_logdet(tmp_path):
    """calibration: gpb200_logdet enqueues exactly one kernel (the log-diagonal sum)"""
    import gpb200 as g
    X, y, _ = make_data(700, 3, 1)
    gp = g.GPE(X.T, y, g.MeanZero(), g.SEIso(0.3, 0.1), -0.5)
    _check("logdet", gp._eng.launch_count, [("logdet", gp._eng.logdet)], tmp_path)
    c0 = gp._eng.launch_count()
    assert _device_kernels(gp._eng.logdet, tmp_path) == 1 and gp._eng.launch_count() - c0 == 1


@pytest.mark.parametrize("kern", ["SEIso", "composite"])
def test_dense_launch_count(kern, tmp_path, monkeypatch):
    """SEIso takes the TMA Gram / trace kernels, the composite kernel the generic ones"""
    import gpb200 as g
    N, d = 700, 3
    X, y, Xs = make_data(N + 200, d, 2, m=600)
    k = g.SEIso(0.3, 0.1) if kern == "SEIso" else g.Mat32Iso(0.2, 0.1) + g.RQIso(0.4, -0.3, 0.2)
    gp = g.GPE(X[:N].T, y[:N], g.MeanConst(0.1), k, -0.5, capacity=N + 300)
    monkeypatch.setenv("GPB200_PREDICT_CHUNK", "256")                  # 3 chunks of test rows
    folds = [np.arange(i, N, 7) for i in range(3)]
    rng = np.random.default_rng(3)
    steps = [
        ("mll", gp.update_mll),
        ("grad", gp.update_dmll),
        ("predict var", lambda: gp.predict_f(Xs.T)),
        ("predict cov", lambda: gp.predict_f(Xs[:200].T, full_cov=True)),
        ("rand", lambda: gp.rand(Xs[:150].T, n=3, rng=rng)),
        ("LOO", gp.dlogp_LOO),
        ("CV folds", lambda: gp.dlogp_CVfold(folds)),
        ("append", lambda: gp.append(X[N:].T, y[N:])),
    ]
    _check(kern, gp._eng.launch_count, steps, tmp_path)


@pytest.mark.parametrize("fused", [0, 1])
def test_triangular_solve_launch_count(fused, tmp_path):
    import gpb200 as g
    X, y, _ = make_data(1500, 3, 4)
    eng = g.Engine(0)
    eng.set_option("trsv_fused", fused)
    gp = g.GPE(X.T, y, g.MeanZero(), g.SEIso(0.3, 0.1), -0.5, engine=eng)
    _check("trsv_fused=%d" % fused, eng.launch_count, [("mll", gp.update_mll), ("solve", lambda: eng.solve(y))], tmp_path)
    eng.close()


def test_row_sharded_group_launch_count(tmp_path):
    import gpb200 as g
    X, y, Xs = make_data(1500, 3, 5, m=300)
    grp = g.LocalGroupEngine(2, rb=1)
    gp = g.GPE(X.T, y, g.MeanConst(0.2), g.Mat32Iso(0.2, 0.1) + g.RQIso(0.4, -0.3, 0.2), -0.5, engine=grp)
    steps = [
        ("mll", gp.update_mll),
        ("grad", gp.update_dmll),
        ("predict var", lambda: gp.predict_f(Xs.T)),
        ("predict cov", lambda: gp.predict_f(Xs[:100].T, full_cov=True)),
    ]
    _check("2 ranks", grp.launch_count, steps, tmp_path)
    grp.close()


@pytest.mark.parametrize("strategy", ["FITC", "DTC", "SoR"])
def test_sparse_launch_count(strategy, tmp_path):
    import gpb200 as g
    rng = np.random.default_rng(6)
    N, M, d = 70000, 60, 2                                          # 3 row chunks (at most 32768 rows each)
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]]
    Xs = rng.standard_normal((300, d))
    gp = getattr(g, strategy)(X.T, Xu.T, y, g.MeanConst(0.1), g.SEIso(-0.3, 0.0), -1.0)
    eng = gp._eng
    steps = [
        ("mll", gp.update_mll),
        ("grad noise", eng.grad_noise),
        ("grad kernel", eng.grad_kernel),
        ("predict var", lambda: gp.predict_f(Xs.T)),
        ("predict cov", lambda: gp.predict_f(Xs[:100].T, full_cov=True)),
    ]
    _check(strategy, eng.launch_count, steps, tmp_path)


def test_fsa_launch_count(tmp_path):
    """N = 70 000 in blocks of 500: several staging chunks; 40 600 test points: the test rows are streamed in sub-chunks"""
    import gpb200 as g
    rng = np.random.default_rng(11)
    N, M, d = 70000, 64, 2
    X = rng.uniform(-3, 3, (N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]]
    order = np.argsort(X[:, 0] + 0.3 * X[:, 1])
    blocks = [order[i:i + 500] for i in range(0, N, 500)]
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), g.SEIso(-0.5, 0.0), -1.0)
    Xs = rng.uniform(-3, 3, (40600, d))
    bpred = [np.arange(j * 4, (j + 1) * 4) for j in range(150)]
    bcov = [np.arange(j * 4, (j + 1) * 4) for j in range(10)]
    eng = gp._eng
    steps = [
        ("mll", gp.update_mll),
        ("grad noise", eng.grad_noise),
        ("grad kernel", eng.grad_kernel),
        ("predict var", lambda: gp.predict_f(Xs.T, bpred)),
        ("predict cov", lambda: gp.predict_f(Xs[:40].T, bcov, full_cov=True)),
    ]
    _check("FSA", eng.launch_count, steps, tmp_path)
