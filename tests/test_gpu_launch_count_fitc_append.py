"""GPU: the launch counter of gpb200_fitc_append against the kernels torch.profiler records (the
tests/test_gpu_launch_count.py pattern): the first append after a factorize (with the L_s L_s' rebuild and the sums over
every row), a later one, one over several staging chunks (at most 32768 rows each) and one that grows the N-sized buffers."""
import json

import numpy as np
import pytest

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
    with open(path) as fh:
        events = json.load(fh)["traceEvents"]
    return sum(1 for e in events if e.get("cat") == "kernel" and not e.get("name", "").startswith(("Memcpy", "Memset")))


@pytest.mark.parametrize("strategy", ["FITC", "SoR"])
def test_append_launch_count(strategy, tmp_path):
    import gpb200 as g
    rng = np.random.default_rng(6)
    N, M, d = 40000, 60, 2
    X = rng.standard_normal((N + 80000, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N + 80000)
    Xu = rng.uniform(-2, 2, (M, d))
    gp = getattr(g, strategy)(X[:N].T, Xu.T, y[:N], g.MeanZero(), g.SEIso(-0.3, 0.0), -1.0)
    eng = gp._eng
    steps = [("first", 5), ("second", 1), ("chunks", 70000), ("tile edge", 128)]
    rows, r0 = [], N
    for name, k in steps:
        c0 = eng.launch_count()
        kernels = _device_kernels(lambda: gp.append(X[r0:r0 + k].T, y[r0:r0 + k]), tmp_path)
        rows.append((name, eng.launch_count() - c0, kernels))
        r0 += k
    for r in rows:
        print("launch count %s %-10s counted %6d  device %6d" % (strategy, *r))
    assert all(c == k for _, c, k in rows), rows
